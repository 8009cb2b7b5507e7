"""ctypes binding of the vGPU DRA ResourceSlice CPU oracle (oracle/kxpu_dra_mdev_oracle.c): the checker of
kxpu_dra_slices_mdev.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_dra_mdev_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_dra_mdev_oracle.so")
_LIB = None

# kxpu_dramdev, as include/kxpu.h declares it (tests compare it with the product binding's dtype)
DRAMDEV_DTYPE = np.dtype([("product", "u1", (64,)), ("mdev_type", "S40"), ("uuid", "S36"), ("iommu_group", "<u4"),
                          ("parent", "S16"), ("pcie_root", "S16"), ("vendor", "S8"), ("device", "S8"), ("numa_mask", "<u8"),
                          ("product_len", "u1"), ("reserved", "u1", (7,))])
assert DRAMDEV_DTYPE.itemsize == 208
WHY = ["product", "mdev_type", "uuid", "parent", "pcie_root", "vendor", "device", "iommu_group", "product_len"]


def build():
    deps = [_SRC, os.path.join(_HERE, "kxpu_dra_oracle.c"), os.path.join(_HERE, "..", "include", "kxpu.h")]
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxo_dra_slices_mdev.restype = C.c_int32
        L.kxo_dra_slices_mdev.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint64, vp, sz, vp, sz, C.POINTER(sz), vp,
                                          C.POINTER(sz), C.POINTER(C.c_int32)]
        _LIB = L
    return _LIB


def _b(s):
    return s.encode() if isinstance(s, str) else s


def dra_slices_mdev(driver, pool, node, generation, devs):
    """(bytes, slice_off) of kxo_dra_slices_mdev, or the failing status: -1 for a bad argument; for a record outside
    the domain (-7, name of the first failing rule)."""
    L = lib()
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == DRAMDEV_DTYPE
    dp = devs.ctypes.data if len(devs) else None
    need, ns, why = C.c_size_t(0), C.c_size_t(0), C.c_int32(-1)
    args = (_b(driver), _b(pool), _b(node), generation, dp, len(devs))
    rc = L.kxo_dra_slices_mdev(*args, None, 0, C.byref(need), None, C.byref(ns), C.byref(why))
    if rc == -7:
        return rc, WHY[why.value] if why.value >= 0 else None
    if rc != -4:
        return rc
    out = np.empty(max(need.value, 1), np.uint8)
    offs = np.empty(ns.value + 1, np.uint64)
    rc = L.kxo_dra_slices_mdev(*args, out.ctypes.data, need.value, C.byref(need), offs.ctypes.data, C.byref(ns),
                               C.byref(why))
    assert rc == 0, rc
    return out[:need.value].tobytes(), offs
