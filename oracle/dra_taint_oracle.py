"""ctypes binding of the DRA taint CPU oracle (oracle/kxpu_dra_taint_oracle.c): the checker of kxpu_dra_slices_taint
and kxpu_dra_slices_mdev_taint.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import dra_mdev_oracle, dra_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_dra_taint_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_dra_taint_oracle.so")
_LIB = None

DRADEV_DTYPE = dra_oracle.DRADEV_DTYPE
DRAMDEV_DTYPE = dra_mdev_oracle.DRAMDEV_DTYPE
WHY = dra_oracle.WHY + ["taint_since"]
WHY_MDEV = dra_mdev_oracle.WHY + ["taint_since"]


def build():
    deps = [_SRC, os.path.join(_HERE, "kxpu_dra_mdev_oracle.c"), os.path.join(_HERE, "kxpu_dra_oracle.c"),
            os.path.join(_HERE, "..", "include", "kxpu.h")]
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        vp, sz, s = C.c_void_p, C.c_size_t, C.c_char_p
        for name in ("kxo_dra_slices_taint", "kxo_dra_slices_mdev_taint"):
            f = getattr(L, name)
            f.restype = C.c_int32
            f.argtypes = [s, s, s, C.c_uint64, vp, sz, s, s, s, vp, vp, sz, C.POINTER(sz), vp, C.POINTER(sz),
                          C.POINTER(C.c_int32)]
        _LIB = L
    return _LIB


def _b(x):
    return x.encode() if isinstance(x, str) else x


def _slices(fn, dtype, why_names, driver, pool, node, generation, devs, key, value, effect, since):
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == dtype
    dp = devs.ctypes.data if len(devs) else None
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
        assert since.shape == (len(devs),)
    sp = None if since is None else since.ctypes.data
    need, ns, why = C.c_size_t(0), C.c_size_t(0), C.c_int32(-1)
    args = (_b(driver), _b(pool), _b(node), generation, dp, len(devs), _b(key), _b(value), _b(effect), sp)
    rc = fn(*args, None, 0, C.byref(need), None, C.byref(ns), C.byref(why))
    if rc == -7:
        return rc, why_names[why.value] if why.value >= 0 else None
    if rc != -4:
        return rc
    out = np.empty(max(need.value, 1), np.uint8)
    offs = np.empty(ns.value + 1, np.uint64)
    rc = fn(*args, out.ctypes.data, need.value, C.byref(need), offs.ctypes.data, C.byref(ns), C.byref(why))
    assert rc == 0, rc
    return out[:need.value].tobytes(), offs


def dra_slices_taint(driver, pool, node, generation, devs, key, value, effect, since):
    """(bytes, slice_off) of kxo_dra_slices_taint, or the failing status: -1 for a bad argument; for a record or a
    taint time outside the domain (-7, name of the first failing rule).  since: None or one int64 per device."""
    return _slices(lib().kxo_dra_slices_taint, DRADEV_DTYPE, WHY, driver, pool, node, generation, devs, key, value,
                   effect, since)


def dra_slices_mdev_taint(driver, pool, node, generation, devs, key, value, effect, since):
    """the same for a pool of vGPUs (kxo_dra_slices_mdev_taint)"""
    return _slices(lib().kxo_dra_slices_mdev_taint, DRAMDEV_DTYPE, WHY_MDEV, driver, pool, node, generation, devs, key,
                   value, effect, since)
