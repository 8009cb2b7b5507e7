"""ctypes binding of the AER CPU oracle (oracle/kxpu_aer_oracle.c): the checker of kxpu_aer_health,
kxpu_dra_slices_taints and kxpu_dra_slices_mdev_taints.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle import dra_taint_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_aer_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_aer_oracle.so")
_LIB = None

DRADEV_DTYPE = dra_taint_oracle.DRADEV_DTYPE
DRAMDEV_DTYPE = dra_taint_oracle.DRAMDEV_DTYPE
WHY = dra_taint_oracle.WHY + ["taint_duplicate"]
WHY_MDEV = dra_taint_oracle.WHY_MDEV + ["taint_duplicate"]
UNKNOWN = (1 << 64) - 1


class Taint(C.Structure):
    _fields_ = [("key", C.c_char_p), ("value", C.c_char_p), ("effect", C.c_char_p)]


def build():
    deps = [_SRC, os.path.join(_HERE, "kxpu_dra_taint_oracle.c"), os.path.join(_HERE, "kxpu_dra_mdev_oracle.c"),
            os.path.join(_HERE, "kxpu_dra_oracle.c"), os.path.join(_HERE, "..", "include", "kxpu.h")]
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        vp, sz, s = C.c_void_p, C.c_size_t, C.c_char_p
        L.kxo_aer_health.restype = C.c_int32
        L.kxo_aer_health.argtypes = [vp, sz, vp, vp, sz, C.c_uint64, C.c_uint64, vp, vp, sz, vp, vp]
        for name in ("kxo_dra_slices_taints", "kxo_dra_slices_mdev_taints"):
            f = getattr(L, name)
            f.restype = C.c_int32
            f.argtypes = [s, s, s, C.c_uint64, vp, sz, vp, sz, vp, vp, sz, C.POINTER(sz), vp, C.POINTER(sz),
                          C.POINTER(C.c_int32)]
        _LIB = L
    return _LIB


def _b(x):
    return x.encode() if isinstance(x, str) else x


def aer_health(text, file_off, file_len, fatal_limit, nonfatal_limit, group_off, group_members):
    """(totals, group_aer) of kxo_aer_health, or the failing status.  Arguments as Kxpu.aer_health."""
    t = np.frombuffer(bytes(text), np.uint8)
    file_off = np.ascontiguousarray(file_off, dtype=np.uint64)
    file_len = np.ascontiguousarray(file_len, dtype=np.uint32)
    group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
    group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
    n, G = len(file_off) // 2, len(group_off) - 1
    totals = np.empty(max(2 * n, 1), np.uint64)
    group_aer = np.empty(max(G, 1), np.uint8)
    rc = lib().kxo_aer_health(t.ctypes.data if len(t) else None, len(t), file_off.ctypes.data if n else None,
                              file_len.ctypes.data if n else None, n, fatal_limit, nonfatal_limit, group_off.ctypes.data,
                              group_members.ctypes.data if len(group_members) else None, G, totals.ctypes.data,
                              group_aer.ctypes.data)
    if rc:
        return rc
    return totals[:2 * n], group_aer[:G]


def _slices(fn, dtype, why_names, driver, pool, node, generation, devs, taints, since):
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == dtype
    dp = devs.ctypes.data if len(devs) else None
    tab = (Taint * max(len(taints), 1))(*[Taint(_b(k), _b(v), _b(e)) for k, v, e in taints])
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
        assert since.size == len(devs) * len(taints)
    sp = None if since is None else since.ctypes.data
    need, ns, why = C.c_size_t(0), C.c_size_t(0), C.c_int32(-1)
    args = (_b(driver), _b(pool), _b(node), generation, dp, len(devs), C.cast(tab, C.c_void_p), len(taints), sp)
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


def dra_slices_taints(driver, pool, node, generation, devs, taints, since):
    """(bytes, slice_off) of kxo_dra_slices_taints, or the failing status: -1 for a bad argument; for a record or a
    taint outside the domain (-7, name of the first failing rule).  taints: [(key, value, effect)]; since: None or an
    int64 [n, len(taints)] array."""
    return _slices(lib().kxo_dra_slices_taints, DRADEV_DTYPE, WHY, driver, pool, node, generation, devs, taints, since)


def dra_slices_mdev_taints(driver, pool, node, generation, devs, taints, since):
    """the same for a pool of vGPUs (kxo_dra_slices_mdev_taints)"""
    return _slices(lib().kxo_dra_slices_mdev_taints, DRAMDEV_DTYPE, WHY_MDEV, driver, pool, node, generation, devs,
                   taints, since)
