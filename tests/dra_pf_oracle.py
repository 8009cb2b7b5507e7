"""The C statement of kxpu_dra_slices_pf, next to tests/pyref_dra_pf.py: a ctypes binding of tests/dra_pf_oracle.c,
compiled once per process into a temporary directory, so the tree stays read-only.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT
from kxpu_b200.binding import DRADEVPF_DTYPE, DraTaint

# the header's record rules in order, then the taint rules
WHY = ["product", "bdf", "pcie_root", "vendor", "device", "iommu_group", "product_len", "physfn", "physfn_device",
       "taint_since", "taint_duplicate"]
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="kxd_"), "libkxd_dra_pf.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "dra_pf_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxd_dra_slices_pf.restype = C.c_int32
        L.kxd_dra_slices_pf.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint64, vp, sz, vp, sz, vp, vp, sz,
                                        C.POINTER(sz), vp, C.POINTER(sz), C.POINTER(C.c_int32)]
        _LIB = L
    return _LIB


def _b(x):
    return x.encode() if isinstance(x, str) else x


def dra_slices_pf(driver, pool, node, generation, devs, taints=(), since=None):
    """(bytes, slice_off), or the failing status: -1 for a bad argument; for a record or a taint time outside the domain
    (-7, name of the first failing rule).  taints: [(key, value, effect)]; since: None or an int64 [n, len(taints)]
    array."""
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == DRADEVPF_DTYPE
    tab = (DraTaint * max(len(taints), 1))(*[DraTaint(_b(k), _b(v), _b(e)) for k, v, e in taints])
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
        assert since.size == len(devs) * len(taints)
    args = (_b(driver), _b(pool), _b(node), generation, devs.ctypes.data if len(devs) else None, len(devs),
            C.cast(tab, C.c_void_p), len(taints), None if since is None else since.ctypes.data)
    need, ns, why = C.c_size_t(0), C.c_size_t(0), C.c_int32(-1)
    f = lib().kxd_dra_slices_pf
    rc = f(*args, None, 0, C.byref(need), None, C.byref(ns), C.byref(why))
    if rc == -7:
        return rc, WHY[why.value] if why.value >= 0 else None
    if rc != -4:
        return rc
    out = np.empty(max(need.value, 1), np.uint8)
    offs = np.empty(ns.value + 1, np.uint64)
    rc = f(*args, out.ctypes.data, need.value, C.byref(need), offs.ctypes.data, C.byref(ns), C.byref(why))
    assert rc == 0, rc
    return out[:need.value].tobytes(), offs
