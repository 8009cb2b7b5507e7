"""The C statement of kxpu_vf_vgpu_drift, next to tests/pyref_vf_vgpu_health.py: a ctypes binding of
tests/vf_vgpu_health_oracle.c, compiled once per process with tests/vf_vgpu_oracle.c (whose current-type rule it uses)
into a temporary directory, so the tree stays read-only.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT

_LIB = None
_HERE = os.path.dirname(os.path.abspath(__file__))


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="kxv_"), "libkxv_vf_vgpu_health.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(_HERE, "vf_vgpu_health_oracle.c"), os.path.join(_HERE, "vf_vgpu_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxv_vf_vgpu_drift.restype = C.c_int
        L.kxv_vf_vgpu_drift.argtypes = [vp, vp, sz, vp, vp, sz, vp, vp, vp]
        _LIB = L
    return _LIB


def vf_vgpu_drift(recs_vt, type_was, group_off, group_members):
    """dict(type_now, status_now, group_first) as lists, or None where the call returns KXPU_E_INVALID."""
    recs_vt = np.ascontiguousarray(recs_vt)
    was = np.ascontiguousarray(type_was, dtype=np.uint32)
    goff = np.ascontiguousarray(group_off, dtype=np.uint32)
    gmem = np.ascontiguousarray(group_members, dtype=np.uint32)
    n, G = len(recs_vt), len(goff) - 1
    now, st, first = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint8), np.zeros(max(G, 1), np.uint32)
    if lib().kxv_vf_vgpu_drift(recs_vt.ctypes.data if n else None, was.ctypes.data if n else None, n, goff.ctypes.data,
                               gmem.ctypes.data if len(gmem) else None, G, now.ctypes.data, st.ctypes.data,
                               first.ctypes.data) != 0:
        return None
    return dict(type_now=now[:n].tolist(), status_now=st[:n].tolist(), group_first=first[:G].tolist())
