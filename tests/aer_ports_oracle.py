"""ctypes binding of the AER port checker (tests/aer_ports_oracle.c): kxpu_aer_ports and kxpu_aer_ports_mdev restated in
C, the second statement next to tests/pyref_aer_ports.py.  The source is compiled once per process into a temporary
directory, so the tree stays read-only.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT
from kxpu_b200.binding import DEVREC_DTYPE, MDEVREC_DTYPE, PCIPATH_DTYPE

MAX_DEPTH = 8
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        here = os.path.dirname(os.path.abspath(__file__))
        out = os.path.join(tempfile.mkdtemp(prefix="kxa_"), "libkxa_aer_ports.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-I", here, "-o", out,
                               os.path.join(here, "aer_ports_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        for f in (L.kxa_aer_ports, L.kxa_aer_ports_mdev):
            f.restype = C.c_int32
            f.argtypes = [vp, vp, sz, vp, vp, vp, C.POINTER(C.c_uint32)]
        _LIB = L
    return _LIB


def aer_ports(recs, paths):
    """(port_off, port_of, port_key) numpy arrays; recs DEVREC_DTYPE (kxpu_aer_ports) or MDEVREC_DTYPE (_mdev)"""
    recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths, PCIPATH_DTYPE)
    assert recs.dtype in (DEVREC_DTYPE, MDEVREC_DTYPE) and len(recs) == len(paths)
    n = len(recs)
    cap = max((MAX_DEPTH - 1) * n, 1)
    off, of, key = np.zeros(n + 1, np.uint32), np.zeros(cap, np.uint32), np.zeros(cap, np.uint64)
    nk = C.c_uint32(0)
    f = lib().kxa_aer_ports_mdev if recs.dtype == MDEVREC_DTYPE else lib().kxa_aer_ports
    assert f(recs.ctypes.data, paths.ctypes.data, n, off.ctypes.data, of.ctypes.data, key.ctypes.data, C.byref(nk)) == 0
    return off, of[:off[n]], key[:nk.value]
