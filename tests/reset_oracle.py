"""ctypes binding of the reset C checker (tests/reset_oracle.c): kxpu_reset_check restated in C, the second statement
next to tests/pyref_reset.py.  The source is compiled once per process into a temporary directory, so the tree stays
read-only; the chains come from the PCIe oracle's path parse (oracle/pcie_oracle.py).

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT
from oracle import pcie_oracle as PO
from kxpu_b200.binding import rules_array

_LIB = None
MAX_DEPTH = 8


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="kxs_"), "libkxs_reset.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "reset_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxs_reset_check.restype = C.c_int
        L.kxs_reset_check.argtypes = [vp, sz, vp, vp, vp, vp, sz, C.c_uint32, vp, vp, sz, vp, vp, vp]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data if len(a) else None


def chains(recs, paths):
    """(chain [n, 8] u64, clen [n] u8) from the PCIe oracle's parse of each record"""
    n = len(recs)
    chain, clen = np.zeros((max(n, 1), MAX_DEPTH), np.uint64), np.zeros(max(n, 1), np.uint8)
    for i in range(n):
        c = PO.parse(recs[i], paths[i])
        chain[i, :len(c)], clen[i] = c, len(c)
    return chain, clen


def reset_check(rules, recs, paths, rrs, allow, group_off, group_members, parsed=None):
    """dict(methods, set_verdict, group_reset) as lists, or None for an invalid CSR.  parsed: chains(recs, paths), when
    the caller has it already."""
    ra = rules_array(rules)
    recs, rrs = np.ascontiguousarray(recs), np.ascontiguousarray(rrs)
    chain, clen = parsed if parsed is not None else chains(recs, paths)
    goff = np.ascontiguousarray(group_off, dtype=np.uint32)
    gmem = np.ascontiguousarray(group_members, dtype=np.uint32)
    n, G = len(recs), len(goff) - 1
    meth, sv, gr = np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.uint32), np.zeros(max(G, 1), np.uint32)
    if lib().kxs_reset_check(_p(ra), len(ra), _p(recs), chain.ctypes.data, clen.ctypes.data, _p(rrs), n, allow,
                             goff.ctypes.data, _p(gmem), G, meth.ctypes.data, sv.ctypes.data, gr.ctypes.data) != 0:
        return None
    return dict(methods=meth[:n].tolist(), set_verdict=sv[:n].tolist(), group_reset=gr[:G].tolist())
