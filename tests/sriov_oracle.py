"""ctypes binding of the SR-IOV C checker (tests/sriov_oracle.c): kxpu_sriov and kxpu_pcie_tree_sriov restated in C, the
second statement next to tests/pyref_sriov.py.  The source is compiled once per process into a temporary directory, so
the tree stays read-only; the chains of the forest come from the PCIe oracle's path parse (oracle/pcie_oracle.py).

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
        out = os.path.join(tempfile.mkdtemp(prefix="kxs_"), "libkxs_sriov.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "sriov_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxs_sriov.restype = C.c_int
        L.kxs_sriov.argtypes = [vp, sz, vp, vp, sz, vp, vp, sz, vp, vp, vp]
        L.kxs_pcie_tree_sriov.restype = C.c_int
        L.kxs_pcie_tree_sriov.argtypes = [vp, vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, vp, C.POINTER(C.c_uint32)]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data if len(a) else None


def sriov(rules, recs, srs, group_off, group_members):
    """dict(pf_of, numvfs, group_sriov) as lists, or None for an invalid CSR."""
    ra = rules_array(rules)
    recs, srs = np.ascontiguousarray(recs), np.ascontiguousarray(srs)
    goff = np.ascontiguousarray(group_off, dtype=np.uint32)
    gmem = np.ascontiguousarray(group_members, dtype=np.uint32)
    n, G = len(recs), len(goff) - 1
    pf_of, nv, gs = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint32), np.zeros(max(G, 1), np.uint32)
    if lib().kxs_sriov(_p(ra), len(ra), _p(recs), _p(srs), n, goff.ctypes.data, _p(gmem), G, pf_of.ctypes.data,
                       nv.ctypes.data, gs.ctypes.data) != 0:
        return None
    return dict(pf_of=pf_of[:n].tolist(), numvfs=nv[:n].tolist(), group_sriov=gs[:G].tolist())


def tree(recs, paths, group_off, group_members, pf_of):
    """dict(group_node, key, parent, depth) as lists, or None for an invalid CSR or pf_of."""
    recs = np.ascontiguousarray(recs)
    n = len(recs)
    chain, clen = np.zeros((max(n, 1), MAX_DEPTH), np.uint64), np.zeros(max(n, 1), np.uint8)
    for i in range(n):
        c = PO.parse(recs[i], paths[i])
        chain[i, :len(c)], clen[i] = c, len(c)
    goff = np.ascontiguousarray(group_off, dtype=np.uint32)
    gmem = np.ascontiguousarray(group_members, dtype=np.uint32)
    pf = np.ascontiguousarray(pf_of, dtype=np.uint32)
    G = len(goff) - 1
    cap = max(MAX_DEPTH * G, 1)
    gnode = np.zeros(max(G, 1), np.uint32)
    key, parent, depth = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32), np.zeros(cap, np.uint8)
    nn = C.c_uint32(0)
    if lib().kxs_pcie_tree_sriov(_p(recs), chain.ctypes.data, clen.ctypes.data, n, goff.ctypes.data, _p(gmem), G, _p(pf),
                                 gnode.ctypes.data, key.ctypes.data, parent.ctypes.data, depth.ctypes.data,
                                 C.byref(nn)) != 0:
        return None
    m = nn.value
    return dict(group_node=gnode[:G].tolist(), key=key[:m].tolist(), parent=parent[:m].tolist(), depth=depth[:m].tolist())
