"""ctypes binding of the mdev PCIe forest's C checker (tests/pcie_mdev_oracle.c): kxpu_pcie_tree_mdev restated in C, the
second statement next to tests/pyref_pcie_mdev.py.  The source is compiled once per process into a temporary directory,
so the tree stays read-only.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT

_LIB = None
MAX_DEPTH = 8


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="kxm_"), "libkxo_pcie_mdev.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "pcie_mdev_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxo_pcie_parse_mdev.restype = C.c_int32
        L.kxo_pcie_parse_mdev.argtypes = [vp, vp, vp]
        L.kxo_pcie_tree_mdev.restype = C.c_int32
        L.kxo_pcie_tree_mdev.argtypes = [vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, C.POINTER(C.c_uint32)]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data if len(a) else None


def parse(rec, path):
    """The chain keys of one record (an MDEVREC_DTYPE row and a PCIPATH_DTYPE row), [] when the path is unknown."""
    rec = np.ascontiguousarray(np.asarray(rec).reshape(1))
    path = np.ascontiguousarray(np.asarray(path).reshape(1))
    chain = np.zeros(MAX_DEPTH, np.uint64)
    n = lib().kxo_pcie_parse_mdev(rec.ctypes.data, path.ctypes.data, chain.ctypes.data)
    return [int(k) for k in chain[:n]]


def tree(recs, paths, group_off, group_members):
    """kxo_pcie_tree_mdev: dict(group_node, key, parent, depth) as lists, or None when the group CSR is invalid."""
    recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths)
    goff = np.ascontiguousarray(group_off, dtype=np.uint32)
    gmem = np.ascontiguousarray(group_members, dtype=np.uint32)
    G = len(goff) - 1
    cap = max(MAX_DEPTH * G, 1)
    gnode = np.zeros(max(G, 1), np.uint32)
    key, parent, depth = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32), np.zeros(cap, np.uint8)
    nn = C.c_uint32(0)
    if lib().kxo_pcie_tree_mdev(_p(recs), _p(paths), len(recs), goff.ctypes.data, _p(gmem), G, gnode.ctypes.data,
                                key.ctypes.data, parent.ctypes.data, depth.ctypes.data, C.byref(nn)) != 0:
        return None
    m = nn.value
    return dict(group_node=gnode[:G].tolist(), key=key[:m].tolist(), parent=parent[:m].tolist(), depth=depth[:m].tolist())
