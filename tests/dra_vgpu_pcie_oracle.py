"""The C statement of kxpu_pcie_ports_mdev, kxpu_dra_slices_mdev_pcie and kxpu_dra_slices_vf_vgpu_pcie, next to
tests/pyref_vgpu_pcie.py: ctypes bindings of tests/dra_vgpu_pcie_oracle.c, compiled once per process and layout into a
temporary directory, so the tree stays read-only.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT
from kxpu_b200.binding import DRAMDEVPCIE_DTYPE, DRAVFVGPUPCIE_DTYPE, MDEVREC_DTYPE, PCIPATH_DTYPE, DraTaint

# the included checkers' record rules in order, the two port rules, then the taint rules
WHY = {"mdev": ["product", "mdev_type", "uuid", "parent", "pcie_root", "vendor", "device", "iommu_group", "product_len",
                "physfn", "physfn_device", "port_key", "port_orphan", "taint_since", "taint_duplicate"],
       "vf_vgpu": ["product", "type_key", "bdf", "parent", "pcie_root", "vendor", "device", "iommu_group", "type_id",
                   "product_len", "port_key", "port_orphan", "taint_since", "taint_duplicate"]}
_LIBS = {}


def lib(layout):
    if layout not in _LIBS:
        here = os.path.dirname(os.path.abspath(__file__))
        out = os.path.join(tempfile.mkdtemp(prefix="kxd_"), "libkxd_vgpu_pcie_%s.so" % layout)
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared"] +
                              (["-DKXD_VF"] if layout == "vf_vgpu" else []) +
                              ["-I", os.path.join(ROOT, "include"), "-I", here, "-o", out,
                               os.path.join(here, "dra_vgpu_pcie_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxd_dra_slices_vgpu_pcie.restype = C.c_int32
        L.kxd_dra_slices_vgpu_pcie.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint64, C.c_char_p, vp, sz, vp, sz,
                                               vp, vp, sz, C.POINTER(sz), vp, C.POINTER(sz), C.POINTER(C.c_int32)]
        if layout == "mdev":
            L.kxd_pcie_ports_mdev.restype = C.c_int32
            L.kxd_pcie_ports_mdev.argtypes = [vp, vp, sz, vp, vp, sz, vp, vp]
        _LIBS[layout] = L
    return _LIBS[layout]


def _b(x):
    return x.encode() if isinstance(x, str) else x


def pcie_ports_mdev(recs, paths, group_off, group_members):
    """(root_port, pcie_switch) uint64 arrays, or the failing status"""
    recs, paths = np.ascontiguousarray(recs, MDEVREC_DTYPE), np.ascontiguousarray(paths, PCIPATH_DTYPE)
    goff = np.ascontiguousarray(group_off, np.uint32)
    gmem = np.ascontiguousarray(group_members, np.uint32)
    G = len(goff) - 1
    rp, sw = np.zeros(max(G, 1), np.uint64), np.zeros(max(G, 1), np.uint64)
    rc = lib("mdev").kxd_pcie_ports_mdev(recs.ctypes.data, paths.ctypes.data, len(recs), goff.ctypes.data,
                                         gmem.ctypes.data, G, rp.ctypes.data, sw.ctypes.data)
    return rc if rc else (rp[:G], sw[:G])


def slices(layout, driver, pool, node, generation, domain, devs, taints=(), since=None):
    """(bytes, slice_off), or the failing status: -1 for a bad argument; for a record or a taint time outside the domain
    (-7, name of the first failing rule)"""
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == (DRAMDEVPCIE_DTYPE if layout == "mdev" else DRAVFVGPUPCIE_DTYPE)
    tab = (DraTaint * max(len(taints), 1))(*[DraTaint(_b(k), _b(v), _b(e)) for k, v, e in taints])
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
        assert since.size == len(devs) * len(taints)
    args = (_b(driver), _b(pool), _b(node), generation, _b(domain), devs.ctypes.data if len(devs) else None, len(devs),
            C.cast(tab, C.c_void_p), len(taints), None if since is None else since.ctypes.data)
    need, ns, why = C.c_size_t(0), C.c_size_t(0), C.c_int32(-1)
    f = lib(layout).kxd_dra_slices_vgpu_pcie
    rc = f(*args, None, 0, C.byref(need), None, C.byref(ns), C.byref(why))
    if rc == -7:
        return rc, WHY[layout][why.value] if why.value >= 0 else None
    if rc != -4:
        return rc
    out = np.empty(max(need.value, 1), np.uint8)
    offs = np.empty(ns.value + 1, np.uint64)
    rc = f(*args, out.ctypes.data, need.value, C.byref(need), offs.ctypes.data, C.byref(ns), C.byref(why))
    assert rc == 0, rc
    return out[:need.value].tobytes(), list(offs)
