"""ctypes binding of the PCIe topology CPU oracle (oracle/kxpu_pcie_oracle.c): the checker of kxpu_pcie_tree and
kxpu_preferred_allocation_pcie, and of the path grammar of one record.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C

import numpy as np

from . import oracle as O

NO_NODE = 0xFFFFFFFF
MAX_DEPTH = 8


def _p(a):
    return a.ctypes.data if a is not None and len(a) else None


def parse(rec, path):
    """The chain keys of one record (a DEVREC_DTYPE row and a PCIPATH_DTYPE row), [] when the path is unknown."""
    rec = np.ascontiguousarray(np.asarray(rec).reshape(1))
    path = np.ascontiguousarray(np.asarray(path).reshape(1))
    chain = np.zeros(MAX_DEPTH, np.uint64)
    n = O.lib().kxo_pcie_parse(rec.ctypes.data, path.ctypes.data, chain.ctypes.data)
    return [int(k) for k in chain[:n]]


def tree(recs, paths, group_off, group_members):
    """kxo_pcie_tree: dict(group_node, key, parent, depth), or None when the group CSR is invalid."""
    recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths)
    group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
    group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
    G = len(group_off) - 1
    cap = max(MAX_DEPTH * G, 1)
    gnode = np.zeros(max(G, 1), np.uint32)
    key, parent, depth = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32), np.zeros(cap, np.uint8)
    nn = C.c_uint32(0)
    rc = O.lib().kxo_pcie_tree(_p(recs), _p(paths), len(recs), group_off.ctypes.data, _p(group_members), G,
                               gnode.ctypes.data, key.ctypes.data, parent.ctypes.data, depth.ctypes.data, C.byref(nn))
    if rc != 0:
        return None
    n = nn.value
    return dict(group_node=gnode[:G], key=key[:n], parent=parent[:n], depth=depth[:n])


def preferred_allocation_pcie(dev_numa, dev_node, parent, depth, requests):
    """[(available, must-include, size)] -> one position list per request, or None when a request or the forest is
    invalid.  dev_node None: no PCIe information."""
    from kxpu_b200.binding import pref_requests
    a = pref_requests(requests)
    dev_numa = np.ascontiguousarray(dev_numa, dtype=np.uint64)
    dn = None if dev_node is None else np.ascontiguousarray(dev_node, dtype=np.uint32)
    parent = np.ascontiguousarray(parent, dtype=np.uint32)
    depth = np.ascontiguousarray(depth, dtype=np.uint8)
    out = np.zeros(max(int(a["size"].sum()), 1), np.uint32)
    out_off = np.zeros(len(requests) + 1, np.uint32)
    rc = O.lib().kxo_preferred_allocation_pcie(_p(dev_numa), _p(dn), len(dev_numa), _p(parent), _p(depth), len(parent),
                                               a["avail_off"].ctypes.data, a["avail"].ctypes.data,
                                               a["must_off"].ctypes.data, a["must"].ctypes.data, a["size"].ctypes.data,
                                               len(requests), out.ctypes.data, out_off.ctypes.data)
    if rc != 0:
        return None
    return [out[out_off[q]:out_off[q + 1]].tolist() for q in range(len(requests))]
