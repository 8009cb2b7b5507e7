"""ctypes binding of the NUMA topology CPU oracle (oracle/kxpu_topo_oracle.c): the checker of kxpu_classify_topo,
kxpu_classify_mdev_topo, kxpu_lw_encode_topo and kxpu_preferred_allocation.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import numpy as np

from . import oracle as O
from . import xpu_oracle as XO


def classify_topo(rules, recs: np.ndarray, mdev=False):
    """kxo_classify_topo / kxo_classify_mdev_topo: the classify dict plus dev_rule and group_numa; None when the rule
    list is invalid."""
    ra = XO.rules_array(rules)
    assert recs.dtype.itemsize == (128 if mdev else 64)
    L = O.lib()
    return O.classify_call(L.kxo_classify_mdev_topo if mdev else L.kxo_classify_topo,
                           (ra.ctypes.data if len(ra) else None, len(ra)), recs, dev=[("dev_rule", np.uint8)],
                           group=[("group_numa", np.uint64)])[1]


def lw_encode_topo(groups, healthy=None, masks=None) -> bytes:
    L = O.lib()
    groups = np.ascontiguousarray(groups, dtype=np.uint32)
    hp = np.ascontiguousarray(healthy, dtype=np.uint8).ctypes.data if healthy is not None else None
    mp = np.ascontiguousarray(masks, dtype=np.uint64) if masks is not None else None
    need = L.kxo_lw_encode_topo(groups.ctypes.data, hp, None if mp is None else mp.ctypes.data, len(groups), None, 0)
    out = np.empty(max(need, 1), np.uint8)
    got = L.kxo_lw_encode_topo(groups.ctypes.data, hp, None if mp is None else mp.ctypes.data, len(groups),
                               out.ctypes.data, need)
    assert got == need
    return out[:need].tobytes()


def preferred_allocation(dev_numa, requests):
    """[(available, must-include, size)] -> one position list per request, or None when a request is invalid."""
    L = O.lib()
    from kxpu_b200.binding import pref_requests
    a = pref_requests(requests)
    dev_numa = np.ascontiguousarray(dev_numa, dtype=np.uint64)
    out = np.zeros(max(int(a["size"].sum()), 1), np.uint32)
    out_off = np.zeros(len(requests) + 1, np.uint32)
    rc = L.kxo_preferred_allocation(dev_numa.ctypes.data if len(dev_numa) else None, len(dev_numa),
                                    a["avail_off"].ctypes.data, a["avail"].ctypes.data, a["must_off"].ctypes.data,
                                    a["must"].ctypes.data, a["size"].ctypes.data, len(requests), out.ctypes.data,
                                    out_off.ctypes.data)
    if rc != 0:
        return None
    return [out[out_off[q]:out_off[q + 1]].tolist() for q in range(len(requests))]
