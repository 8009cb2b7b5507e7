"""ctypes binding of the NUMA topology CPU oracle (oracle/kxpu_topo_oracle.c): the checker of kxpu_classify_topo,
kxpu_classify_mdev_topo, kxpu_lw_encode_topo and kxpu_preferred_allocation.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.  The library links against
libkxpu_mdev_oracle.so and libkxpu_xpu_oracle.so (the grouping), so mdev_oracle.build() runs first.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import mdev_oracle as MO
from . import xpu_oracle as XO
from .oracle import ClassifyOut

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_topo_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_topo_oracle.so")
_LIB = None


def build():
    MO.build()
    deps = [_SRC, os.path.join(_HERE, "libkxpu_mdev_oracle.so"), os.path.join(_HERE, "libkxpu_xpu_oracle.so"),
            os.path.join(_HERE, "..", "include", "kxpu.h")]
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC,
                           "-L" + _HERE, "-lkxpu_mdev_oracle", "-lkxpu_xpu_oracle", "-lkxpu_oracle", "-Wl,-rpath,$ORIGIN"])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        vp, sz = C.c_void_p, C.c_size_t
        for f in (L.kxo_classify_topo, L.kxo_classify_mdev_topo):
            f.restype = C.c_int32
            f.argtypes = [vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp]
        L.kxo_lw_encode_topo.restype = sz
        L.kxo_lw_encode_topo.argtypes = [vp, vp, vp, sz, vp, sz]
        L.kxo_preferred_allocation.restype = C.c_int32
        L.kxo_preferred_allocation.argtypes = [vp, sz, vp, vp, vp, vp, vp, sz, vp, vp]
        _LIB = L
    return _LIB


def classify_topo(rules, recs: np.ndarray, mdev=False):
    """kxo_classify_topo / kxo_classify_mdev_topo: the classify dict plus dev_rule and group_numa; None when the rule
    list is invalid."""
    L = lib()
    ra = XO.rules_array(rules)
    n = len(recs)
    recs = np.ascontiguousarray(recs)
    assert recs.dtype.itemsize == (128 if mdev else 64)
    arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                dev_groups=np.empty(n, np.uint32))
    dev_rule = np.empty(max(n, 1), np.uint8)
    gnuma = np.empty(max(n, 1), np.uint64)
    out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
    fn = L.kxo_classify_mdev_topo if mdev else L.kxo_classify_topo
    rc = fn(ra.ctypes.data if len(ra) else None, len(ra), recs.ctypes.data, n, C.byref(out), dev_rule.ctypes.data,
            gnuma.ctypes.data)
    if rc != 0:
        return None
    g, d, a = out.n_groups, out.n_devids, out.n_accepted
    return dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d],
                group_numa=gnuma[:g])


def lw_encode_topo(groups, healthy=None, masks=None) -> bytes:
    L = lib()
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
    L = lib()
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
