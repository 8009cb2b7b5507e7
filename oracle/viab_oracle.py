"""ctypes binding of the IOMMU group viability CPU oracle (oracle/kxpu_viab_oracle.c): the checker of
kxpu_classify_viable.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.  The library links against
libkxpu_topo_oracle.so and libkxpu_xpu_oracle.so (the grouping and the masks), so topo_oracle.build() runs first.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import topo_oracle as TO
from . import xpu_oracle as XO
from .oracle import ClassifyOut

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_viab_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_viab_oracle.so")
_LIB = None

VIABLE = 0xFFFFFFFF


def build():
    TO.build()
    deps = [_SRC, os.path.join(_HERE, "libkxpu_topo_oracle.so"), os.path.join(_HERE, "libkxpu_xpu_oracle.so"),
            os.path.join(_HERE, "..", "include", "kxpu.h")]
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC,
                           "-L" + _HERE, "-lkxpu_topo_oracle", "-lkxpu_mdev_oracle", "-lkxpu_xpu_oracle", "-lkxpu_oracle",
                           "-Wl,-rpath,$ORIGIN"])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxo_classify_viable.restype = C.c_int32
        L.kxo_classify_viable.argtypes = [vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp, vp]
        _LIB = L
    return _LIB


def classify_viable(rules, recs: np.ndarray, topo=False):
    """kxo_classify_viable: the classify dict plus dev_rule, group_blocker and (topo=True) group_numa.  A failing call
    returns its status instead: -1 for an invalid rule list, -7 for a blocker of group 0xFFFFFFFF."""
    L = lib()
    ra = XO.rules_array(rules)
    n = len(recs)
    recs = np.ascontiguousarray(recs)
    assert recs.dtype.itemsize == 64
    arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                dev_groups=np.empty(n, np.uint32))
    dev_rule = np.empty(max(n, 1), np.uint8)
    gnuma = np.empty(max(n, 1), np.uint64) if topo else None
    gblk = np.empty(max(n, 1), np.uint32)
    out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
    rc = L.kxo_classify_viable(ra.ctypes.data if len(ra) else None, len(ra), recs.ctypes.data, n, C.byref(out),
                               dev_rule.ctypes.data, None if gnuma is None else gnuma.ctypes.data, gblk.ctypes.data)
    if rc != 0:
        return rc
    g, d, a = out.n_groups, out.n_devids, out.n_accepted
    res = dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
               group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
               group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
               dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d],
               group_blocker=gblk[:g])
    if topo:
        res["group_numa"] = gnuma[:g]
    return res
