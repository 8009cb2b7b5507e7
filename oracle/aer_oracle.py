"""ctypes binding of the AER CPU oracle (oracle/kxpu_aer_oracle.c): the checker of kxpu_aer_health,
kxpu_dra_slices_taints and kxpu_dra_slices_mdev_taints.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C

import numpy as np

from oracle import dra_taint_oracle
from oracle import oracle as O
from oracle.dra_oracle import _b, slices_call

DRADEV_DTYPE = dra_taint_oracle.DRADEV_DTYPE
DRAMDEV_DTYPE = dra_taint_oracle.DRAMDEV_DTYPE
WHY = dra_taint_oracle.WHY + ["taint_duplicate"]
WHY_MDEV = dra_taint_oracle.WHY_MDEV + ["taint_duplicate"]
UNKNOWN = (1 << 64) - 1


class Taint(C.Structure):
    _fields_ = [("key", C.c_char_p), ("value", C.c_char_p), ("effect", C.c_char_p)]


def aer_health(text, file_off, file_len, fatal_limit, nonfatal_limit, group_off, group_members):
    """(totals, group_aer) of kxo_aer_health, or the failing status.  Arguments as Kxpu.aer_health."""
    t = np.frombuffer(bytes(text), np.uint8)
    file_off = np.ascontiguousarray(file_off, dtype=np.uint64)
    file_len = np.ascontiguousarray(file_len, dtype=np.uint32)
    group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
    group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
    n, G = len(file_off) // 2, len(group_off) - 1
    totals = np.empty(max(2 * n, 1), np.uint64)
    group_aer = np.empty(max(G, 1), np.uint8)
    rc = O.lib().kxo_aer_health(t.ctypes.data if len(t) else None, len(t), file_off.ctypes.data if n else None,
                                file_len.ctypes.data if n else None, n, fatal_limit, nonfatal_limit,
                                group_off.ctypes.data, group_members.ctypes.data if len(group_members) else None, G,
                                totals.ctypes.data, group_aer.ctypes.data)
    if rc:
        return rc
    return totals[:2 * n], group_aer[:G]


def _slices(fn, dtype, why_names, driver, pool, node, generation, devs, taints, since):
    tab = (Taint * max(len(taints), 1))(*[Taint(_b(k), _b(v), _b(e)) for k, v, e in taints])
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
        assert since.size == len(devs) * len(taints)
    sp = None if since is None else since.ctypes.data
    return slices_call(fn, dtype, why_names, driver, pool, node, generation, devs, C.cast(tab, C.c_void_p), len(taints),
                       sp)


def dra_slices_taints(driver, pool, node, generation, devs, taints, since):
    """(bytes, slice_off) of kxo_dra_slices_taints, or the failing status: -1 for a bad argument; for a record or a
    taint outside the domain (-7, name of the first failing rule).  taints: [(key, value, effect)]; since: None or an
    int64 [n, len(taints)] array."""
    return _slices(O.lib().kxo_dra_slices_taints, DRADEV_DTYPE, WHY, driver, pool, node, generation, devs, taints,
                   since)


def dra_slices_mdev_taints(driver, pool, node, generation, devs, taints, since):
    """the same for a pool of vGPUs (kxo_dra_slices_mdev_taints)"""
    return _slices(O.lib().kxo_dra_slices_mdev_taints, DRAMDEV_DTYPE, WHY_MDEV, driver, pool, node, generation, devs,
                   taints, since)
