"""ctypes binding of the DRA taint CPU oracle (oracle/kxpu_dra_taint_oracle.c): the checker of kxpu_dra_slices_taint
and kxpu_dra_slices_mdev_taint.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import numpy as np

from oracle import dra_mdev_oracle, dra_oracle
from oracle import oracle as O
from oracle.dra_oracle import _b, slices_call

DRADEV_DTYPE = dra_oracle.DRADEV_DTYPE
DRAMDEV_DTYPE = dra_mdev_oracle.DRAMDEV_DTYPE
WHY = dra_oracle.WHY + ["taint_since"]
WHY_MDEV = dra_mdev_oracle.WHY + ["taint_since"]


def _slices(fn, dtype, why_names, driver, pool, node, generation, devs, key, value, effect, since):
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
        assert since.shape == (len(devs),)
    sp = None if since is None else since.ctypes.data
    return slices_call(fn, dtype, why_names, driver, pool, node, generation, devs, _b(key), _b(value), _b(effect), sp)


def dra_slices_taint(driver, pool, node, generation, devs, key, value, effect, since):
    """(bytes, slice_off) of kxo_dra_slices_taint, or the failing status: -1 for a bad argument; for a record or a
    taint time outside the domain (-7, name of the first failing rule).  since: None or one int64 per device."""
    return _slices(O.lib().kxo_dra_slices_taint, DRADEV_DTYPE, WHY, driver, pool, node, generation, devs, key, value,
                   effect, since)


def dra_slices_mdev_taint(driver, pool, node, generation, devs, key, value, effect, since):
    """the same for a pool of vGPUs (kxo_dra_slices_mdev_taint)"""
    return _slices(O.lib().kxo_dra_slices_mdev_taint, DRAMDEV_DTYPE, WHY_MDEV, driver, pool, node, generation, devs,
                   key, value, effect, since)
