"""ctypes binding of the DRA ResourceSlice CPU oracle (oracle/kxpu_dra_oracle.c): the checker of kxpu_dra_slices.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C

import numpy as np

from . import oracle as O
from .oracle import _HERE  # noqa: F401  (the layout tests find include/kxpu.h from it)

# kxpu_dradev, as include/kxpu.h declares it (tests compare it with the product binding's dtype)
DRADEV_DTYPE = np.dtype([("product", "u1", (64,)), ("bdf", "S16"), ("pcie_root", "S16"), ("vendor", "S8"), ("device", "S8"),
                         ("numa_mask", "<u8"), ("iommu_group", "<u4"), ("product_len", "u1"), ("reserved", "u1", (3,))])
assert DRADEV_DTYPE.itemsize == 128
WHY = ["product", "bdf", "pcie_root", "vendor", "device", "iommu_group", "product_len"]


def _b(s):
    return s.encode() if isinstance(s, str) else s


def slices_call(fn, dtype, why_names, driver, pool, node, generation, devs, *rest):
    """The two-call sizing of every kxo_dra_slices* call: fn(driver, pool, node, generation, devs, n, *rest, out, cap,
    &need, slice_off, &n_slices, &why), once to size the outputs and once to fill them.  Returns (bytes, slice_off), or
    the failing status: -1 for a bad argument; for a record outside the domain (-7, why_names[*why])."""
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == dtype
    dp = devs.ctypes.data if len(devs) else None
    need, ns, why = C.c_size_t(0), C.c_size_t(0), C.c_int32(-1)
    args = (_b(driver), _b(pool), _b(node), generation, dp, len(devs)) + rest
    rc = fn(*args, None, 0, C.byref(need), None, C.byref(ns), C.byref(why))
    if rc == -7:
        return rc, why_names[why.value] if why.value >= 0 else None
    if rc != -4:
        return rc
    out = np.empty(max(need.value, 1), np.uint8)
    offs = np.empty(ns.value + 1, np.uint64)
    rc = fn(*args, out.ctypes.data, need.value, C.byref(need), offs.ctypes.data, C.byref(ns), C.byref(why))
    assert rc == 0, rc
    return out[:need.value].tobytes(), offs


def dra_slices(driver, pool, node, generation, devs):
    """(bytes, slice_off) of kxo_dra_slices, or the failing status: -1 for a bad argument; for a record outside the
    domain (-7, name of the first failing rule)."""
    return slices_call(O.lib().kxo_dra_slices, DRADEV_DTYPE, WHY, driver, pool, node, generation, devs)
