"""ctypes binding of the vGPU DRA ResourceSlice CPU oracle (oracle/kxpu_dra_mdev_oracle.c): the checker of
kxpu_dra_slices_mdev.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import numpy as np

from . import oracle as O
from .dra_oracle import slices_call
from .oracle import _HERE  # noqa: F401  (the layout tests find include/kxpu.h from it)

# kxpu_dramdev, as include/kxpu.h declares it (tests compare it with the product binding's dtype)
DRAMDEV_DTYPE = np.dtype([("product", "u1", (64,)), ("mdev_type", "S40"), ("uuid", "S36"), ("iommu_group", "<u4"),
                          ("parent", "S16"), ("pcie_root", "S16"), ("vendor", "S8"), ("device", "S8"), ("numa_mask", "<u8"),
                          ("product_len", "u1"), ("reserved", "u1", (7,))])
assert DRAMDEV_DTYPE.itemsize == 208
WHY = ["product", "mdev_type", "uuid", "parent", "pcie_root", "vendor", "device", "iommu_group", "product_len"]


def dra_slices_mdev(driver, pool, node, generation, devs):
    """(bytes, slice_off) of kxo_dra_slices_mdev, or the failing status: -1 for a bad argument; for a record outside
    the domain (-7, name of the first failing rule)."""
    return slices_call(O.lib().kxo_dra_slices_mdev, DRAMDEV_DTYPE, WHY, driver, pool, node, generation, devs)
