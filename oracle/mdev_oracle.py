"""ctypes binding of the vGPU CPU oracle (oracle/kxpu_mdev_oracle.c): the checker of kxpu_classify_mdev,
kxpu_mdev_names and kxpu_cdi_emit_mdev.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C

import numpy as np

from . import oracle as O
from . import xpu_oracle as XO

MDEVREC_DTYPE = np.dtype([("uuid", "S36"), ("parent", "S16"), ("parent_vendor_txt", "u1", (8,)), ("driver", "S16"),
                          ("type_name", "u1", (40,)), ("iommu_group", "<u4"), ("vendor_len", "u1"), ("name_len", "u1"),
                          ("flags", "u1"), ("reserved0", "u1"), ("reserved1", "<u4")])
MDEVCDI_DTYPE = np.dtype([("uuid", "S36"), ("iommu_group", "<u4"), ("parent", "S16"), ("index", "<u8")])
assert MDEVREC_DTYPE.itemsize == 128 and MDEVCDI_DTYPE.itemsize == 64


def classify_mdev(rules, recs: np.ndarray):
    """kxo_mdev_classify: the classify dict plus dev_rule; None when the rule list is invalid."""
    ra = XO.rules_array(rules)
    assert recs.dtype == MDEVREC_DTYPE
    return O.classify_call(O.lib().kxo_mdev_classify, (ra.ctypes.data if len(ra) else None, len(ra)), recs,
                           dev=[("dev_rule", np.uint8)])[1]


def type_key(name: bytes) -> bytes:
    out = C.create_string_buffer(max(len(name), 1))
    n = O.lib().kxo_type_key(name, len(name), out)
    return out.raw[:n]


def uuid_ok(u: bytes) -> bool:
    return len(u) == 36 and bool(O.lib().kxo_uuid_ok(u))


def mdev_names(recs: np.ndarray, idx):
    """kxo_mdev_names: (blob, offsets) of the type keys of recs[idx]."""
    recs = np.ascontiguousarray(recs)
    idx = np.ascontiguousarray(idx, dtype=np.uint32)
    offs = np.empty(len(idx) + 1, np.uint32)
    out = np.empty(40 * len(idx) + 1, np.uint8)
    need = O.lib().kxo_mdev_names(recs.ctypes.data, idx.ctypes.data, len(idx), out.ctypes.data, offs.ctypes.data)
    return out[:need].tobytes(), offs


def cdi_emit_mdev(fmt: int, kind: bytes, devs: np.ndarray):
    """kxo_cdi_emit_mdev: the document, or None when the kind, a uuid or a parent is outside the domain."""
    L = O.lib()
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == MDEVCDI_DTYPE
    need = L.kxo_cdi_emit_mdev(fmt, kind, devs.ctypes.data, len(devs), None, 0)
    if need == C.c_size_t(-1).value:
        return None
    out = np.empty(max(need, 1), np.uint8)
    got = L.kxo_cdi_emit_mdev(fmt, kind, devs.ctypes.data, len(devs), out.ctypes.data, need)
    assert got == need
    return out[:need].tobytes()
