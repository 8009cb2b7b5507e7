"""ctypes binding of the any-vendor CPU oracle (oracle/kxpu_xpu_oracle.c): the checker of kxpu_classify_rules,
kxpu_cdi_emit_kind and kxpu_alloc_names_kind.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C

import numpy as np

from . import oracle as O
from .oracle import CDIDEV_DTYPE, DEVREC_DTYPE, ClassifyOut  # noqa: F401  (re-exported for the tests)

RULE_DTYPE = np.dtype([("vendor", "S8"), ("driver", "S16"), ("reserved", "<u4", (2,))])
assert RULE_DTYPE.itemsize == 32


def rules_array(rules):
    """[(vendor bytes, driver bytes)] -> kxpu_xpu_rule[] (a structured array passes through)."""
    if isinstance(rules, np.ndarray):
        return np.ascontiguousarray(rules)
    a = np.zeros(len(rules), RULE_DTYPE)
    for i, (v, d) in enumerate(rules):
        a[i]["vendor"], a[i]["driver"] = v, d
    return a


def classify_rules(rules, recs: np.ndarray):
    """kxo_classify_rules: classify's dict plus dev_rule; None when the rule list is invalid."""
    ra = rules_array(rules)
    return O.classify_call(O.lib().kxo_classify_rules, (ra.ctypes.data if len(ra) else None, len(ra)), recs,
                           dev=[("dev_rule", np.uint8)])[1]


def kind_ok(kind: bytes) -> bool:
    return bool(O.lib().kxo_kind_ok(kind))


def cdi_emit_kind(fmt: int, kind: bytes, devs: np.ndarray):
    """kxo_cdi_emit_kind: the document, or None when the kind is outside the supported domain."""
    L = O.lib()
    devs = np.ascontiguousarray(devs)
    need = L.kxo_cdi_emit_kind(fmt, kind, devs.ctypes.data, len(devs), None, 0)
    if need == C.c_size_t(-1).value:
        return None
    out = np.empty(max(need, 1), np.uint8)
    got = L.kxo_cdi_emit_kind(fmt, kind, devs.ctypes.data, len(devs), out.ctypes.data, need)
    assert got == need
    return out[:need].tobytes()


def alloc_names_kind(kind: bytes, idx: np.ndarray):
    """kxo_alloc_names_kind: (blob, offsets), or None when the kind is outside the supported domain."""
    L = O.lib()
    idx = np.ascontiguousarray(idx, dtype=np.uint64)
    offs = np.empty(len(idx) + 1, np.uint32)
    cap = (len(kind) + 22) * len(idx) + 1
    out = np.empty(cap, np.uint8)
    need = L.kxo_alloc_names_kind(kind, idx.ctypes.data, len(idx), out.ctypes.data, cap, offs.ctypes.data)
    if need == C.c_size_t(-1).value:
        return None
    return out[:need].tobytes(), offs
