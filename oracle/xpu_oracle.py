"""ctypes binding of the any-vendor CPU oracle (oracle/kxpu_xpu_oracle.c): the checker of kxpu_classify_rules,
kxpu_cdi_emit_kind and kxpu_alloc_names_kind.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.  The library links
against libkxpu_oracle.so for the yaml.v3 base-60 predicate, so oracle.build() runs first.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import oracle as O
from .oracle import CDIDEV_DTYPE, DEVREC_DTYPE, ClassifyOut  # noqa: F401  (re-exported for the tests)

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_xpu_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_xpu_oracle.so")
_LIB = None


def build():
    O.build()
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(_SRC), os.path.getmtime(os.path.join(_HERE, "libkxpu_oracle.so"))):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC,
                           "-L" + _HERE, "-lkxpu_oracle", "-Wl,-rpath,$ORIGIN"])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        L.kxo_classify_rules.restype = C.c_int32
        L.kxo_classify_rules.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(ClassifyOut), C.c_void_p]
        L.kxo_kind_ok.restype = C.c_int
        L.kxo_kind_ok.argtypes = [C.c_char_p]
        L.kxo_cdi_emit_kind.restype = C.c_size_t
        L.kxo_cdi_emit_kind.argtypes = [C.c_int32, C.c_char_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        L.kxo_alloc_names_kind.restype = C.c_size_t
        L.kxo_alloc_names_kind.argtypes = [C.c_char_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        _LIB = L
    return _LIB


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
    L = lib()
    ra = rules_array(rules)
    n = len(recs)
    recs = np.ascontiguousarray(recs)
    arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                dev_groups=np.empty(n, np.uint32))
    dev_rule = np.empty(max(n, 1), np.uint8)
    out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
    rc = L.kxo_classify_rules(ra.ctypes.data if len(ra) else None, len(ra), recs.ctypes.data, n, C.byref(out),
                              dev_rule.ctypes.data)
    if rc != 0:
        return None
    g, d, a = out.n_groups, out.n_devids, out.n_accepted
    return dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d])


def kind_ok(kind: bytes) -> bool:
    L = lib()
    return bool(L.kxo_kind_ok(kind))


def cdi_emit_kind(fmt: int, kind: bytes, devs: np.ndarray):
    """kxo_cdi_emit_kind: the document, or None when the kind is outside the supported domain."""
    L = lib()
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
    L = lib()
    idx = np.ascontiguousarray(idx, dtype=np.uint64)
    offs = np.empty(len(idx) + 1, np.uint32)
    cap = (len(kind) + 22) * len(idx) + 1
    out = np.empty(cap, np.uint8)
    need = L.kxo_alloc_names_kind(kind, idx.ctypes.data, len(idx), out.ctypes.data, cap, offs.ctypes.data)
    if need == C.c_size_t(-1).value:
        return None
    return out[:need].tobytes(), offs
