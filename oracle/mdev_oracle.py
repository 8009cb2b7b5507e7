"""ctypes binding of the vGPU CPU oracle (oracle/kxpu_mdev_oracle.c): the checker of kxpu_classify_mdev,
kxpu_mdev_names and kxpu_cdi_emit_mdev.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.  The library links
against libkxpu_oracle.so (yaml.v3 base-60 predicate) and libkxpu_xpu_oracle.so (kind domain), so
xpu_oracle.build() runs first.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import xpu_oracle as XO
from .oracle import ClassifyOut

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_mdev_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_mdev_oracle.so")
_LIB = None

MDEVREC_DTYPE = np.dtype([("uuid", "S36"), ("parent", "S16"), ("parent_vendor_txt", "u1", (8,)), ("driver", "S16"),
                          ("type_name", "u1", (40,)), ("iommu_group", "<u4"), ("vendor_len", "u1"), ("name_len", "u1"),
                          ("flags", "u1"), ("reserved0", "u1"), ("reserved1", "<u4")])
MDEVCDI_DTYPE = np.dtype([("uuid", "S36"), ("iommu_group", "<u4"), ("parent", "S16"), ("index", "<u8")])
assert MDEVREC_DTYPE.itemsize == 128 and MDEVCDI_DTYPE.itemsize == 64


def build():
    XO.build()
    deps = [_SRC, os.path.join(_HERE, "libkxpu_oracle.so"), os.path.join(_HERE, "libkxpu_xpu_oracle.so"),
            os.path.join(_HERE, "..", "include", "kxpu.h")]
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC,
                           "-L" + _HERE, "-lkxpu_xpu_oracle", "-lkxpu_oracle", "-Wl,-rpath,$ORIGIN"])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        L.kxo_mdev_classify.restype = C.c_int32
        L.kxo_mdev_classify.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(ClassifyOut), C.c_void_p]
        L.kxo_type_key.restype = C.c_size_t
        L.kxo_type_key.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p]
        L.kxo_uuid_ok.restype = C.c_int
        L.kxo_uuid_ok.argtypes = [C.c_char_p]
        L.kxo_mdev_names.restype = C.c_size_t
        L.kxo_mdev_names.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.kxo_cdi_emit_mdev.restype = C.c_size_t
        L.kxo_cdi_emit_mdev.argtypes = [C.c_int32, C.c_char_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        _LIB = L
    return _LIB


def classify_mdev(rules, recs: np.ndarray):
    """kxo_mdev_classify: the classify dict plus dev_rule; None when the rule list is invalid."""
    L = lib()
    ra = XO.rules_array(rules)
    n = len(recs)
    recs = np.ascontiguousarray(recs)
    assert recs.dtype == MDEVREC_DTYPE
    arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                dev_groups=np.empty(n, np.uint32))
    dev_rule = np.empty(max(n, 1), np.uint8)
    out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
    rc = L.kxo_mdev_classify(ra.ctypes.data if len(ra) else None, len(ra), recs.ctypes.data, n, C.byref(out),
                             dev_rule.ctypes.data)
    if rc != 0:
        return None
    g, d, a = out.n_groups, out.n_devids, out.n_accepted
    return dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d])


def type_key(name: bytes) -> bytes:
    out = C.create_string_buffer(max(len(name), 1))
    n = lib().kxo_type_key(name, len(name), out)
    return out.raw[:n]


def uuid_ok(u: bytes) -> bool:
    return len(u) == 36 and bool(lib().kxo_uuid_ok(u))


def mdev_names(recs: np.ndarray, idx):
    """kxo_mdev_names: (blob, offsets) of the type keys of recs[idx]."""
    recs = np.ascontiguousarray(recs)
    idx = np.ascontiguousarray(idx, dtype=np.uint32)
    offs = np.empty(len(idx) + 1, np.uint32)
    out = np.empty(40 * len(idx) + 1, np.uint8)
    need = lib().kxo_mdev_names(recs.ctypes.data, idx.ctypes.data, len(idx), out.ctypes.data, offs.ctypes.data)
    return out[:need].tobytes(), offs


def cdi_emit_mdev(fmt: int, kind: bytes, devs: np.ndarray):
    """kxo_cdi_emit_mdev: the document, or None when the kind, a uuid or a parent is outside the domain."""
    L = lib()
    devs = np.ascontiguousarray(devs)
    assert devs.dtype == MDEVCDI_DTYPE
    need = L.kxo_cdi_emit_mdev(fmt, kind, devs.ctypes.data, len(devs), None, 0)
    if need == C.c_size_t(-1).value:
        return None
    out = np.empty(max(need, 1), np.uint8)
    got = L.kxo_cdi_emit_mdev(fmt, kind, devs.ctypes.data, len(devs), out.ctypes.data, need)
    assert got == need
    return out[:need].tobytes()
