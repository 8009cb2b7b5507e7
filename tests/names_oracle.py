"""The C statement of kxpu_classify_named, next to tests/pyref_names.py: tests/names_oracle.c (the name table's checks
and slot lookup, compiled once per process into a temporary directory, so the tree stays read-only) over the C classify
oracles.  A slotted candidate is rewritten to carry a five-byte device id that stands for its (rule, slot) -- no real
id has five bytes -- and tests/vf_vgpu_oracle.py classifies the result; those entries' ids are then mapped back to the
lowest candidate with the (rule, slot), and dev_slot is the slot they stand for.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import vf_vgpu_oracle as VV
from conftest import ROOT
from kxpu_b200.binding import NAME_DTYPE, NO_SLOT

_LIB = None
CAND_ERR, DEVICE_ERR = 0x17, 0x08


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="kxn_"), "libkxn_names.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "names_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxn_check.restype, L.kxn_check.argtypes = C.c_int, [vp, sz, sz, C.c_uint32]
        L.kxn_slot.restype, L.kxn_slot.argtypes = C.c_uint32, [vp, sz, C.c_uint32, C.c_char_p, sz]
        _LIB = L
    return _LIB


def table(names):
    """a NAME_DTYPE array from [(rule, device bytes, slot)] (an array passes through)"""
    if isinstance(names, np.ndarray):
        return np.ascontiguousarray(names)
    return np.array([(r, s, d) for r, d, s in names], NAME_DTYPE)


def check(names, n_rules, vgpu_rules=0):
    t = table(names)
    return lib().kxn_check(t.ctypes.data if len(t) else None, len(t), n_rules, vgpu_rules) == 0


def classify_named(rules, vgpu_rules, recs, keys, names, topo=False, viable=False):
    """The outputs of kxpu_classify_named as lists, or None where the call returns KXPU_E_INVALID."""
    t = table(names)
    if not check(t, len(rules), vgpu_rules):
        return None
    recs = np.array(recs, copy=True)
    if keys is None:
        keys = np.zeros(len(recs), VV.VGPUKEY_DTYPE)
    first = {}  # synthetic id -> (lowest candidate with that (rule, slot), slot)
    for i, r in enumerate(recs):
        rule = VV._rule_of(rules, r)
        fl = int(r["flags"])
        if rule is None or vgpu_rules >> rule & 1 or fl & CAND_ERR or fl & DEVICE_ERR or not 2 <= int(r["device_len"]) <= 8:
            continue
        did = bytes(r["device_txt"])[2:int(r["device_len"])].strip(b"\n")
        s = lib().kxn_slot(t.ctypes.data if len(t) else None, len(t), rule, did, len(did))
        if s == NO_SLOT:
            continue
        sid = b"%01x%02x%02x" % (8 + rule % 8, rule, s)  # five bytes, never a real id
        first.setdefault(int.from_bytes(sid, "little"), (i, s))
        recs[i]["device_txt"] = np.frombuffer((b"0x" + sid + b"\n").ljust(8, b"\0"), np.uint8)
        recs[i]["device_len"] = 8
    out = VV.classify_vf_vgpu(rules, vgpu_rules, recs, keys, topo=topo, viable=viable)
    slots = []
    for j, d in enumerate(out["dev_ids"]):
        if not vgpu_rules >> out["dev_rule"][j] & 1 and d in first:
            out["dev_ids"][j], s = first[d]
            slots.append(s)
        else:
            slots.append(NO_SLOT)
    if len(t):
        out["dev_slot"] = slots
    return out
