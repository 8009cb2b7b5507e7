"""The C statements of the vGPU-on-VF calls, next to tests/pyref_vf_vgpu.py:
  - vf_vgpu_types: a ctypes binding of tests/vf_vgpu_oracle.c, compiled once per process into a temporary directory, so
    the tree stays read-only;
  - classify_vf_vgpu: the C classify oracles (oracle/xpu_oracle.py, topo_oracle.py, viab_oracle.py) run on records
    rewritten so that a vGPU rule's records look like passthrough records: a named record carries a device id that
    stands for its key, any other record of such a rule carries KXPU_REC_DRIVER_ERR (no candidate).  The device ids of
    those entries are then mapped back to the lowest candidate carrying the key.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT
from oracle import topo_oracle as TO
from oracle import viab_oracle as VO
from oracle import xpu_oracle as XO
from kxpu_b200.binding import VGPUKEY_DTYPE, vgpu_tables

_LIB = None
DRIVER_ERR, DEVICE_ERR = 0x02, 0x08


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="kxv_"), "libkxv_vf_vgpu.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "vf_vgpu_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxv_vf_vgpu_types.restype = C.c_int
        L.kxv_vf_vgpu_types.argtypes = [vp, sz, vp, vp, sz, vp, vp, vp]
        _LIB = L
    return _LIB


def vf_vgpu_types(recs_vt, tables):
    """dict(keys (list of 48-byte rows), type_id, status) as lists, or None for a table_off that decreases."""
    recs_vt = np.ascontiguousarray(recs_vt)
    blob, toff = vgpu_tables(tables)
    blob = np.ascontiguousarray(blob).copy()
    n = len(recs_vt)
    keys, tid, st = np.zeros(max(n, 1), VGPUKEY_DTYPE), np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint8)
    if lib().kxv_vf_vgpu_types(recs_vt.ctypes.data if n else None, n, blob.ctypes.data if len(blob) else None,
                               toff.ctypes.data, len(toff) - 1, keys.ctypes.data, tid.ctypes.data, st.ctypes.data) != 0:
        return None
    return dict(keys=[k.tobytes() for k in keys[:n]], type_id=tid[:n].tolist(), status=st[:n].tolist())


def _rule_of(rules, r):
    v = bytes(r["vendor_txt"])[2:int(r["vendor_len"])].strip(b"\n") if 2 <= int(r["vendor_len"]) <= 8 else None
    d = bytes(r["driver"]).split(b"\0", 1)[0]
    m = [k for k, (rv, rd) in enumerate(rules) if v == rv and d == rd]
    return m[0] if m else None


def classify_vf_vgpu(rules, vgpu_rules, recs, keys, topo=False, viable=False):
    """The outputs of kxpu_classify_vf_vgpu as lists, from the C classify oracles on rewritten records."""
    recs = np.array(recs, copy=True)
    keys = np.ascontiguousarray(keys)
    ids, first = {}, {}  # key row -> synthetic device id; synthetic id -> lowest candidate carrying the key
    for i, r in enumerate(recs):
        rule = _rule_of(rules, r)
        if rule is None or not vgpu_rules >> rule & 1 or int(r["flags"]) & 0x17:
            continue
        k = keys[i].tobytes()
        if k[47] == 0:
            recs[i]["flags"] = int(recs[i]["flags"]) | DRIVER_ERR  # no key: not a candidate (a blocker flag keeps its meaning)
            continue
        sid = ids.setdefault(k, b"%04x" % (0xF000 + len(ids)) if len(ids) < 0x1000 else None)
        assert sid is not None
        first.setdefault(int.from_bytes(sid, "little"), i)
        recs[i]["device_txt"] = np.frombuffer((b"0x" + sid + b"\n").ljust(8, b"\0"), np.uint8)
        recs[i]["device_len"] = 7
        recs[i]["flags"] = int(recs[i]["flags"]) & ~DEVICE_ERR & 0xFF
    if viable:
        res = VO.classify_viable(rules, recs, topo=topo)
    elif topo:
        res = TO.classify_topo(rules, recs)
    else:
        res = XO.classify_rules(rules, recs)
    out = {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in res.items()}
    out["dev_ids"] = [first[d] if vgpu_rules >> out["dev_rule"][j] & 1 and d in first else d
                      for j, d in enumerate(out["dev_ids"])]
    return out
