"""Independent Python restatement of the vGPU-on-VF calls (include/kxpu.h, additions to ABI v14): kxpu_vf_vgpu_types with
regular expressions over the split lines and a dict from type ID to its first name, and kxpu_classify_vf_vgpu as one
sequential walk over the records with dicts for groups and device-map entries.  It shares no code with the kernels."""
import re

import numpy as np

import pyref_mdev as PM

VT_READ, VT_CUR_ERR = 0x01, 0x02
NONE, NAMED, UNNAMED, BAD = 0, 1, 2, 3
VIABLE = 0xFFFFFFFF
REJECTED = 0xFFFFFFFF
VENDOR_ERR, DRIVER_ERR, IOMMU_ERR, DEVICE_ERR, IS_DIR, NUMA, BLOCKS = 0x01, 0x02, 0x04, 0x08, 0x10, 0x40, 0x80
_LINE = re.compile(rb"[ \t]*([1-9][0-9]*)[ \t]*:[ \t]*(.*?)[ \t]*")
_CUR = re.compile(rb"(0|[1-9][0-9]*)\n?")


def names(tables):
    """{type ID: key} from the tables in priority order: the first line, in table order then line order, naming it."""
    out = {}
    for t in tables:
        for line in t.split(b"\n"):
            if line.endswith(b"\r"):
                line = line[:-1]
            m = _LINE.fullmatch(line)
            if not m or int(m.group(1)) > 0xFFFFFFFF or not 1 <= len(m.group(2)) <= 40:
                continue
            key = PM.type_key(m.group(2))
            if key:
                out.setdefault(int(m.group(1)), key)
    return out


def current(rec):
    """(status, type ID) of the current_vgpu_type of one kxpu_vfvgpurec, before the name lookup."""
    fl, n = int(rec["flags"]), int(rec["cur_len"])
    if not fl & VT_READ:
        return NONE, 0
    if fl & VT_CUR_ERR or n > 16:
        return BAD, 0
    m = _CUR.fullmatch(bytes(rec["cur_txt"])[:n])
    if not m or int(m.group(1)) >= 1 << 32:
        return BAD, 0
    v = int(m.group(1))
    return (NONE, 0) if v == 0 else (UNNAMED, v)


def vf_vgpu_types(recs_vt, tables):
    """dict(keys (list of 48-byte rows), type_id, status) as kxpu_vf_vgpu_types returns them."""
    known = names(tables)
    keys, tid, st = [], [], []
    for r in recs_vt:
        s, v = current(r)
        row = bytes(48)
        if s == UNNAMED and v in known:
            k = known[v]
            s, row = NAMED, k + bytes(47 - len(k)) + bytes([len(k)])
        keys.append(row)
        tid.append(v)
        st.append(s)
    return dict(keys=keys, type_id=tid, status=st)


def _text(f):
    return bytes(f).split(b"\0", 1)[0]


def _id(txt, n):
    if n < 2 or n > 8:
        return None
    return bytes(txt)[2:n].strip(b"\n")


def classify_vf_vgpu(rules, vgpu_rules, recs, keys, topo=False, viable=False):
    """The outputs of kxpu_classify_vf_vgpu (lists) for DEVREC records and 48-byte key rows (bytes each)."""
    n = len(recs)
    rule_of, cand, good = [None] * n, [False] * n, [False] * n
    key_of = [None] * n
    for i, r in enumerate(recs):
        fl = int(r["flags"])
        if fl & (IS_DIR | VENDOR_ERR | DRIVER_ERR | IOMMU_ERR):
            continue
        v = _id(r["vendor_txt"], int(r["vendor_len"]))
        m = [k for k, (rv, rd) in enumerate(rules) if v == rv and _text(r["driver"]) == rd]
        if v is None or not m:
            continue
        rule_of[i] = m[0]
        if vgpu_rules >> m[0] & 1:
            k = bytes(keys[i])
            if k[47] == 0:
                continue
            key_of[i], cand[i], good[i] = k, True, True
        else:
            cand[i] = True
            good[i] = not fl & DEVICE_ERR and _id(r["device_txt"], int(r["device_len"])) is not None
    first_key = {}  # key row -> lowest candidate index carrying it
    for i in range(n):
        if key_of[i] is not None:
            first_key.setdefault(key_of[i], i)
    groups, order, accept = {}, [], [REJECTED] * n
    for i, r in enumerate(recs):
        g = int(r["iommu_group"])
        if not cand[i] or (g not in groups and not good[i]):
            continue
        if g not in groups:
            groups[g] = []
            order.append((g, i))
        accept[i] = sum(len(v) for v in groups.values())
        groups[g].append(i)
    devmap, devorder = {}, []
    for g, i in order:
        r = recs[i]
        if key_of[i] is not None:
            dk = (rule_of[i], "key", first_key[key_of[i]])
            did = first_key[key_of[i]]
        else:
            d = _id(r["device_txt"], int(r["device_len"]))
            dk = (rule_of[i], "id", d)
            did = int.from_bytes(d, "little")
        if dk not in devmap:
            devmap[dk] = []
            devorder.append((dk, did))
        devmap[dk].append(g)
    res = dict(accept_index=accept, n_accepted=sum(len(v) for v in groups.values()), n_groups=len(order),
               n_devids=len(devorder), group_ids=[g for g, _ in order],
               group_off=list(np.cumsum([0] + [len(groups[g]) for g, _ in order])),
               group_members=[m for g, _ in order for m in groups[g]], dev_ids=[did for _, did in devorder],
               dev_off=list(np.cumsum([0] + [len(devmap[k]) for k, _ in devorder])),
               dev_groups=[g for k, _ in devorder for g in devmap[k]], dev_rule=[k[0] for k, _ in devorder])
    if topo:
        res["group_numa"] = [0] * len(order)
        for o, (g, _) in enumerate(order):
            for m in groups[g]:
                fl, node = int(recs[m]["flags"]), int(recs[m]["reserved0"])
                if fl & NUMA and node < 64:
                    res["group_numa"][o] |= 1 << node
    if viable:
        res["group_blocker"] = []
        for g, _ in order:
            b = [i for i, r in enumerate(recs) if not cand[i] and int(r["iommu_group"]) == g
                 and int(r["flags"]) & (BLOCKS | IS_DIR) == BLOCKS]
            res["group_blocker"].append(min(b) if b else VIABLE)
    res["group_off"] = [int(x) for x in res["group_off"]]
    res["dev_off"] = [int(x) for x in res["dev_off"]]
    return res
