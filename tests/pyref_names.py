"""A Python restatement of kxpu_classify_named (include/kxpu.h): kxpu_classify_vf_vgpu's walk with deviceMap entries
keyed by configured resource-name slots.  Independent of tests/names_oracle.py, which states the same on the C oracles.

TEST INFRASTRUCTURE ONLY."""
import numpy as np

from pyref_vf_vgpu import (BLOCKS, DEVICE_ERR, DRIVER_ERR, IOMMU_ERR, IS_DIR, NUMA, REJECTED, VENDOR_ERR, VIABLE, _id,
                           _text)

NO_SLOT = 0xFFFFFFFF


def valid(names, n_rules, vgpu_rules=0):
    """names: [(rule, device bytes, slot)].  False where the call returns KXPU_E_INVALID."""
    if len(names) > 64:
        return False
    seen = set()
    for rule, dev, slot in names:
        if rule >= n_rules or vgpu_rules >> rule & 1 or slot >= len(names) or (rule, dev) in seen:
            return False
        if dev != b"*" and not (len(dev) == 4 and all(c in b"0123456789abcdef" for c in dev)):
            return False
        seen.add((rule, dev))
    return True


def slot_of(names, rule, did):
    exact = [s for r, d, s in names if r == rule and d == did and d != b"*"]
    star = [s for r, d, s in names if r == rule and d == b"*"]
    return exact[0] if exact else star[0] if star else None


def classify_named(rules, vgpu_rules, recs, keys, names, topo=False, viable=False):
    """The outputs (lists) for DEVREC records, 48-byte key rows (bytes each, or None) and [(rule, device, slot)]."""
    if not valid(names, len(rules), vgpu_rules):
        return None
    n = len(recs)
    rule_of, cand, good, key_of = [None] * n, [False] * n, [False] * n, [None] * n
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
            key_of[i], cand[i], good[i] = ("key", k), True, True
        else:
            cand[i] = True
            did = None if fl & DEVICE_ERR else _id(r["device_txt"], int(r["device_len"]))
            good[i] = did is not None
            s = slot_of(names, m[0], did) if good[i] else None
            if s is not None:
                key_of[i] = ("slot", m[0], s)
    first_key = {}  # type key or (rule, slot) -> lowest candidate carrying it
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
        if key_of[i] is not None:
            dk, did = (rule_of[i],) + key_of[i], first_key[key_of[i]]
            slot = key_of[i][2] if key_of[i][0] == "slot" else NO_SLOT
        else:
            d = _id(recs[i]["device_txt"], int(recs[i]["device_len"]))
            dk, did, slot = (rule_of[i], "id", d), int.from_bytes(d, "little"), NO_SLOT
        if dk not in devmap:
            devmap[dk] = []
            devorder.append((dk, did, slot))
        devmap[dk].append(g)
    res = dict(accept_index=accept, n_accepted=sum(len(v) for v in groups.values()), n_groups=len(order),
               n_devids=len(devorder), group_ids=[g for g, _ in order],
               group_off=[int(x) for x in np.cumsum([0] + [len(groups[g]) for g, _ in order])],
               group_members=[m for g, _ in order for m in groups[g]], dev_ids=[did for _, did, _ in devorder],
               dev_off=[int(x) for x in np.cumsum([0] + [len(devmap[k]) for k, _, _ in devorder])],
               dev_groups=[g for k, _, _ in devorder for g in devmap[k]], dev_rule=[k[0] for k, _, _ in devorder])
    if names:
        res["dev_slot"] = [s for _, _, s in devorder]
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
    return res
