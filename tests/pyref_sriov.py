"""Independent Python restatement of the SR-IOV calls (include/kxpu.h, additions to ABI v14): kxpu_sriov with regular
expressions and a dict from PCI address to the first record carrying it, and kxpu_pcie_tree_sriov as pyref_pcie's forest
over chains rewritten through each VF's PF.  It shares no code with the kernels."""
import re

import pyref_pcie as PP

NO_PF = 0xFFFFFFFF
VIABLE = 0xFFFFFFFF
PHYSFN_ERR, NUMVFS_ERR = 0x01, 0x02
DRIVER_ERR = 0x02
_CANON = re.compile(rb"[0-9a-f]{4}:[0-9a-f]{2}:[01][0-9a-f]\.[0-7]")
_NUMVFS = re.compile(rb"(0|[1-9][0-9]{0,4})\n?")


def _text(field):
    return bytes(field).split(b"\0", 1)[0]


def numvfs(txt, length, flags=0):
    """sriov_numvfs: a canonical decimal 0..65535 with at most one trailing '\\n'; anything else 0."""
    if flags & NUMVFS_ERR or length > 8:
        return 0
    m = _NUMVFS.fullmatch(bytes(txt)[:length])
    return int(m.group(1)) if m and int(m.group(1)) <= 65535 else 0


def canonical(addr: bytes) -> bool:
    return _CANON.fullmatch(addr) is not None


def sriov(rules, recs, srs, group_off, group_members):
    """dict(pf_of, numvfs, group_sriov) as lists; rules: [(vendor, driver)] bytes; the CSR of a classify call."""
    first = {}
    for i, r in enumerate(recs):
        b = _text(r["bdf"])
        if canonical(b):
            first.setdefault(b, i)
    pf_of, nv = [], []
    for i, s in enumerate(srs):
        pf = _text(s["physfn"])
        p = first.get(pf, NO_PF) if canonical(pf) and not int(s["flags"]) & PHYSFN_ERR else NO_PF
        pf_of.append(NO_PF if p == i else p)
        nv.append(numvfs(s["numvfs_txt"], int(s["numvfs_len"]), int(s["flags"])))
    drivers = {d for _, d in rules}

    def blocks(i):
        p = pf_of[i]
        if p != NO_PF and _text(recs[p]["driver"]) in drivers and not int(recs[p]["flags"]) & DRIVER_ERR:
            return True
        return nv[i] > 0

    gs = []
    for g in range(len(group_off) - 1):
        members = [int(m) for m in group_members[group_off[g]:group_off[g + 1]]]
        hits = [i for i in members if blocks(i)]
        gs.append(min(hits) if hits else VIABLE)
    return dict(pf_of=pf_of, numvfs=nv, group_sriov=gs)


def tree(recs, paths, group_off, group_members, pf_of):
    """kxpu_pcie_tree_sriov: dict(group_node, key, parent, depth) as lists, or None for an invalid CSR or pf_of.  A member
    whose PF has a known chain shorter than KXPU_PCIE_MAX_DEPTH takes the PF's chain and the PF's own key."""
    n = len(recs)
    if any(int(p) != NO_PF and int(p) >= n for p in pf_of):
        return None
    G = len(group_off) - 1
    for g in range(G):
        if group_off[g + 1] < group_off[g] or any(int(m) >= n for m in group_members[group_off[g]:group_off[g + 1]]):
            return None

    def chain(i):
        p = int(pf_of[i])
        if p != NO_PF:
            pc = PP.record_chain(recs[p], paths[p])
            if 0 < len(pc) < PP.MAX_DEPTH:
                return pc + [PP.component_key(_text(recs[p]["bdf"]).decode())[0]]
        return PP.record_chain(recs[i], paths[i])

    nodes, key, parent, depth, gnode = {}, [], [], [], []
    for g in range(G):
        chains = [c for c in (chain(int(m)) for m in group_members[group_off[g]:group_off[g + 1]]) if c]
        common = []
        if chains:
            common = chains[0]
            for c in chains[1:]:
                k = 0
                while k < min(len(common), len(c)) and common[k] == c[k]:
                    k += 1
                common = common[:k]
        for t in range(len(common)):
            pre = tuple(common[:t + 1])
            if pre not in nodes:
                nodes[pre] = len(key)
                key.append(common[t])
                parent.append(nodes[pre[:-1]] if t else PP.NO_NODE)
                depth.append(t)
        gnode.append(nodes[tuple(common)] if common else PP.NO_NODE)
    return dict(group_node=gnode, key=key, parent=parent, depth=depth)
