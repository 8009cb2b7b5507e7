"""Independent Python restatement of the PCIe topology calls (include/kxpu.h, ABI v7), the second checker next to
oracle/kxpu_pcie_oracle.c:
  - chain: the path grammar as regular expressions over the split path;
  - tree: the forest as a dict from whole prefixes (tuples of keys) to ordinals;
  - preferred: the allocation with the devices' chains as key tuples: X by min() over a key tuple, the candidates by
    one sorted().
"""
import re

import pyref_topo as PT

MAX_DEPTH = 8
NO_NODE = 0xFFFFFFFF
_DOM = r"([0-9a-f]{4}|[1-9a-f][0-9a-f]{4,7})"
_BRIDGE = re.compile(r"pci" + _DOM + r":([0-9a-f]{2})")
_FUNC = re.compile(_DOM + r":([0-9a-f]{2}):([01][0-9a-f])\.([0-7])")


def component_key(c):
    m = _BRIDGE.fullmatch(c)
    if m:
        return (1 << 63) | int(m.group(1), 16) << 16 | int(m.group(2), 16) << 8, "bridge"
    m = _FUNC.fullmatch(c)
    if m:
        return int(m.group(1), 16) << 16 | int(m.group(2), 16) << 8 | int(m.group(3), 16) << 3 | int(m.group(4)), "func"
    return None, None


def chain(bdf: bytes, path: bytes, length: int):
    """The chain keys of a record, [] when the path is unknown."""
    if not 1 <= length <= 120:
        return []
    text = path[:length]
    try:
        parts = text.decode("ascii").split("/")
    except UnicodeDecodeError:
        return []
    if not 2 <= len(parts) <= MAX_DEPTH + 1:
        return []
    keys = []
    for i, c in enumerate(parts):
        k, kind = component_key(c)
        if kind is None or (i == 0 and kind != "bridge"):
            return []
        keys.append(k)
    if parts[-1].encode() != bdf.split(b"\0", 1)[0]:
        return []
    return keys[:-1]


def record_chain(rec, path_row):
    return chain(bytes(rec["bdf"]), bytes(path_row["path"]).ljust(120, b"\0"), int(path_row["len"]))


def tree(recs, paths, group_off, group_members):
    """dict(group_node, key, parent, depth) as lists, or None for an invalid CSR."""
    n = len(recs)
    G = len(group_off) - 1
    for g in range(G):
        if group_off[g + 1] < group_off[g]:
            return None
        if any(int(m) >= n for m in group_members[group_off[g]:group_off[g + 1]]):
            return None
    chains = {}
    nodes = {}  # prefix tuple -> ordinal
    key, parent, depth, gnode = [], [], [], []
    for g in range(G):
        common = None
        for m in group_members[group_off[g]:group_off[g + 1]]:
            m = int(m)
            if m not in chains:
                chains[m] = record_chain(recs[m], paths[m])
            c = chains[m]
            if not c:
                continue
            if common is None:
                common = list(c)
            else:
                k = 0
                while k < min(len(common), len(c)) and common[k] == c[k]:
                    k += 1
                common = common[:k]
        common = common or []
        for t in range(len(common)):
            pre = tuple(common[:t + 1])
            if pre not in nodes:
                nodes[pre] = len(key)
                key.append(common[t])
                parent.append(nodes[pre[:-1]] if t else NO_NODE)
                depth.append(t)
        gnode.append(nodes[tuple(common)] if common else NO_NODE)
    return dict(group_node=gnode, key=key, parent=parent, depth=depth)


def forest_valid(dev_node, parent, depth):
    n_nodes = len(parent)
    for v in range(n_nodes):
        p, d = int(parent[v]), int(depth[v])
        if d >= MAX_DEPTH:
            return False
        if p == NO_NODE:
            if d != 0:
                return False
        elif p >= v or d != int(depth[p]) + 1:
            return False
    return all(int(x) == NO_NODE or int(x) < n_nodes for x in (dev_node if dev_node is not None else []))


def preferred(dev_numa, dev_node, parent, depth, requests):
    """[(available, must-include, size)] -> one position list per request, or None when anything is invalid."""
    if not forest_valid(dev_node, parent, depth):
        return None

    def path_of(p):  # the device's nodes, root first
        v = NO_NODE if dev_node is None else int(dev_node[p])
        out = []
        while v != NO_NODE:
            out.append(v)
            v = int(parent[v])
        return out[::-1]

    answers = []
    for avail, must, size in requests:
        avail, must = [int(x) for x in avail], [int(x) for x in must]
        n = len(dev_numa)
        if (any(p >= n for p in avail + must) or len(set(avail)) != len(avail) or len(set(must)) != len(must)
                or not set(must) <= set(avail) or size < len(must) or size > len(avail)):
            return None
        paths = {p: path_of(p) for p in avail}
        members = {}
        for p in avail:
            for v in paths[p]:
                members.setdefault(v, []).append(p)
        mset = set(must)

        def node_key(v):
            d = int(depth[v])
            up = []
            a = int(parent[v])
            while a != NO_NODE:
                up.append(len(members[a]))
                a = int(parent[a])
            return (len(members[v]), -d, tuple(up), min(members[v]))

        qual = [v for v in members if sum(p in mset for p in members[v]) == len(must) and len(members[v]) >= size]
        X = min(qual, key=node_key) if qual else None
        in_x = [p for p in avail if p not in mset and (X is None or X in paths[p])]

        def lca(p):
            best = None
            for m in must:
                common = [a for a, b in zip(paths[p], paths[m]) if a == b]
                if common and (best is None or len(common) - 1 > best):
                    best = len(common) - 1
            return best

        U = {PT._home(dev_numa[p]) for p in must} - {64}
        c = {}
        for p in in_x:
            c[PT._home(dev_numa[p])] = c.get(PT._home(dev_numa[p]), 0) + 1

        def order(p):
            l = lca(p)
            k = PT._home(dev_numa[p])
            return (MAX_DEPTH if l is None else MAX_DEPTH - 1 - l, 2 if k == 64 else (0 if k in U else 1), -c[k], k, p)
        answers.append(must + sorted(in_x, key=order)[:size - len(must)])
    return answers
