"""Independent Python restatement of kxpu_pcie_tree_mdev (include/kxpu.h, addition to ABI v14), the second checker next
to tests/pcie_mdev_oracle.c: the leaf rule with a regular expression over the split path, the components with
pyref_pcie's expressions, and the forest as a dict from whole prefixes to ordinals, the common prefix by zip().  It shares
no code with the kernels."""
import re

import pyref_pcie as PP

MAX_DEPTH = PP.MAX_DEPTH
NO_NODE = PP.NO_NODE
_UUID = re.compile(r"[0-9a-f]{8}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{12}")


def chain(uuid: bytes, parent: bytes, path: bytes, length: int):
    """The chain keys of an mdev record (its uuid and parent fields, its path), [] when the path is unknown."""
    if not 1 <= length <= 120:
        return []
    try:
        parts = path[:length].decode("ascii").split("/")
    except UnicodeDecodeError:
        return []
    if not 2 <= len(parts) <= MAX_DEPTH + 1:
        return []
    *comps, leaf = parts
    if not _UUID.fullmatch(leaf) or leaf.encode() != bytes(uuid)[:36]:
        return []
    keys = []
    for i, c in enumerate(comps):
        k, kind = PP.component_key(c)
        if kind is None or (i == 0 and kind != "bridge"):
            return []
        keys.append(k)
    if PP.component_key(comps[-1])[1] != "func" or comps[-1].encode() != bytes(parent).split(b"\0", 1)[0]:
        return []
    return keys


def record_chain(rec, path_row):
    return chain(bytes(rec["uuid"]).ljust(36, b"\0"), bytes(rec["parent"]), bytes(path_row["path"]).ljust(120, b"\0"),
                 int(path_row["len"]))


def tree(recs, paths, group_off, group_members):
    """dict(group_node, key, parent, depth) as lists, or None for an invalid CSR."""
    n, G = len(recs), len(group_off) - 1
    for g in range(G):
        if group_off[g + 1] < group_off[g] or any(int(m) >= n for m in group_members[group_off[g]:group_off[g + 1]]):
            return None
    chains = [record_chain(recs[i], paths[i]) for i in range(n)]
    nodes = {}  # whole prefix (tuple of keys) -> ordinal
    out = dict(group_node=[], key=[], parent=[], depth=[])
    for g in range(G):
        known = [chains[int(m)] for m in group_members[group_off[g]:group_off[g + 1]] if chains[int(m)]]
        common = []
        for keys in zip(*known):
            if len(set(keys)) != 1:
                break
            common.append(keys[0])
        for t in range(len(common)):
            pre = tuple(common[:t + 1])
            if pre not in nodes:
                nodes[pre] = len(out["key"])
                out["key"].append(common[t])
                out["parent"].append(nodes[pre[:-1]] if t else NO_NODE)
                out["depth"].append(t)
        out["group_node"].append(nodes[tuple(common)] if common else NO_NODE)
    return out
