"""Independent Python restatement of kxpu_pcie_ports and kxpu_dra_slices_pcie (include/kxpu.h, additions to ABI v14),
the second checker next to tests/dra_pcie_oracle.c.  Paths are parsed with regular expressions, each group's chain is
the longest common prefix of lists, and the slice devices are dicts whose keys are sorted before json.dumps: no
insertion position is computed.  It shares no code with the kernels."""
import json
import re

import numpy as np

import pyref_dra_pf
from pyref_dra import MAX_DEVICES, SLICE, subdomain_ok
from pyref_dra_taint import EFFECTS, SINCE_MAX, TAINT_SLICE, key_ok, time_added, value_ok

NO_KEY = (1 << 64) - 1
MAXD = 8
_DOM = rb"([0-9a-f]{4}|[1-9a-f][0-9a-f]{4,7})"
_HB = re.compile(rb"pci" + _DOM + rb":([0-9a-f]{2})\Z")
_FN = re.compile(_DOM + rb":([0-9a-f]{2}):([01][0-9a-f])\.([0-7])\Z")


def comp_key(c):
    """node key of one path component, or None"""
    if c.startswith(b"pci"):
        m = _HB.match(c)
        return None if not m else 1 << 63 | int(m[1], 16) << 16 | int(m[2], 16) << 8
    m = _FN.match(c)
    return None if not m else int(m[1], 16) << 16 | int(m[2], 16) << 8 | int(m[3], 16) << 3 | int(m[4])


def chain(rec, path):
    """the record's chain (list of keys), [] when the path is unknown"""
    n = int(path["len"])
    if not 0 < n <= 120:
        return []
    comps = bytes(path["path"]).ljust(120, b"\0")[:n].split(b"/")
    if not 2 <= len(comps) <= MAXD + 1:
        return []
    keys = [comp_key(c) for c in comps]
    if any(k is None for k in keys) or not keys[0] >> 63:
        return []
    if comps[-1] != bytes(rec["bdf"]).split(b"\0", 1)[0][:16]:
        return []
    return keys[:-1]


def rule(ch):
    """(root port, switch) of a chain: f0, f1, ... after the last host bridge; f0 and f_j for the greatest odd j"""
    hb = max((t for t, k in enumerate(ch) if k >> 63), default=None)
    fs = [] if hb is None else ch[hb + 1:]
    rp = fs[0] if fs else NO_KEY
    odd = [j for j in range(len(fs)) if j % 2 == 1]
    return rp, fs[odd[-1]] if odd else NO_KEY


def pcie_ports(recs, paths, group_off, group_members):
    """(root_port, switch) lists, or -1 (KXPU_E_INVALID) for decreasing offsets or a member index >= n"""
    G = len(group_off) - 1
    if any(group_off[g + 1] < group_off[g] for g in range(G)):
        return -1
    chains = [chain(recs[i], paths[i]) for i in range(len(recs))]
    rp, sw = [], []
    for g in range(G):
        members = [int(x) for x in group_members[group_off[g]:group_off[g + 1]]]
        if any(i >= len(recs) for i in members):
            return -1
        known = [chains[i] for i in members if chains[i]]
        pre = []
        if known:
            for t in range(min(len(c) for c in known)):
                if len({c[t] for c in known}) > 1:
                    break
                pre.append(known[0][t])
        a, b = rule(pre)
        rp.append(a)
        sw.append(b)
    return rp, sw


def address(key):
    """a function key's sysfs address"""
    dom = key >> 16
    return "%s:%02x:%02x.%d" % ("%04x" % dom if dom <= 0xffff else "%x" % dom, key >> 8 & 0xff, key >> 3 & 0x1f, key & 7)


def domain_ok(d):
    d = d.decode() if isinstance(d, bytes) else d
    if d is None or not subdomain_ok(d, 63):
        return False
    return not any(d == r or d.endswith("." + r) for r in ("kubernetes.io", "k8s.io"))


def why(rec):
    w = pyref_dra_pf.why(rec["pf"])
    if w:
        return w
    rp, sw = int(rec["root_port"]), int(rec["pcie_switch"])
    if any(k != NO_KEY and k >> 48 for k in (rp, sw)):
        return "port_key"
    if sw != NO_KEY and rp == NO_KEY:
        return "port_orphan"
    return None


def device(rec, domain):
    a = dict(pyref_dra_pf.device(rec["pf"])["attributes"])
    if int(rec["root_port"]) != NO_KEY:
        a[domain + "/pcieRootPort"] = {"string": address(int(rec["root_port"]))}
    if int(rec["pcie_switch"]) != NO_KEY:
        a[domain + "/pcieSwitch"] = {"string": address(int(rec["pcie_switch"]))}
    return {"name": "vfio%d" % int(rec["pf"]["dev"]["iommu_group"]), "attributes": {k: a[k] for k in sorted(a)}}


def _s(x):
    return x.decode("ascii", "replace") if isinstance(x, bytes) else x


def slices(driver, pool, node, generation, domain, devs, taints=(), since=None):
    """(bytes, slice_off), or -1 (bad argument), or (-7, reason) as the C oracle returns them"""
    if not (subdomain_ok(driver, 63) and subdomain_ok(pool, 253) and subdomain_ok(node, 253) and 0 <= generation < 1 << 63):
        return -1
    if domain is None or not domain_ok(domain):
        return -1
    domain = _s(domain)
    if since is not None:
        if not 0 < len(taints) <= 4:
            return -1
        for k, v, e in taints:
            if k is None or not (key_ok(k) and value_ok(v) and _s(e) in EFFECTS):
                return -1
        since = np.asarray(since, np.int64).reshape(len(devs), len(taints))
    if len(devs) >= MAX_DEVICES:
        return -7, None
    for i, r in enumerate(devs):
        w = why(r)
        row = [] if since is None else [int(x) for x in since[i]]
        if not w and any(t > SINCE_MAX for t in row):
            w = "taint_since"
        if not w:
            carried = [(_s(taints[t][0]), _s(taints[t][2])) for t in range(len(row)) if row[t] >= 0]
            if len(set(carried)) < len(carried):
                w = "taint_duplicate"
        if w:
            return -7, w
    driver, pool, node = (_s(x) for x in (driver, pool, node))
    per = SLICE if since is None else TAINT_SLICE
    count = max(1, -(-len(devs) // per))
    out, offs = b"", []
    for s in range(count):
        devices = []
        for i in range(s * per, min(len(devs), (s + 1) * per)):
            d = device(devs[i], domain)
            if since is not None and (since[i] >= 0).any():
                d["taints"] = []
                for t, (k, v, e) in enumerate(taints):
                    if since[i, t] >= 0:
                        entry = {"key": _s(k)}
                        if _s(v):
                            entry["value"] = _s(v)
                        entry["effect"] = _s(e)
                        entry["timeAdded"] = time_added(int(since[i, t]))
                        d["taints"].append(entry)
            devices.append(d)
        obj = {"kind": "ResourceSlice", "apiVersion": "resource.k8s.io/v1",
               "metadata": {"generateName": "%s-%s-" % (node, driver)},
               "spec": {"driver": driver, "pool": {"name": pool, "generation": generation, "resourceSliceCount": count},
                        "nodeName": node, "devices": devices}}
        offs.append(len(out))
        out += json.dumps(obj, separators=(",", ":")).encode() + b"\n"
    offs.append(len(out))
    return out, offs
