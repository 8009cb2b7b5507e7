"""Independent Python restatement of kxpu_pcie_ports_mdev, kxpu_dra_slices_mdev_pcie and kxpu_dra_slices_vf_vgpu_pcie
(include/kxpu.h, additions to ABI v14).  The parent chain is pyref_pcie_mdev's chain less its last key, the rule is
pyref_dra_pcie's, and the slice devices are dicts whose keys are sorted before json.dumps: no insertion position is
computed.  It shares no code with the kernels."""
import json

import numpy as np

import pyref_dra_vf_vgpu
import pyref_mdev_pf
from pyref_dra import MAX_DEVICES, SLICE, subdomain_ok
from pyref_dra_pcie import NO_KEY, address, domain_ok, rule
from pyref_dra_taint import EFFECTS, SINCE_MAX, TAINT_SLICE, key_ok, time_added, value_ok
from pyref_pcie_mdev import record_chain


def pcie_ports_mdev(recs, paths, group_off, group_members):
    """(root_port, switch) lists, or -1 (KXPU_E_INVALID) for decreasing offsets or a member index >= n"""
    G = len(group_off) - 1
    if any(group_off[g + 1] < group_off[g] for g in range(G)):
        return -1
    chains = [list(record_chain(recs[i], paths[i]) or [])[:-1] for i in range(len(recs))]
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


def _ports_why(rec):
    rp, sw = int(rec["root_port"]), int(rec["pcie_switch"])
    if any(k != NO_KEY and k >> 48 for k in (rp, sw)):
        return "port_key"
    if sw != NO_KEY and rp == NO_KEY:
        return "port_orphan"
    return None


def _with_ports(dev, rec, domain):
    a = dict(dev["attributes"])
    if int(rec["root_port"]) != NO_KEY:
        a[domain + "/pcieRootPort"] = {"string": address(int(rec["root_port"]))}
    if int(rec["pcie_switch"]) != NO_KEY:
        a[domain + "/pcieSwitch"] = {"string": address(int(rec["pcie_switch"]))}
    return {"name": dev["name"], "attributes": {k: a[k] for k in sorted(a)}}


# per layout: the first member's name, its domain rules and its device
LAYOUTS = {"mdev": ("pf", pyref_mdev_pf.why, pyref_mdev_pf.device),
           "vf_vgpu": ("dev", pyref_dra_vf_vgpu.why, pyref_dra_vf_vgpu.device)}


def _s(x):
    return x.decode("ascii", "replace") if isinstance(x, bytes) else x


def slices(layout, driver, pool, node, generation, domain, devs, taints=(), since=None):
    """(bytes, slice_off), or -1 (bad argument), or (-7, reason) as the C oracles return them"""
    field, why, device = LAYOUTS[layout]
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
        w = why(r[field]) or _ports_why(r)
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
            d = _with_ports(device(devs[i][field]), devs[i], domain)
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
