"""Independent Python restatement of kxpu_dra_slices_pf (include/kxpu.h, addition to ABI v14), the second checker next
to tests/dra_pf_oracle.c: ResourceSlices built as dicts in the stated field order and written with
json.dumps(..., separators=(",", ":")).  Argument and domain checks are the header's, in its order.  It shares no code
with the kernels."""
import json
import re

import numpy as np

import pyref_dra
from pyref_dra import MAX_DEVICES, SLICE, subdomain_ok
from pyref_dra_taint import EFFECTS, SINCE_MAX, TAINT_SLICE, key_ok, time_added, value_ok

_ADDR0 = re.compile(rb"[0-9a-f:.]{0,16}\Z")
_DEVICE = re.compile(rb"[0-9a-f]{0,6}\Z")


def _cut(rec, field):
    return np.asarray(rec)[field].tobytes().split(b"\0", 1)[0]


def why(rec):
    """name of the first domain rule the record breaks, or None"""
    w = pyref_dra.why(rec["dev"])
    if w:
        return w
    if not _ADDR0.match(_cut(rec, "physfn")):
        return "physfn"
    pd = _cut(rec, "physfn_device")
    if not _DEVICE.match(pd) or (pd and not _cut(rec, "physfn")):
        return "physfn_device"
    return None


def device(rec):
    """the v9 device of rec's dev with physfnAddress and physfnDeviceID put in key order"""
    a = dict(pyref_dra.device(rec["dev"])["attributes"])
    if _cut(rec, "physfn"):
        a["physfnAddress"] = {"string": _cut(rec, "physfn").decode()}
    if _cut(rec, "physfn_device"):
        a["physfnDeviceID"] = {"string": _cut(rec, "physfn_device").decode()}
    a = {k: a[k] for k in sorted(a)}  # encoding/json's map key order
    return {"name": "vfio%d" % int(rec["dev"]["iommu_group"]), "attributes": a}


def _s(x):
    return x.decode("ascii", "replace") if isinstance(x, bytes) else x


def slices(driver, pool, node, generation, devs, taints=(), since=None):
    """(bytes, slice_off), or -1 (bad argument), or (-7, reason) as the C oracle returns them.  taints: [(key, value,
    effect)]; since: None or an int [n, len(taints)] array"""
    if not (subdomain_ok(driver, 63) and subdomain_ok(pool, 253) and subdomain_ok(node, 253) and 0 <= generation < 1 << 63):
        return -1
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
            d = device(devs[i])
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
