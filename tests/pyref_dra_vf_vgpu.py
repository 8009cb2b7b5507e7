"""Independent Python restatement of kxpu_dra_slices_vf_vgpu (include/kxpu.h, addition to ABI v14), the second checker
next to tests/dra_vf_vgpu_oracle.c: the ResourceSlices are built as dicts in the stated field order, each taint's
timeAdded comes from datetime, and the slices are written with json.dumps(..., separators=(",", ":")).  Argument and
domain checks are the header's, in its order."""
import json
import re

import numpy as np

from pyref_dra import MAX_DEVICES, SLICE, subdomain_ok
from pyref_dra_taint import EFFECTS, SINCE_MAX, TAINT_SLICE, key_ok, time_added, value_ok

_NAME = re.compile(rb"[A-Za-z0-9_.-]*\Z")
_KEY = re.compile(rb"[A-Za-z0-9_.-]{1,40}\Z")
_ADDR = re.compile(rb"[0-9a-f:.]{1,16}\Z")
_ROOT = re.compile(rb"pci[0-9a-f:]{1,13}\Z")
_VENDOR = re.compile(rb"[0-9a-f]{1,6}\Z")
_DEVICE = re.compile(rb"[0-9a-f]{0,6}\Z")


def _cut(rec, field):
    """the field's bytes before the first NUL"""
    return np.asarray(rec)[field].tobytes().split(b"\0", 1)[0]


def why(rec):
    """name of the first domain rule the record breaks, or None"""
    plen = int(rec["product_len"])
    if plen <= 64 and not _NAME.match(bytes(rec["product"][:plen])):
        return "product"
    if not _KEY.match(_cut(rec, "type_key")):
        return "type_key"
    if not _ADDR.match(_cut(rec, "bdf")):
        return "bdf"
    if not _ADDR.match(_cut(rec, "parent")):
        return "parent"
    root = _cut(rec, "pcie_root")
    if root and not _ROOT.match(root):
        return "pcie_root"
    if not _VENDOR.match(_cut(rec, "vendor")):
        return "vendor"
    if not _DEVICE.match(_cut(rec, "device")):
        return "device"
    if int(rec["iommu_group"]) == 0xFFFFFFFF:
        return "iommu_group"
    if int(rec["type_id"]) == 0:
        return "type_id"
    if plen > 64:
        return "product_len"
    return None


def device(rec):
    g, mask = int(rec["iommu_group"]), int(rec["numa_mask"])
    a = {"iommuGroup": {"int": g}}
    if mask and not mask & (mask - 1):
        a["numaNode"] = {"int": mask.bit_length() - 1}
    a["parentAddress"] = {"string": _cut(rec, "parent").decode()}
    if _cut(rec, "device"):
        a["parentDeviceID"] = {"string": _cut(rec, "device").decode()}
    a["parentVendorID"] = {"string": _cut(rec, "vendor").decode()}
    a["pciAddress"] = {"string": _cut(rec, "bdf").decode()}
    if int(rec["product_len"]):
        a["productName"] = {"string": bytes(rec["product"][:int(rec["product_len"])]).decode()}
    if _cut(rec, "pcie_root"):
        a["resource.kubernetes.io/pcieRoot"] = {"string": _cut(rec, "pcie_root").decode()}
    a["vgpuType"] = {"string": _cut(rec, "type_key").decode()}
    a["vgpuTypeID"] = {"int": int(rec["type_id"])}
    assert list(a) == sorted(a)  # encoding/json's map key order
    return {"name": "vfio%d" % g, "attributes": a}


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
