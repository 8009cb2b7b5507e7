"""Independent Python restatement of the calls for mdev vGPUs on SR-IOV VFs (include/kxpu.h, additions to ABI v14), the
second checker next to tests/mdev_pf_oracle.c: kxpu_mdev_pf with a regular expression and a dict from PCI address to
the first record carrying it, and kxpu_dra_slices_mdev_pf as ResourceSlices built as dicts in the stated field order and
written with json.dumps(..., separators=(",", ":")).  Argument and domain checks are the header's, in its order.  It
shares no code with the kernels."""
import json
import re

import numpy as np

from pyref_dra import MAX_DEVICES, SLICE, subdomain_ok
from pyref_dra_taint import EFFECTS, SINCE_MAX, TAINT_SLICE, key_ok, time_added, value_ok

NO_PF = 0xFFFFFFFF
PHYSFN_ERR = 0x01
_CANON = re.compile(rb"[0-9a-f]{4}:[0-9a-f]{2}:[01][0-9a-f]\.[0-7]\Z")
_NAME = re.compile(rb"[A-Za-z0-9_.-]*\Z")
_TYPE = re.compile(rb"[A-Za-z0-9_.-]{1,40}\Z")
_UUID = re.compile(rb"[0-9a-f]{8}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{12}\Z")
_ADDR = re.compile(rb"[0-9a-f:.]{1,16}\Z")
_ADDR0 = re.compile(rb"[0-9a-f:.]{0,16}\Z")
_ROOT = re.compile(rb"pci[0-9a-f:]{1,13}\Z")
_VENDOR = re.compile(rb"[0-9a-f]{1,6}\Z")
_DEVICE = re.compile(rb"[0-9a-f]{0,6}\Z")


def _text(field):
    return bytes(field).split(b"\0", 1)[0]


def mdev_pf(recs, mrecs, msrs):
    """pf_of as a list: the first PCI record whose address is the mdev's canonical physfn, unless physfn is flagged,
    equals the mdev's own parent or matches nothing"""
    first = {}
    for i, r in enumerate(recs):
        b = _text(r["bdf"])
        if _CANON.match(b):
            first.setdefault(b, i)
    out = []
    for m, s in zip(mrecs, msrs):
        pf = _text(s["physfn"])
        ok = _CANON.match(pf) and not int(s["flags"]) & PHYSFN_ERR and pf != _text(m["parent"])
        out.append(first.get(pf, NO_PF) if ok else NO_PF)
    return out


def _cut(rec, field):
    return np.asarray(rec)[field].tobytes().split(b"\0", 1)[0]


def why(rec):
    """name of the first domain rule the record breaks, or None"""
    d = rec["dev"]
    plen = int(d["product_len"])
    if plen <= 64 and not _NAME.match(bytes(d["product"][:plen])):
        return "product"
    if not _TYPE.match(_cut(d, "mdev_type")):
        return "mdev_type"
    if not _UUID.match(np.asarray(d)["uuid"].tobytes()):
        return "uuid"
    if not _ADDR.match(_cut(d, "parent")):
        return "parent"
    root = _cut(d, "pcie_root")
    if root and not _ROOT.match(root):
        return "pcie_root"
    if not _VENDOR.match(_cut(d, "vendor")):
        return "vendor"
    if not _DEVICE.match(_cut(d, "device")):
        return "device"
    if int(d["iommu_group"]) == 0xFFFFFFFF:
        return "iommu_group"
    if plen > 64:
        return "product_len"
    if not _ADDR0.match(_cut(rec, "physfn")):
        return "physfn"
    pd = _cut(rec, "physfn_device")
    if not _DEVICE.match(pd) or (pd and not _cut(rec, "physfn")):
        return "physfn_device"
    return None


def device(rec):
    d = rec["dev"]
    g, mask = int(d["iommu_group"]), int(d["numa_mask"])
    a = {"iommuGroup": {"int": g}, "mdevType": {"string": _cut(d, "mdev_type").decode()}}
    if mask and not mask & (mask - 1):
        a["numaNode"] = {"int": mask.bit_length() - 1}
    a["parentAddress"] = {"string": _cut(d, "parent").decode()}
    if _cut(d, "device"):
        a["parentDeviceID"] = {"string": _cut(d, "device").decode()}
    a["parentVendorID"] = {"string": _cut(d, "vendor").decode()}
    if _cut(rec, "physfn"):
        a["physfnAddress"] = {"string": _cut(rec, "physfn").decode()}
    if _cut(rec, "physfn_device"):
        a["physfnDeviceID"] = {"string": _cut(rec, "physfn_device").decode()}
    if int(d["product_len"]):
        a["productName"] = {"string": bytes(d["product"][:int(d["product_len"])]).decode()}
    if _cut(d, "pcie_root"):
        a["resource.kubernetes.io/pcieRoot"] = {"string": _cut(d, "pcie_root").decode()}
    a["uuid"] = {"string": np.asarray(d)["uuid"].tobytes().decode()}
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
