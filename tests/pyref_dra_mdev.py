"""Independent Python restatement of kxpu_dra_slices_mdev (include/kxpu.h, ABI v10), the second checker next to
oracle/kxpu_dra_mdev_oracle.c: the ResourceSlices are built as dicts in the stated field order and written with
json.dumps(..., separators=(",", ":")).  Argument and domain checks are the header's, in its order."""
import json
import re

import numpy as np

from pyref_dra import MAX_DEVICES, SLICE, subdomain_ok

_NAME = re.compile(rb"[A-Za-z0-9_.-]*\Z")
_TYPE = re.compile(rb"[A-Za-z0-9_.-]{1,40}\Z")
_UUID = re.compile(rb"[0-9a-f]{8}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{4}-[0-9a-f]{12}\Z")
_PARENT = re.compile(rb"[0-9a-f:.]{1,16}\Z")
_ROOT = re.compile(rb"pci[0-9a-f:]{1,13}\Z")
_VENDOR = re.compile(rb"[0-9a-f]{1,6}\Z")
_DEVICE = re.compile(rb"[0-9a-f]{0,6}\Z")


def _raw(rec, field):
    """all bytes of a fixed-width string field (indexing one would drop its trailing NULs)"""
    return np.asarray(rec)[field].tobytes()


def _cut(rec, field):
    """the field's bytes before the first NUL"""
    return _raw(rec, field).split(b"\0", 1)[0]


def why(rec):
    """name of the first domain rule the record breaks, or None"""
    plen = int(rec["product_len"])
    if plen <= 64 and not _NAME.match(bytes(rec["product"][:plen])):
        return "product"
    if not _TYPE.match(_cut(rec, "mdev_type")):
        return "mdev_type"
    if not _UUID.match(_raw(rec, "uuid")):
        return "uuid"
    if not _PARENT.match(_cut(rec, "parent")):
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
    if plen > 64:
        return "product_len"
    return None


def device(rec):
    g = int(rec["iommu_group"])
    mask = int(rec["numa_mask"])
    a = {"iommuGroup": {"int": g}, "mdevType": {"string": _cut(rec, "mdev_type").decode()}}
    if mask and not mask & (mask - 1):
        a["numaNode"] = {"int": mask.bit_length() - 1}
    a["parentAddress"] = {"string": _cut(rec, "parent").decode()}
    if _cut(rec, "device"):
        a["parentDeviceID"] = {"string": _cut(rec, "device").decode()}
    a["parentVendorID"] = {"string": _cut(rec, "vendor").decode()}
    if int(rec["product_len"]):
        a["productName"] = {"string": bytes(rec["product"][:int(rec["product_len"])]).decode()}
    if _cut(rec, "pcie_root"):
        a["resource.kubernetes.io/pcieRoot"] = {"string": _cut(rec, "pcie_root").decode()}
    a["uuid"] = {"string": _raw(rec, "uuid").decode()}
    assert list(a) == sorted(a)  # encoding/json's map key order
    return {"name": "vfio%d" % g, "attributes": a}


def slices(driver, pool, node, generation, devs):
    """(bytes, slice_off), or -1 (bad argument), or (-7, reason) as the oracle returns them"""
    if not (subdomain_ok(driver, 63) and subdomain_ok(pool, 253) and subdomain_ok(node, 253) and 0 <= generation < 1 << 63):
        return -1
    if len(devs) >= MAX_DEVICES:
        return -7, None
    for r in devs:
        w = why(r)
        if w:
            return -7, w
    driver, pool, node = (x.decode() if isinstance(x, bytes) else x for x in (driver, pool, node))
    count = max(1, -(-len(devs) // SLICE))
    out, offs = b"", []
    for s in range(count):
        obj = {"kind": "ResourceSlice", "apiVersion": "resource.k8s.io/v1",
               "metadata": {"generateName": "%s-%s-" % (node, driver)},
               "spec": {"driver": driver, "pool": {"name": pool, "generation": generation, "resourceSliceCount": count},
                        "nodeName": node, "devices": [device(r) for r in devs[s * SLICE:(s + 1) * SLICE]]}}
        offs.append(len(out))
        out += json.dumps(obj, separators=(",", ":")).encode() + b"\n"
    offs.append(len(out))
    return out, offs
