"""Independent Python restatement of kxpu_dra_slices (include/kxpu.h, ABI v9), the second checker next to
oracle/kxpu_dra_oracle.c: the ResourceSlices are built as dicts in the stated field order and written with
json.dumps(..., separators=(",", ":")).  Argument and domain checks are the header's, in its order."""
import json
import re

SLICE = 128
MAX_DEVICES = 1 << 24
_LABEL = re.compile(r"[a-z0-9]([-a-z0-9]*[a-z0-9])?\Z")
_PRODUCT = re.compile(rb"[A-Za-z0-9_.-]*\Z")
_BDF = re.compile(rb"[0-9a-f:.]{1,16}\Z")
_ROOT = re.compile(rb"pci[0-9a-f:]{1,13}\Z")
_ID = re.compile(rb"[0-9a-f]{1,6}\Z")


def subdomain_ok(s, limit):
    if isinstance(s, bytes):
        try:
            s = s.decode("ascii")
        except UnicodeDecodeError:
            return False
    return 0 < len(s) <= limit and all(len(p) <= 63 and _LABEL.match(p) for p in s.split("."))


def _cut(b):
    """bytes before the first NUL"""
    b = bytes(b)
    return b.split(b"\0", 1)[0]


def why(rec):
    """name of the first domain rule the record breaks, or None"""
    plen = int(rec["product_len"])
    if plen <= 64 and not _PRODUCT.match(bytes(rec["product"][:plen])):
        return "product"
    if not _BDF.match(_cut(rec["bdf"])):
        return "bdf"
    root = _cut(rec["pcie_root"])
    if root and not _ROOT.match(root):
        return "pcie_root"
    for f in ("vendor", "device"):
        if not _ID.match(_cut(rec[f])):
            return f
    if int(rec["iommu_group"]) == 0xFFFFFFFF:
        return "iommu_group"
    if plen > 64:
        return "product_len"
    return None


def device(rec):
    g = int(rec["iommu_group"])
    mask = int(rec["numa_mask"])
    a = {"deviceID": {"string": _cut(rec["device"]).decode()}, "iommuGroup": {"int": g}}
    if mask and not mask & (mask - 1):
        a["numaNode"] = {"int": mask.bit_length() - 1}
    a["pciAddress"] = {"string": _cut(rec["bdf"]).decode()}
    if int(rec["product_len"]):
        a["productName"] = {"string": bytes(rec["product"][:int(rec["product_len"])]).decode()}
    root = _cut(rec["pcie_root"])
    if root:
        a["resource.kubernetes.io/pcieRoot"] = {"string": root.decode()}
    a["vendorID"] = {"string": _cut(rec["vendor"]).decode()}
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
