"""Independent pure-Python restatement of discovery for accelerators of any configured vendor, for small inputs:
createIommuDeviceMap with a (vendor, driver) rule list and the CDI spec with the kind as a parameter.  Written
from the Go source with Python's own str / re / json machinery (like pyref.py), so it shares no code with
oracle/kxpu_xpu_oracle.c."""
import json
import re

from pyref import bdf_ok, yaml_scalar


def cdi_yaml(devs, kind):
    """pyref.cdi_yaml with the CDI kind (CdiVendorClass in the reference) as a parameter; devs: (bdf, group, index)."""
    if not all(bdf_ok(bdf) for bdf, _, _ in devs):
        return None
    out = ["cdiVersion: 0.6.0", "kind: %s" % yaml_scalar(kind)]
    if not devs:
        out.append("devices: []")
        return ("\n".join(out) + "\n").encode()
    out.append("devices:")
    for bdf, group, index in devs:
        ann = {"attach-pci": "true", "bdf": bdf, "cdi.k8s.io/vfio%d" % group: "%s=%d" % (kind, index)}
        out.append("  - name: %s" % yaml_scalar(str(index)))
        out.append("    annotations:")
        for k in sorted(ann):
            out.append("      %s: %s" % (k, yaml_scalar(ann[k])))
        out.append("    containerEdits:")
        out.append("      deviceNodes:")
        out.append("        - path: /dev/vfio/%d" % group)
    return ("\n".join(out) + "\n").encode()


def cdi_json(devs, kind):
    if not all(bdf_ok(bdf) for bdf, _, _ in devs):
        return None
    spec = {"cdiVersion": "0.6.0", "kind": kind}
    if not devs:
        spec["devices"] = None
    else:
        spec["devices"] = [
            {"name": str(index),
             "annotations": dict(sorted({"attach-pci": "true", "bdf": bdf,
                                         "cdi.k8s.io/vfio%d" % group: "%s=%d" % (kind, index)}.items())),
             "containerEdits": {"deviceNodes": [{"path": "/dev/vfio/%d" % group}]}}
            for bdf, group, index in devs]
    spec["containerEdits"] = {}
    return json.dumps(spec, indent=2).encode()


KIND_RE = re.compile(r"[A-Za-z](?:[A-Za-z0-9_.-]*[A-Za-z0-9])?/[A-Za-z](?:[A-Za-z0-9_-]*[A-Za-z0-9])?")


def kind_ok(kind: str) -> bool:
    """The CDI kind domain of kxpu_cdi_emit_kind: vendor/class as CDI pkg/parser accepts them, narrowed to
    letter-first, alphanumeric-last parts, at most 63 bytes."""
    return len(kind) <= 63 and KIND_RE.fullmatch(kind) is not None


def rules_ok(rules) -> bool:
    """kxpu_classify_rules' rule-list validity; rules: list of (vendor bytes, driver bytes) as the NUL-padded
    fields hold them (trailing NULs stripped)."""
    if not 1 <= len(rules) <= 16 or len(set(rules)) != len(rules):
        return False
    for v, d in rules:
        if not 1 <= len(v) <= 6 or b"\n" in v or b"\0" in v:
            return False
        if not 1 <= len(d) <= 15 or b"/" in d or b"\0" in d:
            return False
    return True


def classify_rules(rules, recs):
    """classify() with a (vendor, driver) rule list in place of ("10de", "vfio-pci"): one walk, one busIndex; the
    device map is keyed by (rule of the group's first member, device id).  Returns (iommu_map, device_map, accept)
    with device_map keys (rule index, device id bytes); None for an invalid rule list."""
    if not rules_ok(rules):
        return None
    iommu, devmap, accept = {}, {}, []
    bus = 0
    for r in recs:
        accept.append(None)
        if r.get("is_dir") or r.get("vendor") is None or len(r["vendor"]) < 2:
            continue
        vendor = r["vendor"][2:].strip(b"\n")
        if r.get("driver") is None:
            continue
        match = [k for k, (v, d) in enumerate(rules) if vendor == v and r["driver"] == d]
        if not match:
            continue
        if r.get("group") is None:
            continue
        g = r["group"]
        if g not in iommu:
            if r.get("device") is None or len(r["device"]) < 2:
                continue
            dev = r["device"][2:].strip(b"\n")
            devmap.setdefault((match[0], dev), []).append(g)
        iommu.setdefault(g, []).append((r["bdf"], bus))
        accept[-1] = bus
        bus += 1
    return iommu, devmap, accept
