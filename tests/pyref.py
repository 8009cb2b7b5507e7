"""Independent pure-Python restatement of the reference semantics, for small inputs.
Written from the Go source (pkg/device_plugin/device_plugin.go, cdi/spec.go) with Python's
own str / re / json machinery, so it shares no code with oracle/kxpu_oracle.c."""
import json
import re

GO_SPACE = "\t\n\v\f\r \x85\xa0                　"
MAX_TOKEN = 65536


def scan_lines(data: bytes):
    """bufio.Scanner + ScanLines: yields lines; stops (ErrTooLong) at a line >= 64 KiB."""
    pos, n = 0, len(data)
    while pos < n:
        nl = data.find(b"\n", pos)
        end = n if nl < 0 else nl
        if end - pos >= MAX_TOKEN:
            return
        line = data[pos:end]
        if line.endswith(b"\r"):
            line = line[:-1]
        yield pos, line
        pos = n if nl < 0 else nl + 1


def go_upper(ch: str) -> str:
    u = ch.upper()
    return u if len(u) == 1 else ch  # Go uses the simple (1:1) case mapping


def sanitise(rest: bytes) -> bytes:
    """device_plugin.go:242-251 on the text after the "\\t<id>" prefix."""
    s = rest.decode("utf-8", errors="replace")  # invalid bytes -> U+FFFD, deleted below anyway
    s = s.strip(GO_SPACE)
    s = "".join(go_upper(c) for c in s)
    s = s.replace("/", "_").replace(".", "_")
    s = re.sub(r"[\t\n\f\r ]+", "_", s)
    s = re.sub(r"[^a-zA-Z0-9_.]+", "", s)
    return s.encode()


def get_device_name(data: bytes, vendor: bytes, device: bytes):
    """Returns (line offset, name) or (-1, None).  locateVendor + getDeviceName."""
    it = scan_lines(data)
    for _, line in it:
        if line.startswith(vendor):
            break
    else:
        return -1, None
    prefix = b"\t" + device
    for off, line in it:
        if line.startswith(b"#"):
            continue
        if not line.startswith(b"\t"):
            return -1, None
        if not line.startswith(prefix):
            continue
        return off, sanitise(line[len(prefix):])
    return -1, None


BASE60 = re.compile(r"^[-+]?[0-9][0-9_]*(?::[0-5]?[0-9])+(?:\.[0-9_]*)?$")
# the bdfs over [0-9a-f:.] that yaml.v3 would not write plain or base-60 double-quoted (include/kxpu.h, the bdf domain of
# kxpu_cdi_emit_kind): an int (all digits, 0b + binary digits), a float of resolve.go's yamlStyleFloat, a trailing ':',
# a leading "..."
_BDF_NOT_PLAIN = re.compile(r"[0-9]+|0b[01]+|[0-9]+(\.[0-9]*)?(e[0-9]+)?|\.[0-9]+(e[0-9]+)?|.*:|\.\.\..*", re.S)


def bdf_ok(bdf) -> bool:
    """The bdf (or mdev parent) domain of every CDI spec emitter: 1..16 bytes over [0-9a-f:.] that YAML keeps a string."""
    s = bdf.decode("latin-1") if isinstance(bdf, (bytes, bytearray)) else bdf
    return re.fullmatch(r"[0-9a-f:.]{1,16}", s) is not None and _BDF_NOT_PLAIN.fullmatch(s) is None


def yaml_scalar(s: str) -> str:
    """yaml.v3 stringv for the strings this spec contains."""
    looks_int = re.fullmatch(r"[-+]?[0-9]+", s) is not None
    if looks_int or s in ("true", "false") or BASE60.match(s):
        return '"%s"' % s
    return s


def cdi_yaml(devs):
    """devs: list of (bdf, group, index); None when a bdf is outside bdf_ok."""
    if not all(bdf_ok(bdf) for bdf, _, _ in devs):
        return None
    out = ["cdiVersion: 0.6.0", "kind: nvidia.com/gpu"]
    if not devs:
        out.append("devices: []")
        return ("\n".join(out) + "\n").encode()
    out.append("devices:")
    for bdf, group, index in devs:
        ann = {"attach-pci": "true", "bdf": bdf, "cdi.k8s.io/vfio%d" % group: "nvidia.com/gpu=%d" % index}
        out.append("  - name: %s" % yaml_scalar(str(index)))
        out.append("    annotations:")
        for k in sorted(ann):
            out.append("      %s: %s" % (k, yaml_scalar(ann[k])))
        out.append("    containerEdits:")
        out.append("      deviceNodes:")
        out.append("        - path: /dev/vfio/%d" % group)
    return ("\n".join(out) + "\n").encode()


def cdi_json(devs):
    if not all(bdf_ok(bdf) for bdf, _, _ in devs):
        return None
    spec = {"cdiVersion": "0.6.0", "kind": "nvidia.com/gpu"}
    if not devs:
        spec["devices"] = None
    else:
        spec["devices"] = [
            {"name": str(index),
             "annotations": dict(sorted({"attach-pci": "true", "bdf": bdf,
                                         "cdi.k8s.io/vfio%d" % group: "nvidia.com/gpu=%d" % index}.items())),
             "containerEdits": {"deviceNodes": [{"path": "/dev/vfio/%d" % group}]}}
            for bdf, group, index in devs]
    spec["containerEdits"] = {}
    return json.dumps(spec, indent=2).encode()


def classify(recs):
    """createIommuDeviceMap over records given as dicts; returns (iommu_map, device_map, accept)
    with insertion-ordered dicts (Go maps are unordered; first-seen order is the canonical one)."""
    iommu, devmap, accept = {}, {}, []
    bus = 0
    for r in recs:
        accept.append(None)
        # an id file shorter than 2 bytes makes the reference panic (data[2:], device_plugin.go:189); the
        # documented behaviour here is "skipped like a read error" (DESIGN.md, domain restrictions)
        if r.get("is_dir") or r.get("vendor") is None or len(r["vendor"]) < 2:
            continue
        vendor = r["vendor"][2:].strip(b"\n")
        if vendor != b"10de":
            continue
        if r.get("driver") is None or r["driver"] != b"vfio-pci":
            continue
        if r.get("group") is None:
            continue
        g = r["group"]
        if g not in iommu:
            if r.get("device") is None or len(r["device"]) < 2:
                continue
            dev = r["device"][2:].strip(b"\n")
            devmap.setdefault(dev, []).append(g)
        iommu.setdefault(g, []).append((r["bdf"], bus))
        accept[-1] = bus
        bus += 1
    return iommu, devmap, accept
