"""Plain-Python restatement of kxpu_cdi_emit_vf_vgpu / kxpu_cdi_emit_vf_vgpu_cdev: the CDI spec of a class that serves
vGPUs on SR-IOV VFs, with each VF's type ID and type key in two more annotations.  The JSON document is json.dumps of
the spec as a dict (indent 2, the layout of Go's MarshalIndent for these values); the YAML one is written line by line
with pyref.yaml_scalar's quoting of the bdf and both new values always double-quoted.  annotations() reads a document
back with PyYAML or json and returns each device's annotations as the loader sees them.  parse(...) splits the document
at its device starts, reads each device with a regular expression and accepts the document only when emit() writes the
same bytes from the records read; it returns (status, records)."""
import json
import re

import numpy as np
import yaml

import pyref as P

FMT_YAML, FMT_JSON = 0, 1
KEY = re.compile(rb"[A-Za-z0-9_.-]{1,40}")
KIND = re.compile(rb"[A-Za-z][A-Za-z0-9_.-]*[A-Za-z0-9]?/[A-Za-z][A-Za-z0-9_-]*[A-Za-z0-9]?")


def kind_ok(kind):
    if len(kind) > 63 or not KIND.fullmatch(kind):
        return False
    vendor, klass = kind.split(b"/")
    return all(p[:1].isalpha() and p[-1:].isalnum() for p in (vendor, klass))


def _fields(r):
    d = r["dev"]
    return (bytes(d["bdf"]).decode("latin-1"), int(d["iommu_group"]), int(d["reserved"]), int(d["index"]), int(r["type_id"]),
            bytes(r["key"])[:int(r["key_len"])])


def emit(fmt, kind, recs, cdev=False):
    """The document of VFVGPUCDI_DTYPE records, or None when the kind or a record is outside the domain."""
    kind = kind.encode() if isinstance(kind, str) else kind
    if not kind_ok(kind):
        return None
    devs = []
    for r in recs:
        bdf, group, n, index, tid, key = _fields(r)
        if not P.bdf_ok(bdf) or tid == 0 or not (1 <= int(r["key_len"]) <= 40) or not KEY.fullmatch(key):
            return None
        node = "/dev/vfio/devices/vfio%d" % n if cdev else "/dev/vfio/%d" % group
        ann = {"attach-pci": "true", "bdf": bdf, "cdi.k8s.io/vfio%d" % group: "%s=%d" % (kind.decode(), index),
               "vgpu-type": str(tid), "vgpu-type-key": key.decode()}
        devs.append((str(index), dict(sorted(ann.items())), node))
    k = kind.decode()
    if fmt == FMT_JSON:
        spec = {"cdiVersion": "0.6.0", "kind": k,
                "devices": [{"name": name, "annotations": ann, "containerEdits": {"deviceNodes": [{"path": node}]}}
                            for name, ann, node in devs] or None,
                "containerEdits": {}}
        return json.dumps(spec, indent=2).encode()
    out = ["cdiVersion: 0.6.0", "kind: " + k, "devices:" if devs else "devices: []"]
    for name, ann, node in devs:
        out += ['  - name: "%s"' % name, "    annotations:"]
        for key, v in ann.items():
            quoted = key.startswith("vgpu-type") or key == "attach-pci"
            out.append("      %s: %s" % (key, '"%s"' % v if quoted else P.yaml_scalar(v)))
        out += ["    containerEdits:", "      deviceNodes:", "        - path: " + node]
    return ("\n".join(out) + "\n").encode()


OK, E_INVALID, E_UNSUPPORTED = 0, -1, -7
START = {FMT_YAML: b'\n  - name: "', FMT_JSON: b'\n    {\n      "name": "'}
# index, bdf (YAML: optionally quoted), group, type ID, key (up to 41 bytes, so that a key past 40 reaches the range
# check), then the node: /dev/vfio/<g> or, for the cdev layout, /dev/vfio/devices/vfio<N>
_HEAD = {FMT_YAML: rb'(\d{1,20})"\n    annotations:\n      attach-pci: "true"\n      bdf: ("?)([^"\n]{0,16})\2\n'
                   rb'      cdi\.k8s\.io/vfio(\d{1,10}): [^=\n]*=\d{1,20}\n      vgpu-type: "(\d{1,10})"\n'
                   rb'      vgpu-type-key: "([^"\n]{0,41})"\n    containerEdits:\n      deviceNodes:\n        - path: /dev/vfio/',
         FMT_JSON: rb'(\d{1,20})",\n      "annotations": \{\n        "attach-pci": "true",\n        "bdf": "()([^"]{0,16})",\n'
                   rb'        "cdi\.k8s\.io/vfio(\d{1,10})": "[^=\n]*=\d{1,20}",\n        "vgpu-type": "(\d{1,10})",\n'
                   rb'        "vgpu-type-key": "([^"\n]{0,41})"\n      \},\n      "containerEdits": \{\n        "deviceNodes": \[\n'
                   rb'          \{\n            "path": "/dev/vfio/'}
HEAD = {(fmt, cdev): re.compile(_HEAD[fmt] + (rb"devices/vfio" if cdev else b"") + rb"(\d{1,10})") for fmt in _HEAD
        for cdev in (False, True)}


def parse(fmt, doc, kind, cdev=False):
    """kxpu_cdi_parse_vf_vgpu[_cdev] restated: (status, VFVGPUCDI_DTYPE records).  The group layout's records hold
    vfio_cdev 0; reserved and the key bytes past key_len are 0."""
    from kxpu_b200.binding import CDEV_FIELD, VFVGPUCDI_DTYPE
    kind = kind.encode() if isinstance(kind, str) else kind
    doc = bytes(doc)
    if not kind_ok(kind):
        return E_UNSUPPORTED, None
    starts, at = [], doc.find(START[fmt])
    while at >= 0:
        starts.append(at + len(START[fmt]))
        at = doc.find(START[fmt], at + 1)
    recs = np.zeros(len(starts), VFVGPUCDI_DTYPE)
    for i, p in enumerate(starts):
        m = HEAD[fmt, cdev].match(doc, p)
        if not m or not P.bdf_ok(m.group(3)):
            return E_INVALID, None
        index, group, tid, key, node = int(m.group(1)), int(m.group(4)), int(m.group(5)), m.group(6), int(m.group(7))
        if index >= 1 << 64 or group >= 1 << 32 or tid >= 1 << 32 or node >= 1 << 32 or len(key) > 40:
            return E_INVALID, None
        d = recs[i]["dev"]
        d["bdf"], d["iommu_group"], d[CDEV_FIELD], d["index"] = m.group(3), group, node if cdev else 0, index
        recs[i]["type_id"], recs[i]["key"], recs[i]["key_len"] = tid, key, len(key)
    if emit(fmt, kind, recs, cdev) != doc:
        return E_INVALID, None
    return OK, recs


def annotations(fmt, doc):
    """Each device's annotations, as PyYAML (YAML 1.1 resolution) or json reads them back."""
    spec = yaml.safe_load(doc) if fmt == FMT_YAML else json.loads(doc)
    return [d["annotations"] for d in spec["devices"] or []]


def strip_types(fmt, doc):
    """The document with both vgpu-type lines taken out: kxpu_cdi_emit_kind's (or _cdev's) document of the same records."""
    if fmt == FMT_YAML:
        return re.sub(rb'\n      vgpu-type: "\d+"\n      vgpu-type-key: "[^"\n]*"', b"", doc)
    return re.sub(rb'",\n        "vgpu-type": "\d+",\n        "vgpu-type-key": "[^"\n]*', b"", doc)
