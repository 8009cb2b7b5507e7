"""Plain-Python restatement of kxpu_cdi_emit_vf_vgpu / kxpu_cdi_emit_vf_vgpu_cdev: the CDI spec of a class that serves
vGPUs on SR-IOV VFs, with each VF's type ID and type key in two more annotations.  The JSON document is json.dumps of
the spec as a dict (indent 2, the layout of Go's MarshalIndent for these values); the YAML one is written line by line
with pyref.yaml_scalar's quoting of the bdf and both new values always double-quoted.  annotations() reads a document
back with PyYAML or json and returns each device's annotations as the loader sees them."""
import json
import re

import yaml

import pyref as P

FMT_YAML, FMT_JSON = 0, 1
KEY = re.compile(rb"[A-Za-z0-9_.-]{1,40}")
BDF = re.compile(rb"[0-9a-f:.]{1,16}")
KIND = re.compile(rb"[A-Za-z][A-Za-z0-9_.-]*[A-Za-z0-9]?/[A-Za-z][A-Za-z0-9_-]*[A-Za-z0-9]?")


def kind_ok(kind):
    if len(kind) > 63 or not KIND.fullmatch(kind):
        return False
    vendor, klass = kind.split(b"/")
    return all(p[:1].isalpha() and p[-1:].isalnum() for p in (vendor, klass))


def _fields(r):
    d = r["dev"]
    return (bytes(d["bdf"]).decode(), int(d["iommu_group"]), int(d["reserved"]), int(d["index"]), int(r["type_id"]),
            bytes(r["key"])[:int(r["key_len"])])


def emit(fmt, kind, recs, cdev=False):
    """The document of VFVGPUCDI_DTYPE records, or None when the kind or a record is outside the domain."""
    kind = kind.encode() if isinstance(kind, str) else kind
    if not kind_ok(kind):
        return None
    devs = []
    for r in recs:
        bdf, group, n, index, tid, key = _fields(r)
        if not BDF.fullmatch(bdf.encode()) or tid == 0 or not (1 <= int(r["key_len"]) <= 40) or not KEY.fullmatch(key):
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


def annotations(fmt, doc):
    """Each device's annotations, as PyYAML (YAML 1.1 resolution) or json reads them back."""
    spec = yaml.safe_load(doc) if fmt == FMT_YAML else json.loads(doc)
    return [d["annotations"] for d in spec["devices"] or []]


def strip_types(fmt, doc):
    """The document with both vgpu-type lines taken out: kxpu_cdi_emit_kind's (or _cdev's) document of the same records."""
    if fmt == FMT_YAML:
        return re.sub(rb'\n      vgpu-type: "\d+"\n      vgpu-type-key: "[^"\n]*"', b"", doc)
    return re.sub(rb'",\n        "vgpu-type": "\d+",\n        "vgpu-type-key": "[^"\n]*', b"", doc)
