"""Plain-Python restatement of kxpu_cdi_emit_cdev / kxpu_cdi_parse_cdev: the CDI spec of a passthrough class whose
functions are reached through their VFIO cdevs.  It is generateCDISpec + CdiSpec.Save (written as pyref.cdi_yaml /
cdi_json are, with the kind as an argument) with the device node /dev/vfio/devices/vfio<N>.  parse(...) splits the
document at its device starts, reads each device with a regular expression and accepts the document only when emit()
writes the same bytes from the records read; it returns (status, records)."""
import json
import re

import numpy as np

import pyref
from oracle import xpu_oracle as XO

OK, E_INVALID, E_UNSUPPORTED = 0, -1, -7
FMT_YAML, FMT_JSON = 0, 1
CDEV_FIELD = "reserved"  # kxpu_cdidev.vfio_cdev in the numpy dtype (binding.CDEV_FIELD)


def node_path(n):
    return "/dev/vfio/devices/vfio%d" % n


def _bdf_yaml(bdf):
    return '"%s"' % bdf if pyref.BASE60.match(bdf) else bdf


def emit(fmt, kind, recs):
    """The document of CDIDEV_DTYPE records (N in CDEV_FIELD), or None when the kind or a bdf is outside the supported
    domain."""
    kind = kind.decode() if isinstance(kind, bytes) else kind
    if not XO.kind_ok(kind.encode()):
        return None
    devs = [(r["bdf"].decode("latin-1"), int(r["iommu_group"]), int(r["index"]), int(r[CDEV_FIELD])) for r in recs]
    if not all(pyref.bdf_ok(d[0]) for d in devs):
        return None
    if fmt == FMT_YAML:
        out = ["cdiVersion: 0.6.0", "kind: %s" % kind]
        if not devs:
            return ("\n".join(out) + "\ndevices: []\n").encode()
        out.append("devices:")
        for bdf, group, index, node in devs:
            out += ['  - name: "%d"' % index,
                    "    annotations:",
                    '      attach-pci: "true"',
                    "      bdf: %s" % _bdf_yaml(bdf),
                    "      cdi.k8s.io/vfio%d: %s=%d" % (group, kind, index),
                    "    containerEdits:",
                    "      deviceNodes:",
                    "        - path: %s" % node_path(node)]
        return ("\n".join(out) + "\n").encode()
    spec = {"cdiVersion": "0.6.0", "kind": kind}
    spec["devices"] = [
        {"name": str(index),
         "annotations": {"attach-pci": "true", "bdf": bdf, "cdi.k8s.io/vfio%d" % group: "%s=%d" % (kind, index)},
         "containerEdits": {"deviceNodes": [{"path": node_path(node)}]}}
        for bdf, group, index, node in devs] or None
    spec["containerEdits"] = {}
    return json.dumps(spec, indent=2).encode()


START = {FMT_YAML: b'\n  - name: "', FMT_JSON: b'\n    {\n      "name": "'}
HEAD = {FMT_YAML: re.compile(rb'(\d{1,20})"\n    annotations:\n      attach-pci: "true"\n      bdf: ("?)([^"\n]{0,16})\2\n'
                             rb'      cdi\.k8s\.io/vfio(\d{1,10}): [^=\n]*=\d{1,20}\n    containerEdits:\n'
                             rb'      deviceNodes:\n        - path: /dev/vfio/devices/vfio(\d{1,10})\n'),
        FMT_JSON: re.compile(rb'(\d{1,20})",\n      "annotations": \{\n        "attach-pci": "true",\n        "bdf": "()'
                             rb'([^"]{0,16})",\n        "cdi\.k8s\.io/vfio(\d{1,10})": "[^=\n]*=\d{1,20}"\n      \},\n'
                             rb'      "containerEdits": \{\n        "deviceNodes": \[\n          \{\n'
                             rb'            "path": "/dev/vfio/devices/vfio(\d{1,10})"')}


def parse(fmt, doc, kind):
    kind = kind.encode() if isinstance(kind, str) else kind
    doc = bytes(doc)
    if emit(fmt, kind, np.zeros(0, XO.CDIDEV_DTYPE)) is None:
        return E_UNSUPPORTED, None
    starts, at = [], doc.find(START[fmt])
    while at >= 0:
        starts.append(at + len(START[fmt]))
        at = doc.find(START[fmt], at + 1)
    recs = np.zeros(len(starts), XO.CDIDEV_DTYPE)
    for i, p in enumerate(starts):
        m = HEAD[fmt].match(doc, p)
        if not m or not pyref.bdf_ok(m.group(3)):  # kxpu_cdi_emit_cdev refuses such a bdf
            return E_INVALID, None
        index, group, node = int(m.group(1)), int(m.group(4)), int(m.group(5))
        if index >= 1 << 64 or group >= 1 << 32 or node >= 1 << 32:
            return E_INVALID, None
        recs[i]["bdf"], recs[i]["iommu_group"], recs[i]["index"], recs[i][CDEV_FIELD] = m.group(3), group, index, node
    if emit(fmt, kind, recs) != doc:
        return E_INVALID, None
    return OK, recs
