"""Plain-Python restatement of kxpu_cdi_emit_mdev_cdev / kxpu_cdi_parse_mdev_cdev: the CDI spec of a vGPU class whose mdevs
are reached through their VFIO cdevs.  emit() is pyref_mdev.cdi_yaml / cdi_json (the vGPU document) with each device's
node /dev/vfio/<g> written as /dev/vfio/devices/vfio<N>.  parse(...) splits the document at its device starts, reads
each device with regular expressions and accepts the document only when emit() writes the same bytes from the records
read; it returns (status, records)."""
import re

import numpy as np

import pyref
import pyref_mdev as PM
from oracle import mdev_oracle as MO
from oracle import xpu_oracle as XO

OK, E_INVALID, E_UNSUPPORTED = 0, -1, -7
FMT_YAML, FMT_JSON = 0, 1
# kxpu_mdevcdev: kxpu_mdevcdi, then N and three reserved words (80 bytes)
MDEVCDEV_DTYPE = np.dtype([("dev", MO.MDEVCDI_DTYPE), ("vfio_cdev", "<u4"), ("reserved", "<u4", (3,))])


def node_path(n):
    return b"/dev/vfio/devices/vfio%d" % n


# the node line of one fragment: pyref_mdev writes /dev/vfio/<g> there, once per device and nowhere else
_NODE = {FMT_YAML: re.compile(rb"(\n        - path: )/dev/vfio/\d+\n"),
         FMT_JSON: re.compile(rb'(\n            "path": ")/dev/vfio/\d+"')}
_NODE_END = {FMT_YAML: b"\n", FMT_JSON: b'"'}


def emit(fmt, kind, recs):
    """The document of MDEVCDEV_DTYPE records, or None when the kind, a uuid or a parent is outside the domain."""
    kind = kind.encode() if isinstance(kind, str) else kind
    if not XO.kind_ok(kind):
        return None
    devs = []
    for r in recs:
        d = r["dev"]
        uuid, parent = bytes(d["uuid"]), bytes(d["parent"])
        if len(uuid) != 36 or not PM.uuid_ok(uuid) or not pyref.bdf_ok(parent):
            return None
        devs.append({"index": int(d["index"]), "parent": parent, "group": int(d["iommu_group"]), "uuid": uuid})
    doc = (PM.cdi_yaml if fmt == FMT_YAML else PM.cdi_json)(kind, devs)
    nodes = iter(int(x) for x in recs["vfio_cdev"])
    out = _NODE[fmt].sub(lambda m: m.group(1) + node_path(next(nodes)) + _NODE_END[fmt], doc)
    assert next(nodes, None) is None
    return out


START = {FMT_YAML: b'\n  - name: "', FMT_JSON: b'\n    {\n      "name": "'}
HEAD = {FMT_YAML: re.compile(rb'(\d{1,20})"\n    annotations:\n      attach-pci: "true"\n      bdf: ("?)([^"\n]{0,16})\2\n'
                             rb'      cdi\.k8s\.io/vfio(\d{1,10}): [^=\n]*=\d{1,20}\n      mdev: (.{36})\n'
                             rb'    containerEdits:\n      deviceNodes:\n        - path: /dev/vfio/devices/vfio(\d{1,10})\n',
                             re.S),
        FMT_JSON: re.compile(rb'(\d{1,20})",\n      "annotations": \{\n        "attach-pci": "true",\n        "bdf": "()'
                             rb'([^"]{0,16})",\n        "cdi\.k8s\.io/vfio(\d{1,10})": "[^=\n]*=\d{1,20}",\n'
                             rb'        "mdev": "(.{36})"\n      \},\n      "containerEdits": \{\n        "deviceNodes": \[\n'
                             rb'          \{\n            "path": "/dev/vfio/devices/vfio(\d{1,10})"', re.S)}


def parse(fmt, doc, kind):
    kind = kind.encode() if isinstance(kind, str) else kind
    doc = bytes(doc)
    if emit(fmt, kind, np.zeros(0, MDEVCDEV_DTYPE)) is None:
        return E_UNSUPPORTED, None
    starts, at = [], doc.find(START[fmt])
    while at >= 0:
        starts.append(at + len(START[fmt]))
        at = doc.find(START[fmt], at + 1)
    recs = np.zeros(len(starts), MDEVCDEV_DTYPE)
    for i, p in enumerate(starts):
        m = HEAD[fmt].match(doc, p)
        if not m or not pyref.bdf_ok(m.group(3)) or not PM.uuid_ok(m.group(5)):  # the emitter refuses these
            return E_INVALID, None
        index, group, node = int(m.group(1)), int(m.group(4)), int(m.group(6))
        if index >= 1 << 64 or group >= 1 << 32 or node >= 1 << 32:
            return E_INVALID, None
        recs[i]["dev"] = (m.group(5), group, m.group(3), index)
        recs[i]["vfio_cdev"] = node
    if emit(fmt, kind, recs) != doc:
        return E_INVALID, None
    return OK, recs
