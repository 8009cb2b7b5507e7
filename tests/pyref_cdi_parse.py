"""Plain-Python restatement of kxpu_cdi_parse / kxpu_cdi_parse_mdev: split the document at its device starts, read each
device's fields with a regular expression, and accept the document only if the oracle's emitter (oracle cdi_emit_kind /
cdi_emit_mdev) writes the same bytes from the records read.  parse(...) returns (status, records)."""
import re

import numpy as np

from oracle import mdev_oracle as MO
from oracle import xpu_oracle as XO

OK, E_INVALID, E_UNSUPPORTED = 0, -1, -7
FMT_YAML, FMT_JSON = 0, 1
START = {FMT_YAML: b'\n  - name: "', FMT_JSON: b'\n    {\n      "name": "'}
# index, bdf (YAML: optionally quoted), group; the mdev layout's uuid after its annotation
HEAD = {FMT_YAML: re.compile(rb'(\d{1,20})"\n    annotations:\n      attach-pci: "true"\n      bdf: ("?)([^"\n]{0,16})\2\n'
                             rb'      cdi\.k8s\.io/vfio(\d{1,10}): '),
        FMT_JSON: re.compile(rb'(\d{1,20})",\n      "annotations": \{\n        "attach-pci": "true",\n        "bdf": "()'
                             rb'([^"]{0,16})",\n        "cdi\.k8s\.io/vfio(\d{1,10})": "')}
BDF = re.compile(rb"[0-9a-f:.]{1,16}")
UUID = {FMT_YAML: re.compile(rb'[^=\n]*=\d{1,20}\n      mdev: (.{36})', re.S),
        FMT_JSON: re.compile(rb'[^=\n]*=\d{1,20}",\n        "mdev": "(.{36})', re.S)}


def emit(fmt, kind, recs, mdev):
    return MO.cdi_emit_mdev(fmt, kind, recs) if mdev else XO.cdi_emit_kind(fmt, kind, recs)


def parse(fmt, doc, kind, mdev=False):
    kind = kind.encode() if isinstance(kind, str) else kind
    doc = bytes(doc)
    dtype = MO.MDEVCDI_DTYPE if mdev else XO.CDIDEV_DTYPE
    if emit(fmt, kind, np.zeros(0, dtype), mdev) is None:
        return E_UNSUPPORTED, None
    starts, at = [], doc.find(START[fmt])
    while at >= 0:
        starts.append(at + len(START[fmt]))
        at = doc.find(START[fmt], at + 1)
    recs = np.zeros(len(starts), dtype)
    for i, p in enumerate(starts):
        m = HEAD[fmt].match(doc, p)
        if not m:
            return E_INVALID, None
        index, group = int(m.group(1)), int(m.group(4))
        if index >= 1 << 64 or group >= 1 << 32:
            return E_INVALID, None
        if not BDF.fullmatch(m.group(3)):  # kxpu_cdi_emit_kind refuses such a bdf; the PCI oracle does not check it
            return E_INVALID, None
        if mdev:
            u = UUID[fmt].match(doc, m.end())
            if not u:
                return E_INVALID, None
            recs[i] = (u.group(1), group, m.group(3), index)
        else:
            recs[i]["bdf"], recs[i]["iommu_group"], recs[i]["index"] = m.group(3), group, index
    if emit(fmt, kind, recs, mdev) != doc:
        return E_INVALID, None
    return OK, recs
