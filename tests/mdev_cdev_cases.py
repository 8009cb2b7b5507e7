"""Inputs of the vGPU cdev CDI spec tests (kxpu_cdi_emit_mdev_cdev / kxpu_cdi_parse_mdev_cdev): records with cdev
numbers, their documents, and damaged variants of them.

oracle_doc() derives an mdev cdev document from the C oracle's vGPU document (kxo_cdi_emit_mdev): the two layouts differ
only in each device's node path, so it substitutes /dev/vfio/devices/vfio<N> for the device's /dev/vfio/<g>, in device
order.  pyref_mdev_cdev.emit writes the same document from the Python vGPU restatement; the CPU tests hold the two
against each other."""
import re

import numpy as np

import cdi_parse_cases as CP
import pyref_mdev_cdev as PMC
from oracle import mdev_oracle as MO

FMT_YAML, FMT_JSON = CP.FMT_YAML, CP.FMT_JSON
KIND_SHORT, KIND_LONG = CP.KIND_SHORT, CP.KIND_LONG
MDEVCDEV_DTYPE = PMC.MDEVCDEV_DTYPE
EDGE_N = [0, 9, 10, (1 << 32) - 1]  # one and two digits, and the largest cdev number


def records(n, seed=0):
    """cdi_parse_cases.records(mdev=True) with a cdev number per device: the EDGE_N values first, then random uint32s."""
    a = np.zeros(n, MDEVCDEV_DTYPE)
    a["dev"] = CP.records(n, True, seed)
    rng = np.random.default_rng(seed + 1000)
    a["vfio_cdev"] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    k = min(n, len(EDGE_N))
    a["vfio_cdev"][:k] = EDGE_N[:k]
    return a


_PATH = {FMT_YAML: re.compile(rb"(\n        - path: /dev/vfio/)\d+\n"),
         FMT_JSON: re.compile(rb'(\n            "path": "/dev/vfio/)\d+"')}
_END = {FMT_YAML: b"\n", FMT_JSON: b'"'}


def oracle_doc(fmt, kind, recs):
    """The mdev cdev document of recs from the C oracle's vGPU document, or None when the oracle refuses the input."""
    doc = MO.cdi_emit_mdev(fmt, kind, np.ascontiguousarray(recs["dev"]))
    if doc is None:
        return None
    nodes = iter(int(x) for x in recs["vfio_cdev"])
    end = _END[fmt]
    out = _PATH[fmt].sub(lambda m: m.group(1) + b"devices/vfio%d" % next(nodes) + end, doc)
    assert next(nodes, None) is None
    return out


_CDEV_PATH = {FMT_YAML: re.compile(rb"(\n        - path: /dev/vfio/)devices/vfio\d+\n"),
              FMT_JSON: re.compile(rb'(\n            "path": "/dev/vfio/)devices/vfio\d+"')}


def swap_back(fmt, doc, recs):
    """doc with each device's /dev/vfio/devices/vfio<N> written back as its group's /dev/vfio/<g>, in device order."""
    groups = iter(int(x) for x in recs["dev"]["iommu_group"])
    out = _CDEV_PATH[fmt].sub(lambda m: m.group(1) + b"%d" % next(groups) + _END[fmt], doc)
    assert next(groups, None) is None
    return out


def boundaries(fmt, doc):
    return CP.boundaries(fmt, doc)


def damaged(fmt, kind, seed=1, flips=120):
    """(name, document) pairs built from a five-device mdev cdev document: each is accepted or refused as
    pyref_mdev_cdev.parse says."""
    recs = records(5, seed)
    recs["dev"]["index"] = [3, 1, (1 << 64) - 1, 0, 42]
    recs["dev"]["iommu_group"][4] = (1 << 32) - 1
    recs["vfio_cdev"] = [7, 0, 12, (1 << 32) - 1, 12]
    doc = oracle_doc(fmt, kind, recs)
    out = [("clean", doc)]
    rng = np.random.default_rng(seed)
    for k in range(flips):
        b = bytearray(doc)
        p = int(rng.integers(0, len(b)))
        b[p] = (b[p] + int(rng.integers(1, 256))) & 0xFF
        out.append(("flip%d@%d" % (k, p), bytes(b)))
    for b in boundaries(fmt, doc):
        for d in (-1, 0, 1):
            if 0 <= b + d < len(doc):
                out.append(("truncate@%d" % (b + d), doc[:b + d]))
    end = _END[fmt]
    out += [("trailing_newline", doc + b"\n"), ("trailing_byte", doc + b"x"), ("crlf", doc.replace(b"\n", b"\r\n")),
            ("node_leading_zero", doc.replace(b"devices/vfio7" + end, b"devices/vfio07" + end)),
            ("node_past_u32", doc.replace(b"devices/vfio4294967295", b"devices/vfio4294967296")),
            ("node_empty", doc.replace(b"devices/vfio0" + end, b"devices/vfio" + end)),
            ("node_is_group", doc.replace(b"/dev/vfio/devices/vfio12" + end, b"/dev/vfio/12" + end, 1)),
            ("group_past_u32", doc.replace(b"vfio4294967295" + (b":" if fmt == FMT_YAML else b'"'),
                                           b"vfio4294967296" + (b":" if fmt == FMT_YAML else b'"'))),
            ("uuid_upper", doc.replace(recs["dev"]["uuid"][1], recs["dev"]["uuid"][1].upper(), 1)),
            ("iommu_node", doc.replace(b"/dev/vfio/devices/vfio", b"/dev/iommu/devices/vfio", 1))]
    bs = boundaries(fmt, doc)
    out.append(("duplicated_fragment", doc[:bs[1]] + doc[bs[0]:]))
    out.append(("empty", b""))
    out.append(("zero_devices", oracle_doc(fmt, kind, recs[:0])))
    return recs, out
