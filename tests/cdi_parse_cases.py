"""Inputs of the CDI spec parse tests (kxpu_cdi_parse / kxpu_cdi_parse_mdev): records, their documents from the oracle
emitter, and damaged variants of them."""
import numpy as np

from oracle import mdev_oracle as MO
from oracle import xpu_oracle as XO

FMT_YAML, FMT_JSON = 0, 1
KIND_SHORT = b"nvidia.com/gpu"
KIND_LONG = b"v" * 40 + b".example/" + b"c" * 14  # 63 bytes
assert len(KIND_LONG) == 63


def records(n, mdev=False, seed=0):
    """n records: bdfs that yaml.v3 quotes (bus 01: base 60) and that it does not (bus c1), groups over the whole uint32
    range, distinct indices over the whole uint64 range in shuffled order."""
    rng = np.random.default_rng(seed)
    buses = rng.choice(np.array([0x01, 0x21, 0x3b, 0xc1, 0xe3], np.uint32), n)
    bdf = np.array([b"0000:%02x:%02x.%d" % (b, k & 0x1F, k % 8) for k, b in zip(range(n), buses)], dtype="S16")
    group = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    index = np.unique(rng.integers(0, np.iinfo(np.uint64).max, n + 16, dtype=np.uint64, endpoint=True))[:n]
    index[: min(n, 3)] = [0, 9, 10][: min(n, 3)]  # one-digit and two-digit names too
    rng.shuffle(index)
    if mdev:
        a = np.zeros(n, MO.MDEVCDI_DTYPE)
        a["uuid"] = np.array([b"%08x-%04x-4%03x-8%03x-%012x" % (k, k & 0xFFFF, k & 0xFFF, (k * 7) & 0xFFF, (k * 0x9E3779B1) & 0xFFFFFFFFFFFF)
                              for k in range(n)], dtype="S36")
        a["parent"], a["iommu_group"], a["index"] = bdf, group, index
    else:
        a = np.zeros(n, XO.CDIDEV_DTYPE)
        a["bdf"], a["iommu_group"], a["index"] = bdf, group, index
    return a


def emit(fmt, kind, recs, mdev=False):
    return MO.cdi_emit_mdev(fmt, kind, recs) if mdev else XO.cdi_emit_kind(fmt, kind, recs)


START = {FMT_YAML: b'\n  - name: "', FMT_JSON: b'\n    {\n      "name": "'}


def boundaries(fmt, doc):
    """Offsets where a device fragment begins, plus the document's end."""
    out, at = [], doc.find(START[fmt])
    while at >= 0:
        out.append(at + 1)
        at = doc.find(START[fmt], at + 1)
    return out + [len(doc)]


def damaged(fmt, kind, mdev, seed=1, flips=120):
    """(name, document) pairs built from a five-device document: each is accepted or refused as pyref_cdi_parse says."""
    recs = records(5, mdev, seed)
    recs["index"] = [3, 1, (1 << 64) - 1, 0, 42]
    recs["iommu_group"][4] = (1 << 32) - 1
    doc = emit(fmt, kind, recs, mdev)
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
    out += [("trailing_newline", doc + b"\n"), ("trailing_byte", doc + b"x"), ("crlf", doc.replace(b"\n", b"\r\n")),
            ("leading_zero", doc.replace(b'"1"', b'"01"', 1).replace(b"=1" + (b"\n" if fmt == FMT_YAML else b'"'),
                                                                     b"=01" + (b"\n" if fmt == FMT_YAML else b'"'), 1)),
            ("index_past_u64", doc.replace(b"18446744073709551615", b"18446744073709551616")),
            ("group_past_u32", doc.replace(b"4294967295", b"4294967296")),
            ("name_differs", doc.replace(b"=3" + (b"\n" if fmt == FMT_YAML else b'"'),
                                         b"=4" + (b"\n" if fmt == FMT_YAML else b'"'), 1))]
    bs = boundaries(fmt, doc)
    out.append(("duplicated_fragment", doc[:bs[1]] + doc[bs[0]:]))
    out.append(("duplicated_last", doc[:bs[-2]] + doc[bs[-2]:bs[-1]] + doc[bs[-2]:]))
    out.append(("empty", b""))
    out.append(("zero_devices", emit(fmt, kind, recs[:0], mdev)))
    return recs, out
