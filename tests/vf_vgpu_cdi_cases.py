"""Inputs of the typed VF-vGPU CDI spec tests (kxpu_cdi_emit_vf_vgpu[_cdev] / kxpu_cdi_parse_vf_vgpu[_cdev]): records with
a vGPU type ID and type key per device, over cdi_parse_cases' bdfs (base-60 quoted and plain), groups and indices."""
import numpy as np

import cdi_parse_cases as CP
from kxpu_b200.binding import CDEV_FIELD, VFVGPUCDI_DTYPE

FMT_YAML, FMT_JSON = CP.FMT_YAML, CP.FMT_JSON
KIND_3 = b"a/b"
KIND_14 = b"nvidia.com/gpu"
KIND_63 = CP.KIND_LONG
KINDS = [KIND_3, KIND_14, KIND_63]
# keys that a YAML 1.1 or 1.2 resolver (or JSON, unquoted) would read as something other than a string
TRICKY_KEYS = [b"true", b"No", b"1_000", b"0x1F", b".inf", b"1e5", b"2024-01-01", b"null", b"0o17", b"-.5", b"y", b"1"]
EDGE_KEYS = [b"A", b"k" * 40, b"NVIDIA_H100-4C", b"a.b-c_d"] + TRICKY_KEYS
EDGE_IDS = [1, (1 << 32) - 1, 557, 10, 9]


def records(n, seed=0):
    """n records: the edge IDs and keys first, then IDs over the whole range and keys of 1..40 bytes of the alphabet;
    cdev numbers of every width."""
    base = CP.records(n, False, seed)
    rng = np.random.default_rng(seed + 2000)
    a = np.zeros(n, VFVGPUCDI_DTYPE)
    a["dev"] = base
    a["dev"][CDEV_FIELD] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    a["type_id"] = rng.integers(1, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    alphabet = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_.-", np.uint8)
    lens = rng.integers(1, 41, n)
    keys = np.zeros((n, 40), np.uint8)
    for i in range(min(n, 4096)):  # beyond that, one pattern per length keeps large cases quick
        keys[i, :lens[i]] = alphabet[rng.integers(0, len(alphabet), lens[i])]
    if n > 4096:
        pat = np.stack([np.pad(alphabet[np.arange(L) % len(alphabet)], (0, 40 - L)) for L in range(1, 41)])
        keys[4096:] = pat[lens[4096:] - 1]
    k = min(n, len(EDGE_KEYS))
    for i in range(k):
        keys[i] = 0
        keys[i, :len(EDGE_KEYS[i])] = np.frombuffer(EDGE_KEYS[i], np.uint8)
        lens[i] = len(EDGE_KEYS[i])
    a["key"] = keys.view("S40").reshape(n)
    a["key_len"] = lens
    a["type_id"][:min(n, len(EDGE_IDS))] = EDGE_IDS[:min(n, len(EDGE_IDS))]
    return a


def group_view(recs):
    """the records as the group layout's parser returns them: no cdev number"""
    out = recs.copy()
    out["dev"][CDEV_FIELD] = 0
    return out


def damaged(fmt, kind, cdev=False, seed=1, flips=120):
    """(name, document) pairs built from a five-device typed document from the C oracle (tests/vf_vgpu_cdi_oracle.c), in
    the shape of cdi_parse_cases.damaged: each is accepted or refused as pyref_vf_vgpu_cdi.parse says."""
    import vf_vgpu_cdi_oracle as VO
    recs = records(5, seed)
    recs["dev"]["index"] = [3, 1, (1 << 64) - 1, 0, 42]
    recs["dev"]["iommu_group"][4] = (1 << 32) - 1
    recs["dev"][CDEV_FIELD] = [7, 0, 12, (1 << 32) - 1, 12]
    recs["type_id"] = [5, 1, (1 << 32) - 1, 10, 9]
    keys = [b"A", b"k" * 40, b"NVIDIA_H100-4C", b"a.b-c_d", b"7"]
    recs["key"], recs["key_len"] = keys, [len(k) for k in keys]
    if not cdev:
        recs = group_view(recs)
    doc = VO.emit(fmt, kind, recs, cdev)
    out = [("clean", doc)]
    rng = np.random.default_rng(seed)
    for k in range(flips):
        b = bytearray(doc)
        p = int(rng.integers(0, len(b)))
        b[p] = (b[p] + int(rng.integers(1, 256))) & 0xFF
        out.append(("flip%d@%d" % (k, p), bytes(b)))
    for b in CP.boundaries(fmt, doc):
        for d in (-1, 0, 1):
            if 0 <= b + d < len(doc):
                out.append(("truncate@%d" % (b + d), doc[:b + d]))
    end = b"\n" if fmt == FMT_YAML else b'"'
    tid = (b'vgpu-type: "%d"' if fmt == FMT_YAML else b'"vgpu-type": "%d"')
    key = (b'vgpu-type-key: "%s"' if fmt == FMT_YAML else b'"vgpu-type-key": "%s"')
    node = b"/dev/vfio/devices/vfio%d" if cdev else b"/dev/vfio/%d"
    out += [("trailing_newline", doc + b"\n"), ("trailing_byte", doc + b"x"), ("crlf", doc.replace(b"\n", b"\r\n")),
            ("index_leading_zero", doc.replace(b'"1"', b'"01"', 1).replace(b"=1" + end, b"=01" + end, 1)),
            ("type_leading_zero", doc.replace(tid % 5, tid.replace(b"%d", b"05") % (), 1)),
            ("index_past_u64", doc.replace(b"18446744073709551615", b"18446744073709551616")),
            ("group_past_u32", doc.replace(b"vfio4294967295" + (b":" if fmt == FMT_YAML else b'"'),
                                           b"vfio4294967296" + (b":" if fmt == FMT_YAML else b'"'))),
            ("type_past_u32", doc.replace(tid % ((1 << 32) - 1), tid % (1 << 32), 1)),
            ("type_zero", doc.replace(tid % 1, tid % 0, 1)),
            ("key_41", doc.replace(key % (b"k" * 40), key % (b"k" * 41), 1)),
            ("key_empty", doc.replace(key % b"A", key % b"", 1)),
            ("key_unquoted", doc.replace(key % b"A", key.replace(b'"', b"") % b"A", 1)),
            ("type_unquoted", doc.replace(tid % 5, tid.replace(b'"%d"', b"%d") % 5, 1)),
            ("name_differs", doc.replace(b"=3" + end, b"=4" + end, 1))]
    if cdev:
        out += [("node_past_u32", doc.replace(node % ((1 << 32) - 1), node % (1 << 32), 1)),
                ("node_leading_zero", doc.replace(node % 7 + end, node.replace(b"%d", b"07") % () + end, 1)),
                ("node_is_group", doc.replace(node % 7 + end, b"/dev/vfio/%d" % recs["dev"]["iommu_group"][0] + end, 1))]
    else:
        out += [("node_is_cdev", doc.replace(node % recs["dev"]["iommu_group"][0] + end, b"/dev/vfio/devices/vfio7" + end, 1))]
    bs = CP.boundaries(fmt, doc)
    out.append(("duplicated_fragment", doc[:bs[1]] + doc[bs[0]:]))
    out.append(("duplicated_last", doc[:bs[-2]] + doc[bs[-2]:bs[-1]] + doc[bs[-2]:]))
    out.append(("empty", b""))
    out.append(("zero_devices", VO.emit(fmt, kind, recs[:0], cdev)))
    missed = [name for name, d in out[1:] if d == doc and not name.startswith(("flip", "truncate"))]
    assert not missed, missed  # every named edit found its target
    return recs, out
