"""Inputs of the CDI spec edge tests (tests/test_cdi_edges.py, tests/test_gpu_cdi_edges.py): the six layouts behind one
interface, records of the widest and the narrowest fields, kinds of any length, and documents built so that a fragment
starts, or the document ends, at a chosen byte offset.

Each layout's document comes from a C oracle (oracle/ for the PCI and vGPU layouts, with cdev_cases / mdev_cdev_cases
substituting the cdev node, tests/vf_vgpu_cdi_oracle.c for the typed ones) and from a Python restatement (pyref_xpu,
pyref_cdev, pyref_mdev, pyref_mdev_cdev, pyref_vf_vgpu_cdi).  Records are built the way the layout's parser returns them
(no cdev number in the group-node layouts), so a parse must give them back byte for byte."""
import numpy as np

import cdev_cases as CC
import cdi_parse_cases as CP
import mdev_cdev_cases as MC
import pyref_cdev as PC
import pyref_mdev as PM
import pyref_mdev_cdev as PMC
import pyref_vf_vgpu_cdi as PV
import pyref_xpu as PX
import vf_vgpu_cdi_oracle as VO
from kxpu_b200.binding import CDEV_FIELD, CDIDEV_DTYPE, MDEVCDEV_DTYPE, MDEVCDI_DTYPE, VFVGPUCDI_DTYPE
from oracle import mdev_oracle as MO
from oracle import xpu_oracle as XO

FMT_YAML, FMT_JSON = CP.FMT_YAML, CP.FMT_JSON
FMTS = [FMT_YAML, FMT_JSON]
LAYOUTS = ["pci", "cdev", "mdev", "mdev_cdev", "typed", "typed_cdev"]
CDEV = {"pci": False, "cdev": True, "mdev": False, "mdev_cdev": True, "typed": False, "typed_cdev": True}
MDEV = {"pci": False, "cdev": False, "mdev": True, "mdev_cdev": True, "typed": False, "typed_cdev": False}
TYPED = {"pci": False, "cdev": False, "mdev": False, "mdev_cdev": False, "typed": True, "typed_cdev": True}
DTYPE = {"pci": CDIDEV_DTYPE, "cdev": CDIDEV_DTYPE, "mdev": MDEVCDI_DTYPE, "mdev_cdev": MDEVCDEV_DTYPE,
         "typed": VFVGPUCDI_DTYPE, "typed_cdev": VFVGPUCDI_DTYPE}
# the emit entry points of the C ABI, and the binding's parse_raw switches
EMIT_FN = {"pci": "kxpu_cdi_emit_kind", "cdev": "kxpu_cdi_emit_cdev", "mdev": "kxpu_cdi_emit_mdev",
           "mdev_cdev": "kxpu_cdi_emit_mdev_cdev", "typed": "kxpu_cdi_emit_vf_vgpu", "typed_cdev": "kxpu_cdi_emit_vf_vgpu_cdev"}
PARSE_HOW = {"pci": {}, "cdev": dict(cdev=True), "mdev": dict(mdev=True), "mdev_cdev": dict(mdev=True, cdev=True),
             "typed": dict(typed=True), "typed_cdev": dict(typed=True, cdev=True)}

WIDE_BDF = b"0000:01:02.34567"  # 16 bytes, base 60: double-quoted in YAML, so 18 bytes there
NARROW_BDF = b"a"                # one byte, plain
U64_MAX, U32_MAX = (1 << 64) - 1, (1 << 32) - 1
KEY40 = b"K" * 40


def kind_of(length):
    """A kind of `length` bytes (3..63) in kxpu_cdi_emit_kind's domain."""
    assert 3 <= length <= 63
    return b"v" * (length - 2) + b"/c"


def uuid_of(k):
    return b"%08x-%04x-4%03x-8%03x-%012x" % (k & 0xFFFFFFFF, k & 0xFFFF, k & 0xFFF, (k * 7) & 0xFFF, (k * 0x9E3779B1) & 0xFFFFFFFFFFFF)


def make(layout, bdf, group, index, node=0, type_id=1, key=b"k"):
    """Records of `layout` from per-device fields (arrays or scalars broadcast to len(index)); node is N (written 0 in
    the group-node layouts, as their parsers return it), type_id and key are read by the typed layouts only."""
    index = np.asarray(index, np.uint64)
    n = len(index)
    bc = lambda v, dt: np.broadcast_to(np.asarray(v, dt), (n,))  # noqa: E731
    bdf, group = bc(bdf, "S16"), bc(group, np.uint32)
    node = bc(node if CDEV[layout] else 0, np.uint32)
    a = np.zeros(n, DTYPE[layout])
    if MDEV[layout]:
        d = a["dev"] if layout == "mdev_cdev" else a
        d["uuid"] = [uuid_of(k) for k in range(n)]
        d["parent"], d["iommu_group"], d["index"] = bdf, group, index
        if layout == "mdev_cdev":
            a["vfio_cdev"] = node
        return a
    d = a["dev"] if TYPED[layout] else a
    d["bdf"], d["iommu_group"], d["index"], d[CDEV_FIELD] = bdf, group, index, node
    if TYPED[layout]:
        key = bc(key, "S40")
        a["type_id"], a["key"], a["key_len"] = bc(type_id, np.uint32), key, [len(k) for k in key]
    return a


def widest(layout, n):
    """n records whose every field is at its longest."""
    return make(layout, WIDE_BDF, U32_MAX, np.full(n, U64_MAX, np.uint64), U32_MAX, U32_MAX, KEY40)


def narrowest(layout, n):
    return make(layout, NARROW_BDF, np.arange(n) % 10, np.arange(n) % 10, np.arange(n) % 10, np.arange(n) % 9 + 1, b"k")


def shrunk(layout, cut):
    """One widest record made `cut` bytes shorter in either format (0 <= cut <= 39): the name (written twice) loses
    cut // 2 digits and the bdf cut % 2 bytes (still base 60, so still quoted in YAML)."""
    return make(layout, WIDE_BDF[:16 - cut % 2], U32_MAX, [10 ** (19 - cut // 2)], U32_MAX, U32_MAX, KEY40)


def mixed(layout, n, seed):
    """n records that mix the widest and the narrowest field of every kind, and widths in between."""
    rng = np.random.default_rng(seed)
    pick = lambda lo, hi: np.where(rng.random(n) < 0.5, lo, hi)  # noqa: E731
    digits = lambda top: np.array([int(rng.integers(0, 1 << 62)) % 10 ** int(d) for d in rng.integers(1, top + 1, n)],  # noqa: E731
                                  np.uint64)
    bdf = np.where(rng.random(n) < 0.35, WIDE_BDF, np.where(rng.random(n) < 0.5, NARROW_BDF, b"0000:c1:00.0")).astype("S16")
    index = pick(np.uint64(U64_MAX), digits(19))
    group = pick(U32_MAX, digits(9).astype(np.uint32))
    node = pick(U32_MAX, digits(9).astype(np.uint32))
    tid = np.maximum(pick(U32_MAX, digits(9).astype(np.uint32)), 1)
    keys = [KEY40[:int(k)] for k in pick(40, rng.integers(1, 40, n))]
    return make(layout, bdf, group, index, node, tid, keys)


def oracle_doc(layout, fmt, kind, recs):
    """The C oracle's document (None: a record outside the domain the oracle checks)."""
    recs = np.ascontiguousarray(recs)
    if layout == "pci":
        return XO.cdi_emit_kind(fmt, kind, recs)
    if layout == "cdev":
        return CC.oracle_doc(fmt, kind, recs)
    if layout == "mdev":
        return MO.cdi_emit_mdev(fmt, kind, recs)
    if layout == "mdev_cdev":
        return MC.oracle_doc(fmt, kind, recs)
    return VO.emit(fmt, kind, recs, CDEV[layout])


def pyref_doc(layout, fmt, kind, recs):
    """The Python restatement's document (None outside the domain)."""
    if layout == "pci":
        devs = [(bytes(r["bdf"]).decode("latin-1"), int(r["iommu_group"]), int(r["index"])) for r in recs]
        return (PX.cdi_yaml if fmt == FMT_YAML else PX.cdi_json)(devs, kind.decode())
    if layout == "cdev":
        return PC.emit(fmt, kind, recs)
    if layout == "mdev":
        devs = [{"index": int(r["index"]), "parent": bytes(r["parent"]), "group": int(r["iommu_group"]),
                 "uuid": bytes(r["uuid"])} for r in recs]
        return (PM.cdi_yaml if fmt == FMT_YAML else PM.cdi_json)(kind, devs)
    if layout == "mdev_cdev":
        return PMC.emit(fmt, kind, recs)
    return PV.emit(fmt, kind, recs, CDEV[layout])


def gpu_emit(kx, layout, fmt, kind, recs):
    if layout == "pci":
        return kx.cdi_emit(fmt, recs, kind)
    if layout == "cdev":
        return kx.cdi_emit_cdev(fmt, recs, kind)
    if layout == "mdev":
        return kx.cdi_emit_mdev(fmt, recs, kind)
    if layout == "mdev_cdev":
        return kx.cdi_emit_mdev_cdev(fmt, recs, kind)
    return kx.cdi_emit_vf_vgpu(fmt, recs, kind, cdev=CDEV[layout])


def starts(fmt, doc):
    """Offsets where a device fragment begins."""
    return CP.boundaries(fmt, doc)[:-1]


def tail_len(fmt):
    return len(b'  ],\n  "containerEdits": {}\n}') if fmt == FMT_JSON else 0


def fragments(fmt, doc):
    """The length of every device fragment, as the emitter sizes it: from its start to the next one, the last to the
    document's tail (JSON: the separator after a device is part of its fragment)."""
    s = starts(fmt, doc)
    return [b - a for a, b in zip(s, s[1:] + [len(doc) - tail_len(fmt)])]


def head_len(layout, fmt, kind):
    return starts(fmt, oracle_doc(layout, fmt, kind, widest(layout, 1)))[0]


def width(layout, fmt, kind):
    """The widest fragment of a device that is not the last."""
    return fragments(fmt, oracle_doc(layout, fmt, kind, widest(layout, 2)))[0]


def _shims(layout, fmt, kind, span):
    """Records whose fragments (none of them the last) add up to exactly `span` bytes, each one a shrunk widest."""
    w = width(layout, fmt, kind)
    k = -(-span // w)
    deficit = k * w - span
    cuts = [deficit // k + (1 if i < deficit % k else 0) for i in range(k)]
    assert max(cuts, default=0) <= 39, (span, w, k)
    return np.concatenate([shrunk(layout, c) for c in cuts]) if k else widest(layout, 0)


def start_at(layout, fmt, kind, offset, after=2):
    """A document in which a widest fragment starts at byte `offset` (followed by `after` more widest devices); returns
    (records, document, index of that device)."""
    pre = _shims(layout, fmt, kind, offset - head_len(layout, fmt, kind))
    recs = np.concatenate([pre, widest(layout, 1 + after)])
    doc = oracle_doc(layout, fmt, kind, recs)
    assert starts(fmt, doc)[len(pre)] == offset
    return recs, doc, len(pre)


def end_at(layout, fmt, kind, length):
    """A document of exactly `length` bytes whose last device is a widest one."""
    last = width(layout, fmt, kind) - (1 if fmt == FMT_JSON else 0)
    pre = _shims(layout, fmt, kind, length - head_len(layout, fmt, kind) - last - tail_len(fmt))
    recs = np.concatenate([pre, widest(layout, 1)])
    doc = oracle_doc(layout, fmt, kind, recs)
    assert len(doc) == length
    return recs, doc


def sweep(layout, fmt, kind):
    """One document whose widest fragments start at every offset of a tile: devices of fragment lengths w, w - 1
    alternating (w even) or all w (w odd), so that the widest starts advance by an odd step, 8193 times.  Returns
    (records, document)."""
    w = width(layout, fmt, kind)
    pair = widest(layout, 1) if w % 2 else np.concatenate([widest(layout, 1), shrunk(layout, 1)])
    recs = np.tile(pair, 8193)
    return recs, oracle_doc(layout, fmt, kind, recs)
