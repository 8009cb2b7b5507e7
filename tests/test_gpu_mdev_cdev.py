"""GPU checks of the vGPU cdev CDI spec: kxpu_cdi_emit_mdev_cdev is bit-exact against the oracle-derived document and the
Python restatement (both formats, a short and a 63-byte kind, up to 2^20 vGPUs), and kxpu_cdi_emit_mdev of the same
records is that document with the node paths swapped back; kxpu_cdi_parse_mdev_cdev round-trips those documents at every
16-byte host-buffer phase, gives pyref_mdev_cdev's verdict on damaged documents, and the four layouts refuse each other's
documents; the NOSPACE protocol, the sizing call, KXPU_T_EMIT and the refusals."""
import ctypes as C

import numpy as np
import pytest

import mdev_cdev_cases as K
import pyref_mdev_cdev as PMC
from kxpu_b200 import binding as B

pytestmark = pytest.mark.gpu

CASES = [(fmt, kind) for fmt in (K.FMT_YAML, K.FMT_JSON) for kind in (K.KIND_SHORT, K.KIND_LONG)]
SIZES = [0, 1, 127, 128, 129, 65536, 1 << 20]


def dev(recs):
    return np.ascontiguousarray(recs["dev"])


@pytest.mark.parametrize("fmt,kind", CASES)
@pytest.mark.parametrize("n", SIZES)
def test_emit_bit_exact(kx, fmt, kind, n):
    recs = K.records(n, seed=n + 11)
    want = K.oracle_doc(fmt, kind, recs)
    got = kx.cdi_emit_mdev_cdev(fmt, recs, kind)
    assert got == want
    # the group layout of the same records: the document with each node written back as /dev/vfio/<g>
    assert kx.cdi_emit_mdev(fmt, dev(recs), kind) == K.swap_back(fmt, got, recs)
    if n <= 65536:  # the independent restatement too (the oracle-derived document is checked against it on the CPU)
        assert got == PMC.emit(fmt, kind, recs)


@pytest.mark.parametrize("fmt,kind", CASES)
@pytest.mark.parametrize("n", SIZES)
def test_parse_round_trip(kx, fmt, kind, n):
    recs = K.records(n, seed=n + 7)
    doc = K.oracle_doc(fmt, kind, recs)
    got = kx.cdi_parse_mdev_cdev(fmt, doc, kind)
    assert len(got) == n
    assert got.tobytes() == recs.tobytes()
    if n <= 129:  # the host buffer at every 16-byte phase
        for off in range(16):
            rc, m, out = kx.cdi_parse_raw(fmt, doc, kind, n, offset=off, mdev=True, cdev=True)
            assert (rc, m) == (B.KXPU_OK, n), off
            assert out.tobytes() == recs.tobytes(), off


def test_sizing_call_and_timing(kx):
    recs = K.records(1000, seed=4)
    need = C.c_size_t(0)
    rc = kx.L.kxpu_cdi_emit_mdev_cdev(kx.ctx, K.FMT_JSON, K.KIND_SHORT, recs.ctypes.data, len(recs), None, 0, C.byref(need))
    doc = K.oracle_doc(K.FMT_JSON, K.KIND_SHORT, recs)
    assert (rc, need.value) == (B.E_NOSPACE, len(doc))
    out = np.zeros(len(doc) - 1, np.uint8)
    rc = kx.L.kxpu_cdi_emit_mdev_cdev(kx.ctx, K.FMT_JSON, K.KIND_SHORT, recs.ctypes.data, len(recs), out.ctypes.data,
                                      len(out), C.byref(need))
    assert (rc, need.value) == (B.E_NOSPACE, len(doc))
    assert kx.cdi_emit_mdev_cdev(K.FMT_JSON, recs, K.KIND_SHORT) == doc
    assert kx.timings()[B.T_EMIT] > 0
    kx.cdi_parse_mdev_cdev(K.FMT_JSON, doc, K.KIND_SHORT)
    assert kx.timings()[B.T_EMIT] > 0


def test_emit_refusals(kx):
    recs = K.records(3)
    size = C.byref(C.c_size_t())
    rc = kx.L.kxpu_cdi_emit_mdev_cdev(kx.ctx, K.FMT_YAML, b"no-slash", recs.ctypes.data, 3, None, 0, size)
    assert rc == B.E_UNSUPPORTED
    bad = recs.copy()
    bad["dev"]["uuid"][1] = bad["dev"]["uuid"][1].upper()  # not the canonical lowercase form
    rc = kx.L.kxpu_cdi_emit_mdev_cdev(kx.ctx, K.FMT_YAML, K.KIND_SHORT, bad.ctypes.data, 3, None, 0, size)
    assert rc == B.E_UNSUPPORTED
    bad = recs.copy()
    bad["dev"]["parent"][2] = b"0000:C1:00.0"  # outside [0-9a-f:.]
    rc = kx.L.kxpu_cdi_emit_mdev_cdev(kx.ctx, K.FMT_JSON, K.KIND_SHORT, bad.ctypes.data, 3, None, 0, size)
    assert rc == B.E_UNSUPPORTED
    rc = kx.L.kxpu_cdi_emit_mdev_cdev(kx.ctx, 2, K.KIND_SHORT, recs.ctypes.data, 3, None, 0, size)
    assert rc == B.E_INVALID


@pytest.mark.parametrize("fmt,kind", CASES)
def test_damaged_documents(kx, fmt, kind):
    _, docs = K.damaged(fmt, kind)
    for name, doc in docs:
        st, want = PMC.parse(fmt, doc, kind)
        rc, n, out = kx.cdi_parse_raw(fmt, doc, kind, 8, offset=3, mdev=True, cdev=True)
        assert rc == st, name
        if st == PMC.OK:
            assert n == len(want) and out[:n].tobytes() == want.tobytes(), name
        else:
            assert n == -1, name  # *n untouched
    doc = docs[0][1]
    assert kx.cdi_parse_raw(fmt, doc, b"example.com/other", 8, mdev=True, cdev=True)[0] == B.E_INVALID
    assert kx.cdi_parse_raw(fmt, doc, b"no-slash", 8, mdev=True, cdev=True)[0] == B.E_UNSUPPORTED
    assert kx.cdi_parse_raw(1 - fmt, doc, kind, 8, mdev=True, cdev=True)[0] == B.E_INVALID


@pytest.mark.parametrize("fmt", [K.FMT_YAML, K.FMT_JSON])
def test_layouts_refuse_each_other(kx, fmt):
    """Each of the four layouts' documents parses with its own call only; the zero-device document with all four."""
    recs = K.records(300, seed=8)
    pci = np.zeros(300, B.CDIDEV_DTYPE)
    pci["bdf"], pci["iommu_group"], pci["index"] = recs["dev"]["parent"], recs["dev"]["iommu_group"], recs["dev"]["index"]
    pci[B.CDEV_FIELD] = recs["vfio_cdev"]
    docs = {"pci": kx.cdi_emit(fmt, pci, K.KIND_SHORT), "cdev": kx.cdi_emit_cdev(fmt, pci, K.KIND_SHORT),
            "mdev": kx.cdi_emit_mdev(fmt, dev(recs), K.KIND_SHORT), "mdev_cdev": K.oracle_doc(fmt, K.KIND_SHORT, recs)}
    flags = {"pci": {}, "cdev": {"cdev": True}, "mdev": {"mdev": True}, "mdev_cdev": {"mdev": True, "cdev": True}}
    for dl, doc in docs.items():
        for pl, kw in flags.items():
            rc, n, _ = kx.cdi_parse_raw(fmt, doc, K.KIND_SHORT, 300, **kw)
            assert (rc, n) == ((B.KXPU_OK, 300) if dl == pl else (B.E_INVALID, -1)), (dl, pl)
    zero = K.oracle_doc(fmt, K.KIND_SHORT, recs[:0])
    assert zero == kx.cdi_emit_mdev_cdev(fmt, recs[:0], K.KIND_SHORT) == kx.cdi_emit_mdev(fmt, dev(recs[:0]), K.KIND_SHORT)
    for kw in flags.values():
        assert kx.cdi_parse_raw(fmt, zero, K.KIND_SHORT, 0, **kw)[:2] == (B.KXPU_OK, 0)


def test_nospace_protocol(kx):
    recs = K.records(200, seed=3)
    doc = K.oracle_doc(K.FMT_JSON, K.KIND_SHORT, recs)
    rc, n, _ = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 0, mdev=True, cdev=True)  # out = NULL: the sizing call
    assert (rc, n) == (B.E_NOSPACE, 200)
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 199, mdev=True, cdev=True)
    assert (rc, n) == (B.E_NOSPACE, 200) and not out.tobytes().strip(b"\0")  # nothing written
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 200, mdev=True, cdev=True)
    assert (rc, n) == (B.KXPU_OK, 200) and out.tobytes() == recs.tobytes()
    assert len(doc) // B.CDI_FRAG_MIN >= 200
