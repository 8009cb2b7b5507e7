"""GPU checks of the VFIO cdev CDI spec (ABI v14): kxpu_cdi_emit_cdev is bit-exact against the oracle-derived document
and the Python restatement (both formats, a short and a 63-byte kind, up to 2^20 devices), with the sizing call and
KXPU_T_EMIT; kxpu_cdi_parse_cdev round-trips those documents at every 16-byte host-buffer phase, gives pyref_cdev's
verdict on damaged documents, refuses group-layout documents (and kxpu_cdi_parse refuses cdev ones) and follows the
NOSPACE protocol."""
import ctypes as C

import numpy as np
import pytest

import cdev_cases as K
import pyref_cdev as PC
from kxpu_b200 import binding as B

pytestmark = pytest.mark.gpu

CASES = [(fmt, kind) for fmt in (K.FMT_YAML, K.FMT_JSON) for kind in (K.KIND_SHORT, K.KIND_LONG)]
SIZES = [0, 1, 127, 128, 129, 65536, 1 << 20]


@pytest.mark.parametrize("fmt,kind", CASES)
@pytest.mark.parametrize("n", SIZES)
def test_emit_bit_exact(kx, fmt, kind, n):
    recs = K.records(n, seed=n + 11)
    want = K.oracle_doc(fmt, kind, recs)
    got = kx.cdi_emit_cdev(fmt, recs, kind)
    assert got == want
    if n <= 65536:  # the independent restatement too (the oracle-derived document is checked against it on the CPU)
        assert got == PC.emit(fmt, kind, recs)
        zeroed = recs.copy()
        zeroed[K.CDEV_FIELD] = 0
        assert kx.cdi_emit(fmt, recs, kind) == kx.cdi_emit(fmt, zeroed, kind)  # the group layout ignores vfio_cdev


@pytest.mark.parametrize("fmt,kind", CASES)
@pytest.mark.parametrize("n", SIZES)
def test_parse_round_trip(kx, fmt, kind, n):
    recs = K.records(n, seed=n + 7)
    doc = K.oracle_doc(fmt, kind, recs)
    got = kx.cdi_parse_cdev(fmt, doc, kind)
    assert len(got) == n
    assert got.tobytes() == recs.tobytes()
    if n <= 129:  # the host buffer at every 16-byte phase
        for off in range(16):
            rc, m, out = kx.cdi_parse_raw(fmt, doc, kind, n, offset=off, cdev=True)
            assert (rc, m) == (B.KXPU_OK, n), off
            assert out.tobytes() == recs.tobytes(), off


def test_sizing_call_and_timing(kx):
    recs = K.records(1000, seed=4)
    need = C.c_size_t(0)
    rc = kx.L.kxpu_cdi_emit_cdev(kx.ctx, K.FMT_JSON, K.KIND_SHORT, recs.ctypes.data, len(recs), None, 0, C.byref(need))
    doc = K.oracle_doc(K.FMT_JSON, K.KIND_SHORT, recs)
    assert (rc, need.value) == (B.E_NOSPACE, len(doc))
    out = np.zeros(len(doc) - 1, np.uint8)
    rc = kx.L.kxpu_cdi_emit_cdev(kx.ctx, K.FMT_JSON, K.KIND_SHORT, recs.ctypes.data, len(recs), out.ctypes.data,
                                 len(out), C.byref(need))
    assert (rc, need.value) == (B.E_NOSPACE, len(doc))
    assert kx.cdi_emit_cdev(K.FMT_JSON, recs, K.KIND_SHORT) == doc
    assert kx.timings()[B.T_EMIT] > 0
    kx.cdi_parse_cdev(K.FMT_JSON, doc, K.KIND_SHORT)
    assert kx.timings()[B.T_EMIT] > 0


def test_emit_refusals(kx):
    recs = K.records(3)
    rc = kx.L.kxpu_cdi_emit_cdev(kx.ctx, K.FMT_YAML, b"no-slash", recs.ctypes.data, 3, None, 0, C.byref(C.c_size_t()))
    assert rc == B.E_UNSUPPORTED
    bad = recs.copy()
    bad["bdf"][1] = b"0000:C1:00.0"  # outside [0-9a-f:.]
    rc = kx.L.kxpu_cdi_emit_cdev(kx.ctx, K.FMT_YAML, K.KIND_SHORT, bad.ctypes.data, 3, None, 0, C.byref(C.c_size_t()))
    assert rc == B.E_UNSUPPORTED
    rc = kx.L.kxpu_cdi_emit_cdev(kx.ctx, 2, K.KIND_SHORT, recs.ctypes.data, 3, None, 0, C.byref(C.c_size_t()))
    assert rc == B.E_INVALID


@pytest.mark.parametrize("fmt,kind", CASES)
def test_damaged_documents(kx, fmt, kind):
    _, docs = K.damaged(fmt, kind)
    for name, doc in docs:
        st, want = PC.parse(fmt, doc, kind)
        rc, n, out = kx.cdi_parse_raw(fmt, doc, kind, 8, offset=3, cdev=True)
        assert rc == st, name
        if st == PC.OK:
            assert n == len(want) and out[:n].tobytes() == want.tobytes(), name
        else:
            assert n == -1, name  # *n untouched
    doc = docs[0][1]
    assert kx.cdi_parse_raw(fmt, doc, b"example.com/other", 8, cdev=True)[0] == B.E_INVALID
    assert kx.cdi_parse_raw(fmt, doc, b"no-slash", 8, cdev=True)[0] == B.E_UNSUPPORTED
    assert kx.cdi_parse_raw(1 - fmt, doc, kind, 8, cdev=True)[0] == B.E_INVALID


@pytest.mark.parametrize("fmt", [K.FMT_YAML, K.FMT_JSON])
def test_layouts_refuse_each_other(kx, fmt):
    recs = K.records(300, seed=8)
    cdev_doc = K.oracle_doc(fmt, K.KIND_SHORT, recs)
    group_doc = kx.cdi_emit(fmt, recs, K.KIND_SHORT)
    assert kx.cdi_parse_raw(fmt, group_doc, K.KIND_SHORT, 300, cdev=True)[0] == B.E_INVALID
    assert kx.cdi_parse_raw(fmt, cdev_doc, K.KIND_SHORT, 300)[0] == B.E_INVALID
    assert kx.cdi_parse_raw(fmt, cdev_doc, K.KIND_SHORT, 300, mdev=True)[0] == B.E_INVALID
    # the group parse of the group document returns vfio_cdev = 0, as before
    got = kx.cdi_parse(fmt, group_doc, K.KIND_SHORT)
    assert not got[K.CDEV_FIELD].any() and got["index"].tobytes() == recs["index"].tobytes()
    # the zero-device document is the same bytes in both layouts
    zero = K.oracle_doc(fmt, K.KIND_SHORT, recs[:0])
    assert zero == kx.cdi_emit(fmt, recs[:0], K.KIND_SHORT) == kx.cdi_emit_cdev(fmt, recs[:0], K.KIND_SHORT)
    assert kx.cdi_parse_raw(fmt, zero, K.KIND_SHORT, 0, cdev=True)[:2] == (B.KXPU_OK, 0)


def test_nospace_protocol(kx):
    recs = K.records(200, seed=3)
    doc = K.oracle_doc(K.FMT_JSON, K.KIND_SHORT, recs)
    rc, n, _ = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 0, cdev=True)  # out = NULL: the sizing call
    assert (rc, n) == (B.E_NOSPACE, 200)
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 199, cdev=True)
    assert (rc, n) == (B.E_NOSPACE, 200) and not out.tobytes().strip(b"\0")  # nothing written
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 200, cdev=True)
    assert (rc, n) == (B.KXPU_OK, 200) and out.tobytes() == recs.tobytes()
    assert len(doc) // B.CDI_FRAG_MIN >= 200
