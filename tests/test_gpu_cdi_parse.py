"""GPU checks of kxpu_cdi_parse / kxpu_cdi_parse_mdev: the records of the oracle's documents come back exactly (both
formats, both layouts, a short and a 63-byte kind, up to 2^20 devices, unaligned host buffers), damaged documents get
pyref_cdi_parse's verdict, and KXPU_E_NOSPACE follows the sizing protocol."""
import numpy as np
import pytest

import cdi_parse_cases as K
import pyref_cdi_parse as P
from kxpu_b200 import binding as B

pytestmark = pytest.mark.gpu

CASES = [(fmt, kind, mdev) for fmt in (K.FMT_YAML, K.FMT_JSON) for kind in (K.KIND_SHORT, K.KIND_LONG) for mdev in (False, True)]


@pytest.mark.parametrize("fmt,kind,mdev", CASES)
@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 65536, 1 << 20])
def test_round_trip(kx, fmt, kind, mdev, n):
    recs = K.records(n, mdev, seed=n + 7)
    doc = K.emit(fmt, kind, recs, mdev)
    got = kx.cdi_parse_mdev(fmt, doc, kind) if mdev else kx.cdi_parse(fmt, doc, kind)
    assert len(got) == n
    assert got.tobytes() == recs.tobytes()
    if n <= 129:  # the host buffer at every 16-byte phase
        for off in range(1, 16):
            rc, m, out = kx.cdi_parse_raw(fmt, doc, kind, n, mdev, off)
            assert (rc, m) == (B.KXPU_OK, n), off
            assert out.tobytes() == recs.tobytes(), off


@pytest.mark.parametrize("fmt,kind,mdev", CASES)
def test_damaged_documents(kx, fmt, kind, mdev):
    _, docs = K.damaged(fmt, kind, mdev)
    for name, doc in docs:
        st, want = P.parse(fmt, doc, kind, mdev)
        rc, n, out = kx.cdi_parse_raw(fmt, doc, kind, 8, mdev, 3)
        assert rc == st, name
        if st == P.OK:
            assert n == len(want) and out[:n].tobytes() == want.tobytes(), name
        else:
            assert n == -1, name  # *n untouched
    # the wrong kind: another kind's document, a kind outside the domain
    doc = docs[0][1]
    assert kx.cdi_parse_raw(fmt, doc, b"example.com/other", 8, mdev)[0] == B.E_INVALID
    assert kx.cdi_parse_raw(fmt, doc, b"no-slash", 8, mdev)[0] == B.E_UNSUPPORTED
    assert kx.cdi_parse_raw(1 - fmt, doc, kind, 8, mdev)[0] == B.E_INVALID


def test_pci_document_is_not_an_mdev_document(kx):
    recs = K.records(3)
    doc = K.emit(K.FMT_YAML, K.KIND_SHORT, recs)
    assert kx.cdi_parse_raw(K.FMT_YAML, doc, K.KIND_SHORT, 8, True)[0] == B.E_INVALID


@pytest.mark.parametrize("mdev", [False, True])
def test_nospace_protocol(kx, mdev):
    recs = K.records(200, mdev, seed=3)
    doc = K.emit(K.FMT_JSON, K.KIND_SHORT, recs, mdev)
    rc, n, _ = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 0, mdev)  # out = NULL: the sizing call
    assert (rc, n) == (B.E_NOSPACE, 200)
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 199, mdev)
    assert (rc, n) == (B.E_NOSPACE, 200) and not out.tobytes().strip(b"\0")  # nothing written
    rc, n, out = kx.cdi_parse_raw(K.FMT_JSON, doc, K.KIND_SHORT, 200, mdev)
    assert (rc, n) == (B.KXPU_OK, 200) and out.tobytes() == recs.tobytes()
    assert len(doc) // B.CDI_FRAG_MIN >= 200  # the header's bound holds


def test_parse_is_timed(kx):
    recs = K.records(1000, seed=5)
    kx.cdi_parse(K.FMT_YAML, K.emit(K.FMT_YAML, K.KIND_SHORT, recs), K.KIND_SHORT)
    assert kx.timings()[B.T_EMIT] > 0
