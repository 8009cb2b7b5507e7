"""CPU checks of the CDI spec parse's checkers: pyref_cdi_parse reads back the oracle's documents exactly, refuses what the
oracle would not write, and the index state file of the host's restart resume round-trips."""
import ctypes as C
import os

import numpy as np
import pytest

import cdi_parse_cases as K
import pyref_cdi_parse as P
from conftest import ROOT

CASES = [(fmt, kind, mdev) for fmt in (K.FMT_YAML, K.FMT_JSON) for kind in (K.KIND_SHORT, K.KIND_LONG) for mdev in (False, True)]


@pytest.mark.parametrize("fmt,kind,mdev", CASES)
@pytest.mark.parametrize("n", [0, 1, 2, 127, 129])
def test_pyref_reads_oracle_documents(fmt, kind, mdev, n):
    recs = K.records(n, mdev, seed=n)
    doc = K.emit(fmt, kind, recs, mdev)
    st, got = P.parse(fmt, doc, kind, mdev)
    assert st == P.OK
    assert got.tobytes() == recs.tobytes()


@pytest.mark.parametrize("fmt,kind,mdev", CASES)
def test_pyref_verdicts(fmt, kind, mdev):
    recs, docs = K.damaged(fmt, kind, mdev)
    verdict = {}
    for name, doc in docs:
        st, got = P.parse(fmt, doc, kind, mdev)
        verdict[name] = st
        if st == P.OK:  # accepted means the oracle writes these very bytes from the records read
            assert K.emit(fmt, kind, got, mdev) == doc, name
    assert verdict["clean"] == P.OK and verdict["zero_devices"] == P.OK
    for name in ("trailing_newline", "trailing_byte", "crlf", "leading_zero", "index_past_u64", "group_past_u32",
                 "name_differs", "empty"):
        assert verdict[name] == P.E_INVALID, name
    # YAML has no tail: a document cut where a device begins is the document of the devices before it
    cuts = set(K.boundaries(fmt, K.emit(fmt, kind, recs, mdev))[1:-1]) if fmt == K.FMT_YAML else set()
    for k, v in verdict.items():
        if k.startswith("truncate@"):
            assert v == (P.OK if int(k[9:]) in cuts else P.E_INVALID), k
    assert verdict["duplicated_fragment"] == P.OK  # two equal records: the emitter writes that too
    other = b"example.com/other"
    assert P.parse(fmt, K.emit(fmt, kind, recs, mdev), other, mdev)[0] == P.E_INVALID
    assert P.parse(fmt, K.emit(fmt, kind, recs, mdev), b"no-slash", mdev)[0] == P.E_UNSUPPORTED


def host():
    L = C.CDLL(os.path.join(ROOT, "kata-xpu-device-plugin_b200", "lib", "libkxpu_host.so"))
    L.kxh_index_state_format.restype = C.c_int
    L.kxh_index_state_format.argtypes = [C.c_uint64, C.c_uint64, C.c_char_p, C.c_size_t]
    L.kxh_index_state_parse.restype = C.c_int
    L.kxh_index_state_parse.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    return L


def parse_state(L, text):
    p, m = C.c_uint64(7), C.c_uint64(7)
    ok = L.kxh_index_state_parse(text, len(text), C.byref(p), C.byref(m))
    return (p.value, m.value) if ok else None


@pytest.mark.parametrize("pci,mdev", [(0, 0), (3, 0), (0, 17), (1 << 40, 12345), ((1 << 64) - 1, (1 << 64) - 1)])
def test_index_state_round_trip(pci, mdev):
    L = host()
    buf = C.create_string_buffer(128)
    n = L.kxh_index_state_format(pci, mdev, buf, len(buf))
    assert buf.raw[:n] == b"pci %d\nmdev %d\n" % (pci, mdev)
    assert parse_state(L, buf.raw[:n]) == (pci, mdev)


@pytest.mark.parametrize("text", [b"", b"pci 1\n", b"pci 1\nmdev 2", b"pci 1\nmdev 2\n\n", b"pci 01\nmdev 0\n",
                                  b"pci 1\nmdev -2\n", b"mdev 1\npci 1\n", b"pci  1\nmdev 1\n", b"pci 1\r\nmdev 1\n",
                                  b"pci 18446744073709551616\nmdev 0\n", b"pci \nmdev 0\n", b"pci 1\nmdev 1\nx"])
def test_index_state_malformed(text):
    assert parse_state(host(), text) is None
