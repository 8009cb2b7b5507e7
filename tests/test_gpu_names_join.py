"""kxpu_pciids_join_device on the big-text path: the select pass hands out row handles, then one launch names the rows
while the other blocks of the same launch join the keys.  Every case is checked against the oracle: the table (keys
and lines), the name of every row, and the line every key's row handle stands for."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def big_path_ctx():
    """A new context whose small texts also take the big-text kernels (KXPU_NO_SMALL=1, read at creation)."""
    import kxpu_b200 as K
    old = os.environ.get("KXPU_NO_SMALL")
    os.environ["KXPU_NO_SMALL"] = "1"
    try:
        return K.Kxpu(0)
    finally:
        if old is None:
            del os.environ["KXPU_NO_SMALL"]
        else:
            os.environ["KXPU_NO_SMALL"] = old


@pytest.fixture(scope="module")
def kb():
    k = big_path_ctx()
    yield k
    k.close()


@pytest.fixture
def fresh_kb():
    """A big-path context that starts from the default table and blob sizes."""
    k = big_path_ctx()
    yield k
    k.close()


def expected_lines(want, q):
    """Line offset of the oracle's row of every key (-1 = miss)."""
    if len(want) == 0:
        return np.full(len(q), -1, np.int64)
    order = np.argsort(want["key"])
    sk = want["key"][order]
    pos = np.minimum(np.searchsorted(sk, q), len(sk) - 1)
    return np.where(sk[pos] == q, want["line_off"][order][pos].astype(np.int64), -1)


def join_and_check(kx, oracle, text, q, pad=0):
    """One kxpu_pciids_join_device call; keys and row handles `pad` 4-byte words into their buffers (pad = 1: not
    16-byte aligned).  The words around the row handles must stay untouched."""
    from kxpu_b200 import binding as B
    buf = np.frombuffer(text, np.uint8)
    q = np.ascontiguousarray(q, np.uint32)
    nq = len(q)
    d_text = kx.dev_alloc(max(len(buf), 16))
    d_q = kx.dev_alloc(4 * (nq + pad + 1))
    d_r = kx.dev_alloc(4 * (nq + pad + 1))
    try:
        if len(buf):
            kx.upload(d_text, buf)
        kx.upload(d_q, np.concatenate([np.zeros(pad, np.uint32), q, np.zeros(1, np.uint32)]))
        kx.upload(d_r, np.full(nq + pad + 1, -7, np.int32))
        t = kx.pciids_join_device(d_text, len(buf), d_q + 4 * pad, nq, d_r + 4 * pad)
        try:
            tm = kx.timings()
            assert tm[B.T_LOOKUP] == 0.0  # the join runs inside the finalize's launches
            want = oracle.table_build(text)
            keys, offs, rows = kx.table_export(t)
            assert t.rows == len(want)
            assert np.array_equal(keys, want["key"]) and np.array_equal(offs, want["line_off"])
            assert sorted(rows.tolist()) == list(range(t.rows))  # dense row handles
            blob, noffs = kx.names_blob(t, rows)
            oblob, ooffs = oracle.names_bulk(text, want["line_off"])
            assert np.array_equal(noffs, ooffs) and blob == oblob
            got = kx.download(d_r, 4 * (nq + pad + 1), np.int32)
            assert (got[:pad] == -7).all() and got[pad + nq] == -7
            got = got[pad:pad + nq]
            line_of_row = np.full(t.rows + 1, -1, np.int64)
            line_of_row[rows] = offs.astype(np.int64)
            assert (got >= -1).all() and (got < max(t.rows, 1)).all()
            got_line = np.where(got >= 0, line_of_row[np.maximum(got, 0)], -1)
            assert np.array_equal(got_line, expected_lines(want, q))
            return t.rows, int((got >= 0).sum())
        finally:
            t.free()
    finally:
        for d in (d_text, d_q, d_r):
            kx.dev_free(d)


@pytest.mark.parametrize("nq", [0, 1, 255, 256, 257, 4097, 1 << 20])
def test_key_counts(nq, kb, oracle, pci_text, oracle_rows, workloads):
    q = workloads.make_queries(oracle_rows["key"], nq, 21) if nq else np.zeros(0, np.uint32)
    rows, hits = join_and_check(kb, oracle, pci_text, q)
    assert rows == len(oracle_rows) and (hits > 0 or nq < 4)


def rows_text(n_rows, vendor=0x1234):
    return b"%04x  Vendor\n" % vendor + b"".join(b"\t%04x  Device %d\n" % (d, d) for d in range(n_rows))


@pytest.mark.parametrize("text", [b"", b"\n", b"1234  V\n", rows_text(1), rows_text(7), rows_text(13), rows_text(1003),
                                  rows_text(64) + rows_text(9, 0x1234) + rows_text(57, 0x4321)],
                         ids=["empty", "newline", "vendor-only", "one-row", "7-rows", "13-rows", "1003-rows", "repeated-vendor"])
def test_small_texts(text, kb, oracle):
    q = np.array([0x12340000, 0x12340001, 0x12340006, 0x123403ea, 0x43210005, 0x12350000, 0xffffffff], np.uint32)
    join_and_check(kb, oracle, text, q)


def test_unaligned_keys_and_rows(kb, oracle, pci_text, oracle_rows, workloads):
    for pad in (1, 2, 3):
        join_and_check(kb, oracle, pci_text, workloads.make_queries(oracle_rows["key"], 5000 + pad, pad), pad=pad)


def test_table_that_must_grow(fresh_kb, oracle, workloads):
    """40 000 keys do not fit the 2^16 slots a context starts with: the table grows and both launches run again."""
    text = b"abcd  Big\n" + b"".join(b"\t%04x  x %d\n" % (d, d) for d in range(40000))
    want = oracle.table_build(text)
    q = np.concatenate([workloads.make_queries(want["key"], 70000, 3), np.array([0xabcd9c40, 0xffffffff], np.uint32)])
    rows, _ = join_and_check(fresh_kb, oracle, text, q)
    assert rows == 40000


def test_blob_that_must_grow(fresh_kb, oracle, workloads):
    """More than 4 MiB of names (the first blob a 5+ MB text gets): the blob overflows, grows and both launches run
    again.  The names are longer than the 128-byte window, so they take the long-line path."""
    name = b"Very long device name / with spaces. and dots " * 4
    text = b"".join(b"%04x  V\n" % v + b"".join(b"\t%04x  " % d + name + b"%d\n" % d for d in range(12000)) for v in (0x1111, 0x2222))
    want = oracle.table_build(text)
    _, ooffs = oracle.names_bulk(text, want["line_off"])
    assert len(text) > (4 << 20) and int(ooffs[-1]) > (4 << 20)
    join_and_check(fresh_kb, oracle, text, workloads.make_queries(want["key"], 30000, 4))


def test_text_that_takes_the_cut_off_rerun(kb, oracle, pci_text, workloads):
    """A line of 70 000 bytes: the parse raises the long-line hint, the select pass stands back, the host computes the
    bufio.ErrTooLong cut-off and runs both launches again; device lines behind the cut-off are no rows."""
    head = pci_text[:pci_text.find(b"\n", 200000) + 1]
    text = head + b"3333  " + b"x" * 70000 + b"\n\t0003  hidden\n" + b"4444  f\n\t0004  h\n"
    want = oracle.table_build(text)
    q = np.concatenate([workloads.make_queries(want["key"], 3000, 5), np.array([0x33330003, 0x44440004], np.uint32)])
    join_and_check(kb, oracle, text, q)
