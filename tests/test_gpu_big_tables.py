"""GPU parity of the pci.ids path on tables far larger than the real file's 18 856 rows, against the oracle.

The library picks its code path from the table size: the table grows x16 when it ran full and x4 when it
crossed its load limit (several attempts in one call), the name blob grows when it overflowed, the fold of
resolve_chunks_kernel loads before it claims once the table (cap > 2^20 slots) no longer sits in L2, and the
finalize scans 32 slots per warp for tables of 2^19 slots and more.  Texts of 71 k, 778 k and 12.4 M keys
from workloads.synthetic_pci_ids (every vendor block alive: nothing can be skipped) reach each of these, and
every test asserts the precondition of its regime.  Every test builds its own context: the table-size hint
a context carries from one load to the next decides where the next load starts."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T_RESOLVE = 7  # kxpu.h KXPU_T_RESOLVE: nonzero only when the big-text kernels ran


@pytest.fixture
def fresh(monkeypatch):
    """fresh(**env) -> a new context created under the given KXPU_* environment; closed at teardown."""
    import kxpu_b200 as K
    made = []

    def make(**env):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        k = K.Kxpu(0)
        made.append(k)
        return k
    yield make
    for k in made:
        k.close()


@pytest.fixture(scope="module")
def text_778k(workloads, oracle):
    text = workloads.synthetic_pci_ids(4096, 190)
    return text, oracle.table_build(text)


@pytest.fixture(scope="module")
def text_12m(workloads, oracle):
    text = workloads.synthetic_pci_ids(65536, 190)
    return text, oracle.table_build(text)


def expected_rows(want, q):
    """Line offset the oracle's table gives each key of q (-1 on a miss)."""
    order = np.argsort(want["key"], kind="stable")
    sk = want["key"][order]
    pos = np.searchsorted(sk, q)
    pos[pos >= len(sk)] = 0
    return np.where(sk[pos] == q, want["line_off"][order][pos].astype(np.int64), -1)


def check_loaded(kx, oracle, workloads, tab, text, want, seed, extra_keys=()):
    """Whole-table parity of a loaded table: keys and line offsets of every row, the names of every row (one
    blob, no per-row objects) and 2^20 lookups.  Returns the name bytes of the table."""
    keys, offs, rows = kx.table_export(tab)
    assert len(keys) == len(want)
    assert np.array_equal(keys, want["key"]) and np.array_equal(offs, want["line_off"])
    blob, noffs = kx.names_blob(tab, rows)
    oblob, ooffs = oracle.names_bulk(text, want["line_off"])
    assert np.array_equal(noffs, ooffs)
    assert blob == oblob
    q = np.concatenate([workloads.make_queries(want["key"], 1 << 20, seed), np.asarray(extra_keys, np.uint32)]).astype(np.uint32)
    r = kx.lookup(tab, q)
    line_of_row = np.full(tab.rows + 1, -1, np.int64)
    line_of_row[rows] = offs.astype(np.int64)
    got = np.where(r >= 0, line_of_row[np.maximum(r, 0)], -1)
    assert np.array_equal(got, expected_rows(want, q))
    return len(blob)


def load_and_check(kx, oracle, workloads, text, want, seed, extra_keys=()):
    """Load `text` with kxpu_pciids_load and check the whole table.  Returns (resolve ms, name bytes)."""
    tab = kx.pciids_load(text)
    try:
        resolve_ms = kx.timings()[T_RESOLVE]  # before any other call clears the stage timings
        return resolve_ms, check_loaded(kx, oracle, workloads, tab, text, want, seed, extra_keys)
    finally:
        tab.free()


def check_pci_ids(kx, oracle_rows, golden, tab):
    """The real file's table: oracle rows and the golden dump sha256."""
    keys, offs, rows = kx.table_export(tab)
    assert np.array_equal(keys, oracle_rows["key"]) and np.array_equal(offs, oracle_rows["line_off"])
    blob, noffs = kx.names_blob(tab, rows)
    dump = b"".join(b"%04x:%04x\t%s\n" % (k >> 16, k & 0xFFFF, blob[noffs[i]:noffs[i + 1]]) for i, k in enumerate(keys.tolist()))
    assert hashlib.sha256(dump).hexdigest() == golden["dump_sha256"]


def start_cap(prev_keys, n):
    """Slots the next load of an n-byte text starts with after a load of prev_keys keys on the same context:
    the size hint (kx_note_table_size) shrunk while it exceeds a table of one key per 6 bytes."""
    cap = 1 << 16
    while cap < (1 << 28) and cap // 2 < prev_keys + prev_keys // 8:
        cap <<= 1
    while cap > (1 << 16) and cap // 2 > n // 6 + 1:
        cap >>= 1
    return cap


@pytest.mark.parametrize("path", ["small", "big"])
def test_71k_keys_outgrow_the_first_table(path, fresh, oracle, workloads):
    """71 680 keys > the 2^16 slots a fresh context starts with: the table runs full and grows x16 to 2^20.  The
    3 MB text fits the cooperative small-text kernel (its names phase then scans 32 slots per warp); with
    KXPU_NO_SMALL=1 it goes through parse + resolve (claim-first fold, cap <= 2^20) + select_finalize (scan_w 32)."""
    kx = fresh(**({"KXPU_NO_SMALL": "1"} if path == "big" else {}))
    text = workloads.synthetic_pci_ids(1024, 70, subs_per_dev=0)
    want = oracle.table_build(text)
    assert len(want) == 71680 > (1 << 16)
    resolve_ms, _ = load_and_check(kx, oracle, workloads, text, want, 71)
    assert (resolve_ms == 0) == (path == "small")


def _variant(text, kind, workloads):
    if kind == "plain":
        return text
    if kind == "devices_only":
        # no subsystem lines: ~48 device lines per 2 KiB chunk, more than one per lane, so a warp of the fold
        # takes each chunk's head lines in two rounds (with subsystem lines a chunk holds ~26)
        return workloads.synthetic_pci_ids(4096, 190, subs_per_dev=0)
    if kind == "copies2":  # every key has a losing duplicate in the dead second copy
        return np.concatenate([text, text])
    if kind == "long_line":
        # a >= 64 KiB line at three quarters of the text: bufio.ErrTooLong cuts the rest off.  The parse still
        # folds every key, so the table grows in the same call as the finalize asks for the cut-off
        block = len(text) // 4096
        cut = 3072 * block
        assert text[cut - 1] == 0x0a and text[cut] != 0x09
        return np.concatenate([text[:cut], np.frombuffer(b"#" + b"x" * 70000 + b"\n", np.uint8), text[cut:]])
    if kind == "ffff":  # key 0xffffffff lives in the dedicated slot `cap`
        head = b"ffff  Illegal Vendor ID\n\tffff  All ones\n\t0000  Zero\n"
        return np.concatenate([np.frombuffer(head, np.uint8), text])
    raise AssertionError(kind)


@pytest.mark.parametrize("kind", ["plain", "devices_only", "copies2", "long_line", "ffff"])
def test_778k_keys_load_first_fold(kind, fresh, oracle, workloads, text_778k):
    """778 240 keys > 2^19 = the load limit of a 2^20 table, so the final table has >= 2^21 slots: the fold of
    resolve_chunks_kernel takes its load-first branch and the finalize scans 32 slots per warp.  Over 4 MiB of
    names > the 4 MiB first blob: the blob is grown and the text parsed again."""
    kx = fresh()
    text = _variant(text_778k[0], kind, workloads)
    want = text_778k[1] if kind in ("plain", "copies2") else oracle.table_build(text)
    assert len(want) > (1 << 19)
    extra = [0xffffffff, 0xffff0000, 0xfffffffe, 0]
    resolve_ms, name_bytes = load_and_check(kx, oracle, workloads, text, want, 778, extra)
    assert resolve_ms > 0  # 60 MB: the big-text kernels
    assert name_bytes > (4 << 20)
    if kind == "ffff":
        assert int(want["key"][0]) == 0xffffffff
    if kind == "long_line":
        assert len(want) < len(text_778k[1])


def test_12m_keys_design_case(fresh, oracle, workloads, text_12m):
    """DESIGN.md's 12.4 M-key, 0.96 GB all-alive text on a fresh context: from 2^16 slots the table must grow
    at least three times (12.45 M keys > 2^23, the load limit of a 2^24 table) and the blob from 4 MiB to
    hundreds of MiB, all in one call."""
    import torch
    kx = fresh()
    text, want = text_12m
    assert len(want) == 12451840 > (1 << 23)
    resolve_ms, name_bytes = load_and_check(kx, oracle, workloads, text, want, 12)
    assert resolve_ms > 0 and name_bytes > (256 << 20)
    free, total = torch.cuda.mem_get_info(0)  # the arena stays parked in the context after the table is freed
    print("12.4M-key load: %.2f GiB of %.2f GiB device memory in use" % ((total - free) / 2**30, total / 2**30))


def test_context_history(fresh, oracle, workloads, oracle_rows, golden, pci_text, text_778k, text_12m):
    """One context, four loads: each must equal what a fresh context computes (the oracle).  After the
    778 k-key load the size hint starts pci.ids at 2^18 slots, four times its usual table, so the small-text
    kernel's names phase scans 32 slots per warp; after the 12.4 M-key load it also starts with the big blob."""
    kx = fresh()
    load_and_check(kx, oracle, workloads, text_778k[0], text_778k[1], 1)
    assert start_cap(len(text_778k[1]), len(pci_text)) == 1 << 18
    tab = kx.pciids_load(pci_text)
    try:
        assert kx.timings()[T_RESOLVE] == 0
        check_pci_ids(kx, oracle_rows, golden, tab)
    finally:
        tab.free()
    load_and_check(kx, oracle, workloads, text_12m[0], text_12m[1], 2)
    assert start_cap(len(text_12m[1]), len(pci_text)) == 1 << 18
    # zero-copy join: text, keys and row handles in mapped pinned host memory
    q = workloads.make_queries(oracle_rows["key"], 4096, 3)
    h_text, p1 = kx.pinned(len(pci_text))
    h_q, p2 = kx.pinned(len(q) * 4, np.uint32)
    h_r, p3 = kx.pinned(len(q) * 4, np.int32)
    try:
        h_text[:] = np.frombuffer(pci_text, np.uint8)
        h_q[:] = q
        h_r[:] = -7
        tab, rows = kx.pciids_join(h_text, h_q, rows_out=h_r)
        try:
            assert kx.timings()[T_RESOLVE] == 0
            check_pci_ids(kx, oracle_rows, golden, tab)
            _, offs, trows = kx.table_export(tab)
            line_of_row = np.full(tab.rows + 1, -1, np.int64)
            line_of_row[trows] = offs.astype(np.int64)
            got = np.where(rows >= 0, line_of_row[np.maximum(rows, 0)], -1)
            assert np.array_equal(got, expected_rows(oracle_rows, q))
        finally:
            tab.free()
    finally:
        for p in (p1, p2, p3):
            kx.pinned_free(p)
