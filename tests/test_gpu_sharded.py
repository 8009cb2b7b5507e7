"""GPU parity of the sharded pci.ids load + join at its edges, against the oracle run on the WHOLE text.

kxpu_ctx_create_multi with ordinal 0 repeated runs the real peer-memory exchange between contexts of one process
(phase A, the per-rank winner slab written by the slab branch of select_finalize_kernel, merge_kernel,
join_gather_kernel, gather_copy_kernel and the collective retry decisions of csrc/comm.cu), so all of this runs on
one GPU.  Every load is checked on EVERY rank: all keys and line offsets, the name of every row (the rows of ranks
>= 1 reach their names through the merge's rebasing by the rounded blobs in front of them), the row handle of every
joined key (identical on all ranks) and the result-buffer words behind nq_total.

Texts are built so that plan_shards cuts exactly where a test wants it: parts of equal length (padded with comment
lines behind their first line) make the cut land between them, and the tests assert that it does.  The capacity
tests assert the winner rows / name bytes of every shard they meant to build, so that they cannot drift away from
their edge.  Inputs that one rank refuses after the epoch bump are only tested on a group of one rank: with more,
its peers would wait for a push that never comes."""
import functools

import numpy as np
import pytest

from test_gpu_pciids import UNICODE_CRLF_TEXT, _big_random_text, name_length_text, random_pciids_texts, structural_fuzz_texts
from test_oracle import EDGE_TEXTS

pytestmark = pytest.mark.gpu

SENTINEL = -7
GUARD = 5              # result-buffer words behind nq_total that a load must leave alone
SLAB_ROWS = 65536      # winner rows of one rank's peer slab
SLAB_BLOB = 2 << 20    # sanitised name bytes of one rank's peer slab
MERGED_BLOB = 4 << 20  # name bytes of a fresh group's merged table (grows x4)
JOIN_CAP = 1 << 21     # keys of one sharded join over peer memory
EDGE_KEYS = [0x10de2330, 0x10de0001, 0x10de0002, 0x10df0001, 0, 0xffffffff]
ALNUM = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789", np.uint8)


@pytest.fixture
def group():
    """group(R) -> a new group of R contexts on GPU 0.  Making a group closes the one made before it (one group
    is alive at a time); the last one is closed at teardown."""
    import kxpu_b200 as K
    live = []

    def make(nranks):
        while live:
            live.pop().close()
        live.append(K.KxpuMulti([0] * nranks))
        return live[-1]
    yield make
    while live:
        live.pop().close()


@functools.lru_cache(maxsize=4)
def _expect(oracle, text):
    """The oracle on the whole text: its table and the names of all its rows (kxpu_names layout)."""
    want = oracle.table_build(text)
    blob, offs = oracle.names_bulk(text, want["line_off"])
    return want, blob, offs


def queries(oracle, text, n, seed):
    """n keys: about 3/4 hits from the oracle's table, present vendors with random devices, random keys, 0 and ~0."""
    want = _expect(oracle, text)[0]
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    if len(want):
        pick = rng.random(n)
        k = want["key"][rng.integers(0, len(want), n)]
        q = np.where(pick < 0.75, k, np.where(pick < 0.9, (k & 0xffff0000) | (q & 0xffff), q)).astype(np.uint32)
    q[:min(n, 2)] = [0, 0xffffffff][:min(n, 2)]
    return q


def expected_lines(want, q):
    """Line offset of every key of q in the oracle's table, -1 on a miss."""
    if not len(want):
        return np.full(len(q), -1, np.int64)
    order = np.argsort(want["key"], kind="stable")
    sk = want["key"][order]
    pos = np.searchsorted(sk, q)
    pos[pos >= len(sk)] = 0
    return np.where(sk[pos] == q, want["line_off"][order][pos].astype(np.int64), -1)


def shard_winners(oracle, text, cuts):
    """[(winner rows, sanitised name bytes)] of every shard: the rows of the whole text's table whose line lies in
    it (winners are globally unique, so each row is owned by exactly one shard)."""
    want, _, offs = _expect(oracle, text)
    lens = np.diff(offs.astype(np.int64))
    line = want["line_off"]
    return [(int(((line >= a) & (line < b)).sum()), int(lens[(line >= a) & (line < b)].sum())) for a, b in cuts]


def _same(got, want, what, rank):
    if not np.array_equal(got, want):
        n = min(len(got), len(want))
        bad = np.flatnonzero(np.asarray(got[:n]) != np.asarray(want[:n]))
        at = int(bad[0]) if len(bad) else n
        raise AssertionError("rank %d: %s differ (%d vs %d entries), first at %d: %r vs %r" % (
            rank, what, len(got), len(want), at, got[at] if at < len(got) else None, want[at] if at < len(want) else None))


class Sharded:
    """One sharded load (+ join) of `text` on group `m`, with every shard's global_base shifted by base_shift.
    slices: the (lo, hi) key range of every rank (default: equal slices in rank order); result: per rank "aligned",
    "offset" (the result buffer 4 bytes past a 16-byte boundary) or None (no result buffer).  Result buffers hold
    nq_total + GUARD words of SENTINEL before the load."""

    def __init__(self, m, text, keys=None, slices=None, result=None, base_shift=0):
        import kxpu_b200 as K
        R = len(m.ctxs)
        self.m, self.text, self.base_shift = m, text, base_shift
        self.keys = np.zeros(0, np.uint32) if keys is None else np.ascontiguousarray(keys, np.uint32)
        self.nq = len(self.keys)
        self.cuts = K.plan_shards(text, R)
        if slices is None:
            per = -(-self.nq // R)
            slices = [(min(r * per, self.nq), min((r + 1) * per, self.nq)) for r in range(R)]
        self.slices, self.result = slices, result or ["aligned"] * R
        self.shards, self.res, self.bufs, self.tabs = [], [], [], []
        try:
            for r, (a, b) in enumerate(self.cuts):
                kx = m.ctxs[r]
                sh = dict(d_text=self._upload(kx, text[a:b]), n=b - a, global_base=a + base_shift)
                dr = None
                if self.nq:
                    lo, hi = slices[r]
                    sh.update(nq=hi - lo, key_offset=lo)
                    if hi > lo:
                        sh["d_keys"] = self._upload(kx, self.keys[lo:hi].tobytes())
                    if self.result[r]:
                        skew = 4 if self.result[r] == "offset" else 0
                        dr = self._alloc(kx, skew + (self.nq + GUARD) * 4) + skew
                        kx.upload(dr, np.full(self.nq + GUARD, SENTINEL, np.int32))
                        sh["d_rows_all"] = dr
                self.res.append(dr)
                self.shards.append(sh)
        except BaseException:
            self.free()
            raise

    def _alloc(self, kx, nbytes):
        d = kx.dev_alloc(max(nbytes, 16))
        self.bufs.append((kx, d))
        return d

    def _upload(self, kx, data):
        d = self._alloc(kx, len(data))
        if len(data):
            kx.upload(d, np.frombuffer(data, np.uint8))
        return d

    def join(self):
        self.tabs = self.m.pciids_join(self.shards, self.nq)
        return self

    def results(self, r):
        """Rank r's result buffer: nq_total row handles, then the guard words."""
        return self.m.ctxs[r].download(self.res[r], (self.nq + GUARD) * 4, np.int32)

    def check(self, oracle):
        """Every rank against the oracle on the whole text; returns shard_winners of the cut."""
        want, wblob, woffs = _expect(oracle, self.text)
        exp = expected_lines(want, self.keys)
        exp = np.where(exp >= 0, exp + self.base_shift, -1)
        first = None
        for r, t in enumerate(self.tabs):
            kx = self.m.ctxs[r]
            keys, offs, rows = kx.table_export(t)
            _same(keys, want["key"], "keys", r)
            _same(offs, want["line_off"] + np.uint64(self.base_shift), "line offsets", r)
            blob, noffs = kx.names_blob(t, rows)
            if not (np.array_equal(noffs, woffs) and blob == wblob):
                bad = next((i for i in range(len(woffs) - 1) if i + 1 >= len(noffs) or
                            blob[noffs[i]:noffs[i + 1]] != wblob[woffs[i]:woffs[i + 1]]), None)
                raise AssertionError("rank %d: names differ, first at row %r (line %d)" % (
                    r, bad, int(want["line_off"][bad]) if bad is not None else -1))
            if self.nq and self.res[r] is not None:
                got = self.results(r)
                assert (got[self.nq:] == SENTINEL).all(), ("rank %d: words behind nq_total written" % r, got[self.nq:])
                got = got[:self.nq]
                line_of_row = np.full(int(rows.max()) + 2 if len(rows) else 1, -2, np.int64)
                line_of_row[rows] = offs.astype(np.int64)
                assert ((got >= -1) & (got < len(line_of_row))).all(), "rank %d: handles out of range" % r
                _same(np.where(got >= 0, line_of_row[np.maximum(got, 0)], -1), exp, "joined lines", r)
                if first is None:
                    first = got
                _same(got, first, "row handles (vs the first rank with a result buffer)", r)
        return shard_winners(oracle, self.text, self.cuts)

    def free(self):
        for t in self.tabs:
            t.free()
        self.tabs = []
        for kx, d in self.bufs:
            kx.dev_free(d)
        self.bufs = []


def check_sharded(m, oracle, text, keys=None, **kw):
    """Sharded load (+ join) of text on group m, checked on every rank; returns shard_winners of the cut."""
    s = Sharded(m, text, keys, **kw)
    try:
        return s.join().check(oracle)
    finally:
        s.free()


# ------------------------------------------------------------------ texts
def padded(parts):
    """Parts, each starting with a top-level line, padded with comment lines behind their first line to one length
    L (comments neither end a block nor start a shard), joined.  plan_shards(text, len(parts)) cuts exactly between
    them.  Returns (text, L)."""
    L = max(len(p) for p in parts) + 2
    out = []
    for p in parts:
        head = p.index(b"\n") + 1
        pad, fill = L - len(p), []
        while pad:
            k = min(pad, 1000)
            k -= 1 if pad - k == 1 else 0
            fill.append(b"#" + b"p" * (k - 2) + b"\n")
            pad -= k
        out.append(p[:head] + b"".join(fill) + p[head:])
    return b"".join(out), L


def assert_cuts(text, nranks, L):
    import kxpu_b200 as K
    assert K.plan_shards(text, nranks) == [(r * L, (r + 1) * L) for r in range(nranks)]


def block(vendor, lens, rng, dev0=0):
    """A vendor block with one device line per entry of lens, names of [A-Z0-9] (sanitised length = raw length)."""
    names = ALNUM[rng.integers(0, len(ALNUM), int(sum(lens)))].tobytes()
    lines, at = [b"%04x  Vendor %04x\n" % (vendor, vendor)], 0
    for d, ln in enumerate(lens):
        lines.append(b"\t%04x  " % (dev0 + d) + names[at:at + ln] + b"\n")
        at += ln
    return b"".join(lines)


def name_length_shards(nranks):
    """Rank 0 a small block, ranks 1.. one name-length block each (every finalize name path in a slab that is not
    rank 0's), cut exactly between them."""
    parts = [b"0001  Small\n\t0001  short name\n"] + [name_length_text(0x1234 + k)[0] for k in range(nranks - 1)]
    text, L = padded(parts)
    assert_cuts(text, nranks, L)
    return text


def text_cases(oracle, nranks):
    """(text, keys) through the sharded path: the single-path tests' edge texts, seeded random texts and byte fuzz,
    CRLF / non-ASCII names, the all-ones key and the name-length blocks."""
    for text in EDGE_TEXTS:
        yield text, np.array(EDGE_KEYS, np.uint32)
    for text, keys in random_pciids_texts():
        yield text, np.array(keys + [0, 0xffffffff], np.uint32)
    for text, keys in structural_fuzz_texts():
        yield text, np.array(keys, np.uint32)
    rng = np.random.default_rng(77)
    for n_lines, vendors, dup in [(12000, 300, 0.3), (40000, 50, 0.6), (60000, 4000, 0.05)]:
        text = _big_random_text(rng, n_lines, vendors, dup)
        yield text, queries(oracle, text, 3000, n_lines)
    yield UNICODE_CRLF_TEXT, np.array([0x10de0000 + i for i in range(1, 9)], np.uint32)
    ffff, _ = padded([b"0001  One\n\t0001  a\n", b"ffff  Illegal Vendor ID\n\tffff  all ones\n\t0000  zeros\n",
                      b"0000  zero vendor\n\t0000  z\n\tffff  zf\n"])
    yield ffff, np.array([0xffffffff, 0xffff0000, 0, 0x0000ffff, 0x00010001, 0xfffffffe], np.uint32)
    if nranks > 1:
        text = name_length_shards(nranks)
        yield text, queries(oracle, text, 2000, 3)


# ------------------------------------------------------------------ tests
@pytest.mark.parametrize("nranks", [2, 3, 5, 8])
def test_texts_on_every_rank(nranks, group, oracle):
    """Edge texts, random texts and byte fuzz with the single-path tests' seeds, CRLF and non-ASCII names, the
    all-ones key under vendor ffff (dedicated slot) and names around every finalize window in ranks >= 1."""
    m = group(nranks)
    n = 0
    for text, keys in text_cases(oracle, nranks):
        check_sharded(m, oracle, text, keys)
        n += 1
    assert n == len(EDGE_TEXTS) + 12 + 60 + 3 + 2 + (nranks > 1)


def test_names_of_every_rank_come_from_its_slab(group, oracle):
    """Eight ranks with names of their own: the winners of every rank and their names, rank r's blob behind the
    16-byte-rounded blobs of ranks < r (blob sizes that are not multiples of 16)."""
    rng = np.random.default_rng(12)
    parts = [block(0x4000 + r, list(rng.integers(1, 200, 300 + 37 * r)), rng) for r in range(8)]
    text, L = padded(parts)
    assert_cuts(text, 8, L)
    win = check_sharded(group(8), oracle, text, queries(oracle, text, 4000, 12))
    assert [w[0] for w in win] == [300 + 37 * r for r in range(8)]
    assert any(w[1] % 16 for w in win[:-1])


CUT_LAYOUTS = {
    # a vendor's first block (no device lines) in shard 0, its duplicate with devices in shard 1: the devices miss
    "first_block_empty": [b"10de  first\n", b"10de  again\n\t0001  hidden\n\t0002  hidden\n10df  x\n\t0001  y\n"],
    "first_block_empty_far": [b"10de  first\n1111  a\n\t0001  x\n", b"2222  b\n\t0001  y\n",
                              b"10de  again\n\t0001  hidden\n"],
    # a vendor seen first in the last shard; an earlier vendor repeated there
    "first_in_last": [b"1111  a\n\t0001  x\n", b"2222  b\n\t0001  y\n",
                      b"3333  c\n\t0001  z\n\t0002  w\n1111  again\n\t0002  hidden\n"],
    # shards that start with a blank line and with a class line (both end the block in front of them)
    "blank_and_class": [b"1111  a\n\t0001  x\n", b"\n\t0002  orphan after blank\n2222  b\n\t0001  y\n",
                        b"C 03  Display\n\t00  VGA\n\t0003  under a class\n3333  c\n\t0001  z\n"],
}


@pytest.mark.parametrize("layout", sorted(CUT_LAYOUTS))
def test_cut_layouts(layout, group, oracle):
    parts = CUT_LAYOUTS[layout]
    text, L = padded(parts)
    assert_cuts(text, len(parts), L)
    keys = np.array([v << 16 | d for v in (0x10de, 0x10df, 0x1111, 0x2222, 0x3333, 0x0003) for d in range(4)], np.uint32)
    check_sharded(group(len(parts)), oracle, text, keys)


@pytest.mark.parametrize("nranks", [5, 8])
def test_empty_shards(nranks, group, oracle):
    """More ranks than top-level lines: the later ranks get empty shards and still take part in every phase."""
    import kxpu_b200 as K
    m = group(nranks)
    for text in (b"10de  NV\n\t0001  a\n10df  x\n\t0002  b\n", b"\tonly\n\tdevice lines\n", b"10de  NV\n\t0001  a",
                 b"10de  NV\n" + b"".join(b"\t%04x  d\n" % d for d in range(3000))):
        assert sum(a == b for a, b in K.plan_shards(text, nranks)) >= nranks - 2
        check_sharded(m, oracle, text, np.array(EDGE_KEYS + [0x10de0bb7], np.uint32))


def _cutoff_text(nranks, where, content, cr, terminated=True):
    """One part per rank; part `where` holds a device line of `content` bytes in front of its newline (the last of
    them a CR when cr), or an unterminated final line of that length."""
    line = b"\t0003  " + b"L" * (content - 7 - cr) + b"\r" * cr
    parts = []
    for k in range(nranks):
        p = b"%04x  Vendor %d\n\t0001  first %d\n" % (0x2000 + k, k, k)
        if k == where and terminated:
            p += line + b"\n"
        p += b"\t0002  after %d\n%04x  Next %d\n\t0001  n\n" % (k, 0x3000 + k, k)
        if k == where and not terminated:
            p += line
        parts.append(p)
    text, L = padded(parts)
    assert_cuts(text, nranks, L)
    keys = np.array([(v + k) << 16 | d for v in (0x2000, 0x3000) for k in range(nranks) for d in (1, 2, 3)], np.uint32)
    return text, keys


@pytest.mark.parametrize("nranks", [3, 5])
def test_cutoff_across_shards(nranks, group, oracle):
    """bufio.ErrTooLong: a line of 65 536 content bytes cuts off everything behind it in every shard (the global
    minimum of the shards' cut-offs); 65 535 bytes only raise the long-line hint and the retry with exact cut-offs.
    With and without a trailing CR, in the first, a middle and the last shard, and as an unterminated final line."""
    m = group(nranks)
    for where in (0, nranks // 2, nranks - 1):
        for content in (65535, 65536):
            for cr in (0, 1):
                text, keys = _cutoff_text(nranks, where, content, cr)
                win = [w[0] for w in check_sharded(m, oracle, text, keys)]
                # the cut-off is there (65 536) or not (65 535): rows of the shards behind the long line's
                assert win[where + 1:] == [0 if content == 65536 else 3] * (nranks - 1 - where), (where, content, cr, win)
                assert win[where] == (1 if content == 65536 else 4) and win[:where] == [3] * where, (where, content, cr, win)
    for content in (65535, 65536):
        for cr in (0, 1):
            text, keys = _cutoff_text(nranks, nranks - 1, content, cr, terminated=False)
            check_sharded(m, oracle, text, keys)


def _refused(m, oracle, text, status, message):
    import kxpu_b200 as K
    with pytest.raises(K.KxpuError) as e:
        check_sharded(m, oracle, text)
    assert e.value.status == status and message in str(e.value), str(e.value)


def test_slab_row_limit(group, oracle, pci_text):
    """A rank's slab holds 65 536 winner rows: exactly that many load, one more is KXPU_E_CAPACITY.  The same group
    loads pci.ids correctly after the refusal."""
    from kxpu_b200.binding import E_CAPACITY
    rng = np.random.default_rng(4)
    q = queries(oracle, pci_text, 5000, 4)
    for extra in (0, 1):
        text, L = padded([b"0001  Small\n\t0001  A\n", block(0x1000, [1] * SLAB_ROWS, rng) + block(0x1001, [1] * extra, rng)])
        assert_cuts(text, 2, L)
        assert [w[0] for w in shard_winners(oracle, text, [(0, L), (L, 2 * L)])] == [1, SLAB_ROWS + extra]
        m = group(2)
        if extra:
            _refused(m, oracle, text, E_CAPACITY, "outgrow the peer slab")
        else:
            check_sharded(m, oracle, text, queries(oracle, text, 5000, 5))
        check_sharded(m, oracle, pci_text, q)


def test_slab_blob_limit(group, oracle, pci_text):
    """A rank's slab holds 2 MiB of sanitised names: exactly 2 MiB load, 2 MiB + 1 is KXPU_E_CAPACITY."""
    from kxpu_b200.binding import E_CAPACITY
    rng = np.random.default_rng(6)
    q = queries(oracle, pci_text, 5000, 6)
    n = SLAB_BLOB // 64
    for extra in (0, 1):
        text, L = padded([b"0001  Small\n\t0001  ABC\n", block(0x1000, [64] * (n - 1) + [64 + extra], rng)])
        assert_cuts(text, 2, L)
        assert shard_winners(oracle, text, [(0, L), (L, 2 * L)]) == [(1, 3), (n, SLAB_BLOB + extra)]
        m = group(2)
        if extra:
            _refused(m, oracle, text, E_CAPACITY, "outgrow the peer slab")
        else:
            check_sharded(m, oracle, text, queries(oracle, text, 5000, 7))
        check_sharded(m, oracle, pci_text, q)


@pytest.mark.parametrize("nranks,per_rank", [(4, 19661 * 64), (8, SLAB_BLOB)])
def test_merged_blob_growth(nranks, per_rank, group, oracle, pci_text):
    """Four ranks of ~1.2 MiB of names outgrow a fresh group's 4 MiB merged blob: the whole group retries with
    16 MiB.  Eight ranks of exactly 2 MiB fill the grown blob exactly.  Every name is checked afterwards."""
    rng = np.random.default_rng(nranks)
    text, L = padded([block(0x1000 + r, [64] * (per_rank // 64), rng) for r in range(nranks)])
    assert_cuts(text, nranks, L)
    m = group(nranks)
    win = check_sharded(m, oracle, text, queries(oracle, text, 20000, nranks))
    assert [w[1] for w in win] == [per_rank] * nranks
    total = sum((w[1] + 15) // 16 * 16 for w in win)
    assert total > MERGED_BLOB and (nranks == 4 or total == 4 * MERGED_BLOB)
    check_sharded(m, oracle, pci_text, queries(oracle, pci_text, 5000, 8))


def _slice_cases(nranks):
    """(lengths of the key slices in rank order, rank order of the slices, result modes) covering slices of 0, 1,
    1023, 1024, 1025 and 4097 keys at key_offset of every residue mod 4 and nq_total of every residue mod 4."""
    cases = []
    for s in range(4):
        for i, n in enumerate((0, 1, 1023, 1024, 1025, 4097)):
            lens = [0] * nranks
            lens[0], lens[nranks // 2] = s, n
            lens[-1] += 3 + (s + i) % 4
            c = len(cases)
            order = list(range(nranks)) if c % 2 == 0 else list(reversed(range(nranks)))
            modes = ["offset" if (r + c) % 3 == 0 else "aligned" for r in range(nranks)]
            if c % 4 == 1:
                modes[c % nranks] = None
            cases.append((lens, order, modes))
    cases.append(([0] * (nranks - 1) + [5003], list(range(nranks)), ["aligned"] * nranks))  # all keys on the last rank
    return cases


@pytest.mark.parametrize("nranks", [3, 8])
def test_key_slices(nranks, group, oracle, pci_text):
    """join_gather_kernel's vector path (1024 keys at key_offset % 4 == 0) and scalar path, gather_copy_kernel's
    uint4 body and 0-3 word tail, result buffers off a 16-byte boundary (cudaMemcpyAsync) and missing, slices
    handed out in and against rank order; nq_total == 2^21 is accepted, 2^21 + 1 is refused before anything is
    enqueued and the group still works."""
    import kxpu_b200 as K
    from kxpu_b200.binding import E_UNSUPPORTED
    m = group(nranks)
    seen, tails = set(), set()
    for lens, order, modes in _slice_cases(nranks):
        nq = sum(lens)
        offs = np.concatenate([[0], np.cumsum(lens)])
        slices = [None] * nranks
        for k, r in enumerate(order):
            slices[r] = (int(offs[k]), int(offs[k + 1]))
        seen |= {(hi - lo, lo % 4) for lo, hi in slices if hi - lo in (1, 1023, 1024, 1025, 4097)}
        tails.add(nq % 4)
        check_sharded(m, oracle, pci_text, queries(oracle, pci_text, nq, nq), slices=slices, result=modes)
    assert tails == {0, 1, 2, 3} and all((n, s) in seen for n in (1, 1023, 1024, 1025, 4097) for s in range(4))
    q = queries(oracle, pci_text, JOIN_CAP, 21)
    check_sharded(m, oracle, pci_text, q)
    s = Sharded(m, pci_text, np.concatenate([q, q[:1]]))
    try:
        with pytest.raises(K.KxpuError) as e:
            s.join()
        assert e.value.status == E_UNSUPPORTED
        for r in range(nranks):
            assert (s.results(r) == SENTINEL).all(), r
    finally:
        s.free()
    check_sharded(m, oracle, pci_text, q[:777])


def test_exchange_buffers_and_live_tables(group, oracle, pci_text):
    """Different texts one after the other on one group (a consumer reading the other exchange buffer, an old
    phase-A block or stale slab rows gets different bytes), with the tables of load k alive while load k + 1 runs:
    a merge never writes into another load's table."""
    rng = np.random.default_rng(70)
    long_line = b"3333  " + b"x" * 70000 + b"\n\t0003  hidden\n"
    seq = [pci_text, pci_text, pci_text, b"10de  NV\n\t0001  a\n", b"", _big_random_text(rng, 12000, 300, 0.3), pci_text,
           b"1111  one\n\t0001  a\n2222  two\n\t0002  b\n" * 2000 + long_line + b"4444  four\n\t0004  hidden\n" * 50,
           b"".join(block(0x100 + v, [3] * 20000, rng) for v in range(4))]
    m = group(4)
    live = []
    try:
        for i, text in enumerate(seq):
            live.append(Sharded(m, text, queries(oracle, text, 3000, i)))
            live[-1].join()
            for s in live:  # load i - 1, whose tables stayed alive while load i ran, then load i
                s.check(oracle)
            if len(live) == 2:
                live.pop(0).free()
    finally:
        for s in live:
            s.free()


def test_large_global_offsets(group, oracle, pci_text):
    """Every shard's global_base shifted by one constant: offsets cross 2^32 inside a shard, and the last byte sits
    at 2^44 - 2 (the 44-bit anchor of the parse's carry word).  Rows, names, joins and the cut-off all move along."""
    rng = np.random.default_rng(44)
    cut, _ = _cutoff_text(3, 1, 65536, 0)
    texts = [pci_text, _big_random_text(rng, 40000, 50, 0.6), name_length_shards(3), cut]
    m = group(3)
    for text in texts:
        for shift in ((1 << 32) - 1000, (1 << 44) - 1 - len(text)):
            check_sharded(m, oracle, text, queries(oracle, text, 3000, shift & 0xffff), base_shift=shift)


def test_offset_limit_on_one_rank(group, oracle, pci_text):
    """base + n == 2^44 is refused (KXPU_E_UNSUPPORTED) and leaves the group usable; base + n == 2^44 - 1 loads.
    One rank only: a rank that refuses after the epoch bump would leave its peers waiting."""
    import kxpu_b200 as K
    from kxpu_b200.binding import E_UNSUPPORTED
    m = group(1)
    q = queries(oracle, pci_text, 3000, 1)
    s = Sharded(m, pci_text, q, base_shift=(1 << 44) - len(pci_text))
    try:
        with pytest.raises(K.KxpuError) as e:
            s.join()
        assert e.value.status == E_UNSUPPORTED
        assert (s.results(0) == SENTINEL).all()
    finally:
        s.free()
    check_sharded(m, oracle, pci_text, q, base_shift=(1 << 44) - 1 - len(pci_text))
    check_sharded(m, oracle, pci_text, q)


@pytest.mark.parametrize("rch", ["1", "3", "8"])
@pytest.mark.parametrize("scan_w", ["8", "32"])
def test_kernel_variants(rch, scan_w, group, oracle, pci_text, monkeypatch):
    """Range lengths of the parse (KXPU_RCH) and finalize scan widths (KXPU_SCAN_W), read when the group's contexts
    are created."""
    monkeypatch.setenv("KXPU_RCH", rch)
    monkeypatch.setenv("KXPU_SCAN_W", scan_w)
    m = group(3)
    rng = np.random.default_rng(int(rch))
    for text in (pci_text, _big_random_text(rng, 9000, 120, 0.4), name_length_shards(3)):
        check_sharded(m, oracle, text, queries(oracle, text, 3000, int(rch)))
