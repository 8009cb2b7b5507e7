"""SURVEY 8(f) row 4: subsystem rows and the class / subclass / prog-if section, GPU vs oracle (kxo_full_build, itself
pinned by the Python restatement pyref_full.py in test_oracle.py)."""
import numpy as np
import pytest

import full_texts as F
from kxpu_b200.binding import E_INVALID, KxpuError

pytestmark = pytest.mark.gpu

T_RESOLVE = 7  # kxpu.h KXPU_T_RESOLVE: nonzero only when the big-text kernels built the (vendor,device) table
EDGE_PROBES = np.array([0, 1, 65535, 65536, 1 << 24, 1 << 63, (1 << 64) - 2, (1 << 64) - 1], np.uint64)


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


def wrong_kind_keys(rows):
    """keys shaped like the rows of `rows` (kind -> oracle rows) that no lookup of any kind may find: vendor ids past
    16 bits, class keys with nonzero low 16 bits, subclass keys with nonzero low 8 bits, type bytes 0 and >= 4"""
    v = rows[0]["key"][:64].astype(np.uint64)
    k2 = rows[2]["key"].astype(np.uint64)
    typ = k2 >> np.uint64(24)
    cls, sub = k2[typ == 1][:64], k2[typ == 2][:64]
    low = k2 & np.uint64(0xffffff)
    out = [v | np.uint64(1 << 16), v | np.uint64(1 << 40), cls | np.uint64(1), cls | np.uint64(0x100), cls | np.uint64(0x8000),
           sub | np.uint64(1), sub | np.uint64(0x80), low[:64]]
    out += [low[:64] | np.uint64(t << 24) for t in (4, 5, 0xff)] + [k2[:64] | np.uint64(1 << 32)]
    return np.concatenate(out)


def check_full(kx, oracle, text, tail=b"", join=False, extra=()):
    """The (vendor,device) table and all three row kinds of the full model on `text` against the oracle: the export,
    and lookups of sampled rows, their neighbours, the rows of the other kinds, malformed keys and `extra` keys.
    `tail` follows the text in the device buffer, behind n = len(text): nothing may read it.  join: the table comes
    from kxpu_pciids_join_device instead of kxpu_pciids_load_device."""
    buf = np.frombuffer(text + tail, np.uint8)
    n = len(text)
    d = kx.dev_alloc(max(len(buf), 16))
    if len(buf):
        kx.upload(d, buf)
    orows = oracle.table_build(text)
    d_q = d_r = None
    if join:
        q = np.concatenate([orows["key"][::7], np.array([0, 0xffffffff, 0x12340001], np.uint32)]).astype(np.uint32)
        d_q, d_r = kx.dev_alloc(q.nbytes), kx.dev_alloc(q.nbytes)
        kx.upload(d_q, q)
        tab = kx.pciids_join_device(d, n, d_q, len(q), d_r)
    else:
        tab = kx.pciids_load_device(d, n)
    full = kx.full_load_device(d, n, tab)
    try:
        keys, offs, _ = kx.table_export(tab)
        assert np.array_equal(keys, orows["key"]) and np.array_equal(offs, orows["line_off"]), "(vendor,device) table"
        want = {kind: oracle.full_build(text, kind) for kind in (0, 1, 2)}
        others = np.concatenate([want[k]["key"][:: max(1, len(want[k]) // 200)] for k in (0, 1, 2)]).astype(np.uint64)
        for kind in (0, 1, 2):
            w = want[kind]
            keys, offs = kx.full_export(full, kind)
            assert np.array_equal(keys, w["key"]) and np.array_equal(offs, w["line_off"]), kind
            pick = w["key"][:: max(1, len(w) // 400)].astype(np.uint64)
            q = np.concatenate([pick, pick ^ np.uint64(1 << 5), EDGE_PROBES, others, wrong_kind_keys(want),
                                np.asarray(extra, np.uint64)])
            got = kx.full_lookup(full, kind, q)
            table = dict(zip(w["key"].tolist(), w["line_off"].tolist()))
            exp = np.array([table.get(int(k), -1) for k in q], np.int64)
            assert np.array_equal(got, exp), kind
    finally:
        kx.full_free(full)
        tab.free()
        for p in (d, d_q, d_r):
            if p is not None:
                kx.dev_free(p)


def test_real_pci_ids_full_model(kx, oracle, pci_text):
    want = [len(oracle.full_build(pci_text, k)) for k in (0, 1, 2)]
    assert want == [2388, 16297, 210]  # SURVEY.md 8(a) A0: vendors, subsystem lines, 22 + 114 + 74 class-section lines
    check_full(kx, oracle, pci_text)


def test_full_model_first_occurrence_and_edges(kx, oracle, pci_text, workloads):
    cut = pci_text.find(b"\n", 1400000) + 1
    check_full(kx, oracle, pci_text * 2)                         # every block twice: the first copy wins at every level
    check_full(kx, oracle, pci_text[700000:cut] + pci_text)      # later vendors first, class section twice
    for t in F.EDGE_TEXTS:
        check_full(kx, oracle, t)
    # lines whose governing lines sit one or many 2 KiB chunks back
    big = b"abcd  Vendor\n\t0001  dev\n" + b"".join(b"\t\t%04x %04x  subsystem number %d\n" % (i >> 8, i & 0xffff, i) for i in range(9000))
    big += b"C ff  class\n\t01  sub\n" + b"".join(b"\t\t%02x  prog-if %d\n" % (i & 0xff, i) for i in range(400))
    check_full(kx, oracle, big)
    # more subsystem rows than the first subsystem hash table (2^17 slots) and more prog-if rows than the first
    # prog-if table (2^12 slots) hold: both are grown x4 and built again
    text = workloads.synthetic_pci_ids(512, 64, subs_per_dev=8).tobytes()
    classes = b"".join(b"C %02x  Class %d\n\t%02x  Subclass\n" % (c, c, c) + b"".join(b"\t\t%02x  Prog-if %d\n" % (p, p) for p in range(256))
                       for c in range(20))
    text += classes
    assert len(oracle.full_build(text, 1)) == 262144 > (1 << 17)
    progifs = oracle.full_build(text, 2)
    assert int(((progifs["key"] >> np.uint64(24)) == 3).sum()) == 5120 > (1 << 12)
    check_full(kx, oracle, text)


def test_full_model_all_ones_subsystem_key(kx, oracle):
    """\\t\\tffff ffff under device ffff of vendor ffff has the key 2^64 - 1, the hash table's empty-slot marker: it
    lives in a slot of its own, and the keys around it keep their own lines."""
    want = oracle.full_build(F.ALL_ONES, 1)
    assert want["key"].tolist() == F.ALL_ONES_KEYS and want["line_off"].tolist() == F.ALL_ONES_OFFS
    check_full(kx, oracle, F.ALL_ONES)
    check_full(kx, oracle, F.ALL_ONES + F.ALL_ONES.replace(b"  ", b"  dup "))  # a later ffff block loses


def test_full_model_all_ones_first_then_200k_keys(kx, oracle):
    """The all-ones block first, then 200 000 subsystem keys, among them keys whose home slot is the all-ones key's
    own in the first (2^17) and the grown (2^19) table: they probe through the slot that ~0 taken for an ordinary
    key would have marked with its earlier line."""
    text = F.all_ones_first()
    want = oracle.full_build(text, 1)
    assert len(want) > 200000 > (1 << 17) and want["key"][0] == (1 << 64) - 1
    check_full(kx, oracle, text)


def test_full_model_cutoff(kx, oracle):
    """A line of 65 535 bytes is kept; one of 65 536 (or 65 535 and a '\\r') ends the scan.  Rows behind the cut
    leave the export and the lookup of every kind: the lookups probe every row of the same text without the cut."""
    for text, uncut, kept in F.cutoff_texts():
        extra = np.concatenate([oracle.full_build(uncut, k)["key"] for k in (0, 1, 2)])
        got = sum(len(oracle.full_build(text, k)) for k in (0, 1, 2))
        assert (got == len(extra)) == kept
        check_full(kx, oracle, text, extra=extra)


def test_full_model_chunk_seams(kx, oracle):
    """Every line kind with its head on every offset within 41 bytes of a 2 KiB chunk boundary; governing lines 31,
    32, 33, 64 and 65 chunks in front of their rows (the look-back reads 32 chunk summaries per round); texts of
    2048 k - 1, 2048 k and 2048 k + 1 bytes."""
    text = F.seam_text()
    assert len(oracle.full_build(text, 0)) > 256
    check_full(kx, oracle, text)
    for t in F.lookback_texts() + F.length_texts():
        assert len(oracle.full_build(t, 1)) + len(oracle.full_build(t, 2)) > 0
        check_full(kx, oracle, t)


@pytest.mark.parametrize("path", ["small", "big"])
def test_full_model_both_load_paths(path, fresh, oracle, pci_text, workloads):
    """The full model reads the (vendor,device) table's vendor_first, slots and cut-off directly: on tables from the
    cooperative small-text kernel and from the big-text kernels (KXPU_NO_SMALL=1), one of them grown past the 2^16
    slots a fresh context starts with."""
    kx = fresh(**({"KXPU_NO_SMALL": "1"} if path == "big" else {}))
    d = kx.dev_alloc(len(pci_text))
    kx.upload(d, np.frombuffer(pci_text, np.uint8))
    kx.pciids_load_device(d, len(pci_text)).free()
    assert (kx.timings()[T_RESOLVE] == 0) == (path == "small")
    kx.dev_free(d)
    grown = workloads.synthetic_pci_ids(1024, 70, subs_per_dev=1).tobytes()
    assert len(oracle.table_build(grown)) == 71680 > (1 << 16)
    cut = F.cutoff_texts()
    for t in (pci_text, F.ALL_ONES, F.seam_text(), cut[0][0], cut[4][0], cut[11][0], grown):
        check_full(kx, oracle, t)


def test_full_model_on_joined_table(kx, oracle, pci_text):
    cut = F.cutoff_texts()
    for t in (pci_text, F.ALL_ONES, F.seam_text(), cut[1][0], cut[5][0]):
        check_full(kx, oracle, t, join=True)


POISON = [b"d  V\n\t0001  d\n\t\tffff ffff  x\n", b"\t\tffff ffff  x\n\t\t07  p\n\t0001  d\nC 01\n", b"\t0001  d\n\t\t1111 2222  y\n"]
ENDS = [b"abc", b"1234  V\n\t0001  D\n", b"C 05  K\n\t06  SC\n"]


def test_full_model_poisoned_tail(kx, oracle):
    """The bytes behind n in the device buffer hold lines that would change the answer if they were read (and hex
    digits that would complete an unterminated vendor line `abc` at n): the table and the full model equal the
    oracle on text[:n].  n a multiple of 2048, of 16 only, and of neither."""
    head = b"5678  W\n\t0002  E\n\t\t1111 2222  s\n"
    for n in (64, 4096, 4112, 6143, 6149, 10240):
        for end in ENDS:
            text = head + F.pad_to(len(head), n - len(end)) + end
            assert len(text) == n
            for poison in POISON:
                check_full(kx, oracle, text, tail=poison * (4096 // len(poison) + 2))


def test_full_model_lookup_of_the_wrong_kind(kx, oracle, pci_text):
    """Keys of another kind, or malformed for their kind, find nothing; kinds other than 0, 1, 2 are invalid."""
    rows = {k: oracle.full_build(pci_text, k) for k in (0, 1, 2)}
    buf = np.frombuffer(pci_text, np.uint8)
    d = kx.dev_alloc(len(buf))
    kx.upload(d, buf)
    tab = kx.pciids_load_device(d, len(buf))
    full = kx.full_load_device(d, len(buf), tab)
    try:
        bad = wrong_kind_keys(rows)
        probes = {0: np.concatenate([bad[bad >= 65536], np.array([65536, 65536 + 0x10de, (1 << 32) | 0x10de], np.uint64)]),
                  1: np.concatenate([bad, rows[0]["key"], rows[2]["key"]]).astype(np.uint64),
                  2: np.concatenate([bad, rows[0]["key"][rows[0]["key"] > 0]]).astype(np.uint64)}
        for kind, q in probes.items():
            assert not set(q.tolist()) & set(rows[kind]["key"].tolist())
            assert (kx.full_lookup(full, kind, q) == -1).all(), kind
        for kind in (-1, 3):
            with pytest.raises(KxpuError) as e:
                kx.full_export(full, kind)
            assert e.value.status == E_INVALID
            with pytest.raises(KxpuError) as e:
                kx.full_lookup(full, kind, rows[0]["key"][:4])
            assert e.value.status == E_INVALID
    finally:
        kx.full_free(full)
        tab.free()
        kx.dev_free(d)


def test_full_model_fuzz(kx, oracle):
    rng = np.random.default_rng(12)
    pool = [b"%04x  V\n", b"\t%04x  D\n", b"\t\t%04x %04x  S\n", b"C %02x  K\n", b"\t%02x  SC\n", b"\t\t%02x  PI\n", b"# c\n", b"\n", b"zz\n", b"\t\n",
            b"\t\t\n", b"%04X  V\n", b"\t%04x  D\r\n", b"\t\t%04x %04X  S\r\n", b"C %02X  K\r\n", b"\t\t%02x  PI\r\n", b"\r\n"]
    ids = [0, 1, 2, 3, 4, 5, 0xff, 0xabcd, 0xfffe, 0xffff]
    for trial in range(40):
        parts = []
        for _ in range(int(rng.integers(1, 2500))):
            f = pool[int(rng.integers(0, len(pool)))]
            k = f.count(b"%")
            two = b"%02" in f
            parts.append(f % tuple(ids[int(rng.integers(0, len(ids)))] & (0xff if two else 0xffff) for _ in range(k)) if k else f)
        check_full(kx, oracle, b"".join(parts))
