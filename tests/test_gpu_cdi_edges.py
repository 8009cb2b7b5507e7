"""GPU checks of the CDI spec emit and parse at their edges, for all six layouts and both formats, against the C oracles
and the Python restatements (tests/cdi_edge_cases.py):
  - emit: records that mix the widest and the narrowest fields, kinds of 3, 22, 23 and 63 bytes (both sides of the
    emitter's short / long instantiation split), counts around the 128-device tile; bit-exact, and the sizing call
    returns the length;
  - parse at every tile phase: a widest fragment starting at every offset from 8192 - HALO to 8192 + 16 of the first
    tile boundary, documents ending at every offset of the last HALO + 16 bytes of a tile and the first 32 of the next,
    and one document whose widest fragments start at every offset of a tile (kinds of 22 and 63 bytes);
  - the typed parse over the damaged corpus, verdicts and records equal to pyref_vf_vgpu_cdi.parse;
  - the bdf domain: every refused class in every emit call is KXPU_E_UNSUPPORTED with nothing written, the accepted
    short corpus is emitted as the oracle writes it, and a document carrying a refused bdf does not parse;
  - the decode's look-back (k_cdi_decode, one epoch per call) interleaved with emits on fresh contexts under
    KXPU_SCAN_EPOCH_LIMIT, and as the first look-back call of a fresh context."""
import ctypes as C
import itertools

import numpy as np
import pytest

import cdi_edge_cases as E
import pyref
import pyref_vf_vgpu_cdi as PV
import vf_vgpu_cdi_cases as VC
from kxpu_b200 import binding as B

pytestmark = pytest.mark.gpu

PT = 8192
HALO = {"pci": 512, "cdev": 512, "mdev": 512, "mdev_cdev": 528, "typed": 576, "typed_cdev": 576}
COUNTS = [1, 127, 128, 129, 255, 256, 257, 4097]
GRID = [(layout, fmt) for layout in E.LAYOUTS for fmt in E.FMTS]


def _parse(kx, layout, fmt, kind, doc, offset=0):
    return kx.cdi_parse_raw(fmt, doc, kind, len(doc) // B.CDI_FRAG_MIN + 1, offset=offset, **E.PARSE_HOW[layout])


def _check_parse(kx, layout, fmt, kind, doc, recs, what):
    rc, n, out = _parse(kx, layout, fmt, kind, doc)
    assert (rc, n) == (B.KXPU_OK, len(recs)), (what, rc, kx.L.kxpu_last_error(kx.ctx))
    assert out[:n].tobytes() == recs.tobytes(), what


@pytest.mark.parametrize("layout,fmt", GRID)
@pytest.mark.parametrize("klen", [3, 22, 23, 63])
def test_emit_mixed_widths(kx, layout, fmt, klen):
    kind = E.kind_of(klen)
    fn = getattr(kx.L, E.EMIT_FN[layout])
    phases = set()
    for n in COUNTS:
        recs = E.mixed(layout, n, seed=n * 7 + klen)
        want = E.oracle_doc(layout, fmt, kind, recs)
        if n <= 257:
            assert want == E.pyref_doc(layout, fmt, kind, recs), n
        got = E.gpu_emit(kx, layout, fmt, kind, recs)
        assert got == want, (n, len(got), len(want))
        need = C.c_size_t(0)
        rc = fn(kx.ctx, fmt, kind, recs.ctypes.data, n, None, 0, C.byref(need))
        assert (rc, need.value) == (B.E_NOSPACE, len(want)), n
        if n >= 127:
            phases |= {s % 16 for s in E.starts(fmt, want)}
    assert phases == set(range(16))  # fragments start at every 16-byte phase of the output
    widest = E.widest(layout, 300)
    assert E.gpu_emit(kx, layout, fmt, kind, widest) == E.oracle_doc(layout, fmt, kind, widest)


@pytest.mark.parametrize("layout,fmt", GRID)
@pytest.mark.parametrize("klen", [22, 63])
def test_parse_starts_at_every_phase_of_the_first_tile(kx, layout, fmt, klen):
    """One document per offset: a widest fragment starts at offset t of the document, for every t from 8192 - HALO to
    8192 + 16 (the last starts whose fragment reaches into the halo of tile 0, and the first of tile 1)."""
    kind = E.kind_of(klen)
    offs = range(PT - HALO[layout], PT + 17)
    for t in offs:
        recs, doc, k = E.start_at(layout, fmt, kind, t)
        assert E.starts(fmt, doc)[k] == t and E.fragments(fmt, doc)[k] == E.width(layout, fmt, kind)
        _check_parse(kx, layout, fmt, kind, doc, recs, t)


@pytest.mark.parametrize("layout,fmt", GRID)
@pytest.mark.parametrize("klen", [22, 63])
def test_parse_ends_at_every_phase_around_a_tile_boundary(kx, layout, fmt, klen):
    """One document per length: the document ends at every offset of the last HALO + 16 bytes of tile 0 and the first
    32 of tile 1, its last device a widest one."""
    kind = E.kind_of(klen)
    for end in range(PT - HALO[layout] - 16, PT + 32):
        recs, doc = E.end_at(layout, fmt, kind, end)
        assert len(doc) == end
        _check_parse(kx, layout, fmt, kind, doc, recs, end)


@pytest.mark.parametrize("layout,fmt", GRID)
@pytest.mark.parametrize("klen", [22, 63])
def test_parse_sweep_every_offset_of_a_tile(kx, layout, fmt, klen):
    """One document of 8193 widest-fragment starts that advance by an odd step: a widest fragment starts at every
    offset of a tile, most of them far into the document, in one call; also from host buffers 1 and 15 bytes
    past 16-byte alignment."""
    kind = E.kind_of(klen)
    recs, doc = E.sweep(layout, fmt, kind)
    w = E.width(layout, fmt, kind)
    assert {s % PT for s, f in zip(E.starts(fmt, doc), E.fragments(fmt, doc)) if f == w} == set(range(PT))
    _check_parse(kx, layout, fmt, kind, doc, recs, "sweep")
    for off in (1, 15):
        rc, n, out = _parse(kx, layout, fmt, kind, doc, offset=off)
        assert (rc, n) == (B.KXPU_OK, len(recs)) and out[:n].tobytes() == recs.tobytes(), off


@pytest.mark.parametrize("cdev", [False, True])
@pytest.mark.parametrize("klen", [3, 22, 63])
@pytest.mark.parametrize("fmt", E.FMTS)
def test_typed_parse_damaged_corpus(kx, fmt, klen, cdev):
    kind = E.kind_of(klen)
    layout = "typed_cdev" if cdev else "typed"
    recs, docs = VC.damaged(fmt, kind, cdev)
    accepted = 0
    for name, doc in docs:
        st, want = PV.parse(fmt, doc, kind, cdev)
        rc, n, out = _parse(kx, layout, fmt, kind, doc)
        if st == PV.OK:
            assert (rc, n) == (B.KXPU_OK, len(want)), name
            assert out[:n].tobytes() == want.tobytes(), name
            accepted += 1
        else:
            assert (rc, n) == (B.E_INVALID, -1), (name, rc, n)
    assert accepted >= 3


@pytest.mark.parametrize("fmt", E.FMTS)
def test_layouts_refuse_each_other_widest(kx, fmt):
    """The widest records, 300 devices of each layout with a 63-byte kind: each parser reads its own layout's document
    and refuses the other five."""
    kind = E.kind_of(63)
    docs = {layout: E.gpu_emit(kx, layout, fmt, kind, E.widest(layout, 300)) for layout in E.LAYOUTS}
    for dname, doc in docs.items():
        assert doc == E.oracle_doc(dname, fmt, kind, E.widest(dname, 300))
        for pname in E.LAYOUTS:
            rc, n, out = _parse(kx, pname, fmt, kind, doc)
            if dname == pname:
                assert (rc, n) == (B.KXPU_OK, 300) and out[:n].tobytes() == E.widest(dname, 300).tobytes()
            else:
                assert (rc, n) == (B.E_INVALID, -1), (dname, pname)


REFUSED = [b"1", b"42", b"017", b"0b1", b"0b0101", b"1.5", b".5", b"0.", b"1e3", b"08", b"1.e3", b".5e3",
           b"1234567890123456", b"0000:", b"1:", b"a:", b":", b"0000:c1:00.0:", b"...", b"...a", b"....0000:c1:00"]


@pytest.mark.parametrize("layout", E.LAYOUTS)
def test_refused_bdfs_write_nothing(kx, layout):
    good = E.mixed(layout, 300, seed=11)
    fns = [getattr(kx.L, E.EMIT_FN[layout])] + ([kx.L.kxpu_cdi_emit] if layout == "pci" else [])
    for bdf in REFUSED:
        assert not pyref.bdf_ok(bdf), bdf
        bad = good.copy()
        field = bad["dev"] if layout in ("mdev_cdev", "typed", "typed_cdev") else bad
        field["parent" if E.MDEV[layout] else "bdf"][257] = bdf
        for fmt in E.FMTS:
            assert E.pyref_doc(layout, fmt, b"nvidia.com/gpu", bad) is None
            for fn in fns:
                args = (kx.ctx, fmt) + (() if fn is kx.L.kxpu_cdi_emit else (b"nvidia.com/gpu",))
                out = np.full(1 << 18, 0xA5, np.uint8)
                need = C.c_size_t(12345)
                rc = fn(*args, bad.ctypes.data, len(bad), out.ctypes.data, len(out), C.byref(need))
                assert rc == B.E_UNSUPPORTED, (bdf, fmt)
                assert (out == 0xA5).all() and need.value == 12345, (bdf, fmt)
                rc = fn(*args, bad.ctypes.data, len(bad), None, 0, C.byref(need))  # the sizing call too
                assert rc == B.E_UNSUPPORTED and need.value == 12345, (bdf, fmt)


@pytest.mark.parametrize("layout", E.LAYOUTS)
def test_accepted_short_corpus_in_one_call(kx, layout):
    """Every accepted string of 1..3 bytes over [0-9a-f:.] (and the 4-byte ones in the PCI layout) in one document,
    equal to the oracle's; and that document with one bdf made a refused plain one does not parse."""
    alpha = "0123456789abcdef:."
    top = 4 if layout == "pci" else 3
    good = [s.encode() for n in range(1, top + 1) for s in map("".join, itertools.product(alpha, repeat=n)) if pyref.bdf_ok(s)]
    recs = E.make(layout, good, 7, np.arange(len(good)), 9, 3, b"k")
    for fmt in E.FMTS:
        doc = E.gpu_emit(kx, layout, fmt, b"a/b", recs)
        assert doc == E.oracle_doc(layout, fmt, b"a/b", recs)
        _check_parse(kx, layout, fmt, b"a/b", doc, recs, "corpus")
        one = E.make(layout, [b"0000:c1:00.0", b"a"], 7, [0, 1], 9, 3, b"k")
        doc = E.oracle_doc(layout, fmt, b"a/b", one)
        q = b"bdf: a\n" if fmt == E.FMT_YAML else b'"bdf": "a"'
        assert doc.count(q) == 1
        for bdf in (b"1", b"1.5", b"0b1", b"1e3", b".5"):
            rc, n, _ = _parse(kx, layout, fmt, b"a/b", doc.replace(q, q.replace(b"a", bdf)))
            assert (rc, n) == (B.E_INVALID, -1), (fmt, bdf)
        assert _parse(kx, layout, fmt, b"a/b", doc)[:2] == (B.KXPU_OK, 2)


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


def _script(seed):
    """Emit and parse calls of all six layouts, each spanning at least two tiles (emit: 128 devices, decode: 8192
    bytes), with the expected answers."""
    rng = np.random.default_rng(seed)
    calls = []
    for layout in E.LAYOUTS:
        for fmt in E.FMTS:
            n = int(rng.integers(129, 700))
            kind = E.kind_of(int(rng.choice([3, 22, 63])))
            recs = E.mixed(layout, n, seed=int(rng.integers(0, 1 << 30)))
            doc = E.oracle_doc(layout, fmt, kind, recs)
            assert len(doc) > PT and n > 128
            calls += [("emit", layout, fmt, kind, recs, doc), ("parse", layout, fmt, kind, recs, doc)]
    order = rng.permutation(len(calls))
    return [calls[i] for i in order]


def _run(kx, call, what):
    op, layout, fmt, kind, recs, doc = call
    if op == "emit":
        assert E.gpu_emit(kx, layout, fmt, kind, recs) == doc, what
    else:
        _check_parse(kx, layout, fmt, kind, doc, recs, what)


@pytest.mark.parametrize("limit", ["2", "3", "5"])
def test_interleaved_under_epoch_wrap(fresh, limit):
    """A fresh context with KXPU_SCAN_EPOCH_LIMIT = limit runs three rounds of 24 interleaved emits and parses: the
    epoch wraps every one to four calls, and a stale tile word carrying the running epoch would shift a decode's record
    slots or an emit's offsets."""
    kx = fresh(KXPU_SCAN_EPOCH_LIMIT=limit)
    for r in range(3):
        for i, c in enumerate(_script(100 + r)):
            _run(kx, c, "round %d call %d" % (r, i))


@pytest.mark.parametrize("layout", E.LAYOUTS)
def test_first_call_of_a_fresh_context_is_a_parse(fresh, layout):
    """A context runs emits and parses and is destroyed; a new one (whose state buffer can be the old one's memory,
    holding words of the same epochs) makes a multi-tile parse its first look-back call."""
    script = _script(300)
    old = fresh()
    for i, c in enumerate(script[:12]):
        _run(old, c, "old context, call %d" % i)
    old.close()
    kx = fresh()
    first = next(c for c in _script(301) if c[0] == "parse" and c[1] == layout)
    _run(kx, first, "first call")
