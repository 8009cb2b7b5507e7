"""CPU checks of the CDI spec emit and parse at their edges, for all six layouts (group, cdev, mdev, mdev cdev, typed,
typed cdev) and both formats:
  - the widest fragment of every layout, format and kind length fits the tile bound of the kernel instantiation the
    emitter picks for it, and, with the start pattern, the parse's halo for the layout (the constants restated here are
    checked against the sources);
  - the shortest fragment is at least KXPU_CDI_FRAG_MIN;
  - the bdf domain: every short string over [0-9a-f:.] is accepted or refused alike by the Python predicate, the C
    checker and every emitter restatement, and YAML reads every accepted bdf back as the same string;
  - the typed parse's restatement (pyref_vf_vgpu_cdi.parse) over a damaged-document corpus;
  - the edge-case generators place what they promise (the GPU tests rely on them)."""
import itertools
import json
import os
import re

import numpy as np
import pytest
import yaml

import cdi_edge_cases as E
import pyref
import pyref_vf_vgpu_cdi as PV
import vf_vgpu_cdi_cases as VC
from conftest import ROOT

CSRC = os.path.join(ROOT, "kata-xpu-device-plugin_b200", "csrc")
KIND_LENS = [3, 21, 22, 23, 62, 63]
# emit.cu: the fragment bound of each k_cdi_fused instantiation (short kinds, long kinds); cdi_parse.cu: HALO<LAYOUT>
MAX_FRAG, MAX_FRAG_LONG, MAX_FRAG_MDEV, CDEV_EXTRA, TYPED_EXTRA = 368, 416, 480, 12, 104
BOUNDS = {"pci": (MAX_FRAG, MAX_FRAG_LONG), "cdev": (MAX_FRAG + CDEV_EXTRA, MAX_FRAG_LONG + CDEV_EXTRA),
          "mdev": (MAX_FRAG_MDEV, MAX_FRAG_MDEV), "mdev_cdev": (MAX_FRAG_MDEV + CDEV_EXTRA, MAX_FRAG_MDEV + CDEV_EXTRA),
          "typed": (MAX_FRAG + TYPED_EXTRA, MAX_FRAG_LONG + TYPED_EXTRA),
          "typed_cdev": (MAX_FRAG + CDEV_EXTRA + TYPED_EXTRA, MAX_FRAG_LONG + CDEV_EXTRA + TYPED_EXTRA)}
HALO = {"pci": 512, "cdev": 512, "mdev": 512, "mdev_cdev": 528, "typed": 576, "typed_cdev": 576}
PAT_MAX, PT = 32, 8192
FRAG_MIN = 166


def test_constants_match_the_sources():
    emit = open(os.path.join(CSRC, "emit.cu")).read()
    cdi = open(os.path.join(CSRC, "cdi.cuh")).read()
    parse = open(os.path.join(CSRC, "cdi_parse.cu")).read()
    for pat in (r"constexpr int MAX_FRAG = 368;", r"constexpr int MAX_FRAG_LONG = 416;", r"constexpr int MAX_FRAG_MDEV = 480;",
                r'#define KX_CDEV_NODE "devices/vfio"', r"constexpr int MAX_FRAG_MDEV_CDEV = MAX_FRAG_MDEV \+ CDEV_EXTRA;",
                r"constexpr int TYPED_EXTRA = \(int\)sizeof\(KX_JV4 KX_JV9\) - 1 \+ 10 \+ 40;  // 104",
                r"constexpr int MAX_FRAG_TYPED = MAX_FRAG \+ TYPED_EXTRA, MAX_FRAG_TYPED_LONG = MAX_FRAG_LONG \+ TYPED_EXTRA;",
                r"constexpr int MAX_FRAG_TYPED_CDEV = MAX_FRAG_CDEV \+ TYPED_EXTRA, MAX_FRAG_TYPED_CDEV_LONG = MAX_FRAG_CDEV_LONG \+ TYPED_EXTRA;",
                # the host's estimate of a call's longest fragment, which picks the instantiation
                r"const uint32_t frag = E\.lit_total \+ 2 \* 20 \+ 2 \* 10 \+ 15 \+ 2 \+ 2 \+ \(mdev \? 36 : 0\) \+ \(typed \? 10 \+ 40 : 0\);"):
        assert re.search(pat, emit), pat
    for pat in (r"KX_CDI_FRAG_MAX = 480;", r"KX_CDI_FRAG_MAX_MDEV_CDEV = KX_CDI_FRAG_MAX \+ 12;", r"KX_CDI_FRAG_MAX_TYPED = 532;"):
        assert re.search(pat, cdi), pat
    for pat in (r"constexpr int PT = 8192;", r"constexpr int PAT_MAX = 32;",
                r"HALO = is_typed_layout<LAYOUT> \? 576 : LAYOUT == LAYOUT_MDEV_CDEV \? 528 : 512;"):
        assert re.search(pat, parse), pat
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert "#define KXPU_CDI_FRAG_MIN %d" % FRAG_MIN in hdr


def _longest_fields(layout, fmt):
    """What the longest fields add to a fragment: the name twice, the group and the group or N, the bdf (YAML: base-60
    quoted), the JSON separator, the uuid, the type ID and the key."""
    return (2 * 20 + 2 * 10 + (18 if fmt == E.FMT_YAML else 16 + 2) + (36 if E.MDEV[layout] else 0)
            + (10 + 40 if E.TYPED[layout] else 0))


@pytest.mark.parametrize("layout", E.LAYOUTS)
@pytest.mark.parametrize("fmt", E.FMTS)
def test_widest_fragment_fits_tile_and_halo(layout, fmt):
    """For every kind length, the widest fragment (restatement and C oracle agree on it) fits the bound of the
    instantiation the emitter's host code picks, and the fragment plus the start pattern fits the parse's halo."""
    seen = {}
    for klen in KIND_LENS:
        kind = E.kind_of(klen)
        recs = E.widest(layout, 3)
        doc = E.oracle_doc(layout, fmt, kind, recs)
        assert doc == E.pyref_doc(layout, fmt, kind, recs)
        frags = E.fragments(fmt, doc)
        w = max(frags)
        assert frags[0] == w == frags[1] and frags[2] == w - (1 if fmt == E.FMT_JSON else 0)
        lits = w - _longest_fields(layout, fmt)
        est = lits + 2 * 20 + 2 * 10 + 15 + 2 + 2 + (36 if E.MDEV[layout] else 0) + (50 if E.TYPED[layout] else 0)
        short, long_ = BOUNDS[layout]
        bound = long_ if est > short else short
        assert w <= est <= bound, (klen, w, est, bound)  # est > bound would be a call refused as KXPU_E_INVALID
        assert w + PAT_MAX <= HALO[layout], (klen, w)
        seen[klen] = (w, bound)
    if fmt == E.FMT_JSON and layout in ("pci", "cdev", "typed", "typed_cdev"):
        # the 22-byte kinds are the last on the short instantiation, one byte inside it
        assert seen[22][1] == BOUNDS[layout][0] and seen[22][0] == BOUNDS[layout][0] - 1
        assert seen[23][1] == BOUNDS[layout][1]


@pytest.mark.parametrize("layout", E.LAYOUTS)
@pytest.mark.parametrize("fmt", E.FMTS)
def test_shortest_fragment_is_at_least_frag_min(layout, fmt):
    for kind in (b"a/b", E.kind_of(22), E.kind_of(63)):
        recs = E.narrowest(layout, 12)
        doc = E.oracle_doc(layout, fmt, kind, recs)
        assert doc == E.pyref_doc(layout, fmt, kind, recs)
        shortest = min(E.fragments(fmt, doc))
        assert shortest >= FRAG_MIN
        if (layout, fmt, kind) == ("pci", E.FMT_YAML, b"a/b"):
            assert shortest == FRAG_MIN
        assert len(doc) // FRAG_MIN >= len(recs)


def _short_corpus():
    """Every string of 1..4 bytes over [0-9a-f:.], then seeded ones of 5..16 bytes drawn so that every refused class
    occurs at every length."""
    alpha = "0123456789abcdef:."
    out = ["".join(t) for n in range(1, 5) for t in itertools.product(alpha, repeat=n)]
    rng = np.random.default_rng(7)
    for n in range(5, 17):
        for sub in (alpha, "0123456789", "0123456789.", "0123456789.e", "01"):
            for _ in range(150):
                s = "".join(rng.choice(list(sub), n))
                out += [s, "0b" + s[2:], s[:-1] + ":", "..." + s[3:], "." + s[1:]]
    return list(dict.fromkeys(out))


@pytest.fixture(scope="module")
def corpus():
    c = _short_corpus()
    return c, [pyref.bdf_ok(s) for s in c]


def test_bdf_domain_classes(corpus):
    """The predicate refuses exactly the five classes, and a plain one-byte bdf stays inside."""
    strings, ok = corpus
    cls = [re.compile(p) for p in (r"[0-9]+", r"0b[01]+", r"[0-9]+(\.[0-9]*)?(e[0-9]+)?|\.[0-9]+(e[0-9]+)?", r".*:", r"\.\.\..*")]
    hits = [0] * len(cls)
    for s, good in zip(strings, ok):
        m = [bool(c.fullmatch(s)) for c in cls]
        assert good == (not any(m)), s
        hits = [h + x for h, x in zip(hits, m)]
    assert all(h > 100 for h in hits), hits
    for s in ("1", "42", "017", "0b1", "1.5", ".5", "0.", "1e3", "08", "0000:", "1:", "a:", ":", "...", "...a"):
        assert not pyref.bdf_ok(s), s
    for s in ("a", "0000:c1:00.0", "0000:01:00.0", "1e", ".", "..", "0b", "0b2", "1.5.", ".e3", ":a", "a:b", "0000:01:02.34567"):
        assert pyref.bdf_ok(s), s


def test_bdf_domain_checkers_agree_and_yaml_reads_strings(corpus):
    """The C checker refuses exactly what the predicate refuses, one string at a time; every restatement refuses a
    document holding one; the accepted corpus, as bdf and as mdev parent, is one document per layout on which the C
    oracle and the restatement agree, and which PyYAML (YAML 1.1, as CDI loaders built on goyaml.v2 read it) and json
    read back with every bdf the same str."""
    strings, ok = corpus
    enc = [s.encode() for s in strings]
    typed = E.make("typed", enc, 5, np.arange(len(enc)), 0, 1, b"k")
    for i, good in enumerate(ok):
        assert (E.oracle_doc("typed", E.FMT_YAML, b"a/b", typed[i:i + 1]) is not None) == good, strings[i]
    bad = [i for i, g in enumerate(ok) if not g]
    for layout in E.LAYOUTS:
        for i in bad[::97]:
            one = E.make(layout, [enc[i]], 5, [0], 1)
            for fmt in E.FMTS:
                assert E.pyref_doc(layout, fmt, b"a/b", one) is None, (layout, strings[i])
    good = [s for s, g in zip(enc, ok) if g]
    loader = getattr(yaml, "CSafeLoader", yaml.SafeLoader)  # libyaml's parser, PyYAML's YAML 1.1 resolver either way
    for layout in E.LAYOUTS:
        # the whole accepted corpus in the group layout, a sample in the others (as bdf and as mdev parent)
        part = good if layout == "pci" else good[::7]
        recs = E.make(layout, part, 5, np.arange(len(part)), 3, 1, b"k")
        for fmt in E.FMTS:
            doc = E.oracle_doc(layout, fmt, b"a/b", recs)
            assert doc == E.pyref_doc(layout, fmt, b"a/b", recs), layout
            spec = yaml.load(doc, Loader=loader) if fmt == E.FMT_YAML else json.loads(doc)
            back = [d["annotations"]["bdf"] for d in spec["devices"]]
            assert back == [s.decode() for s in part], layout
    # and the refused corpus, written the way the emitters would write it, is not read back as its own string
    lost, sample = 0, bad[::37]
    for i in sample:
        s = strings[i]
        v = '"%s"' % s if pyref.BASE60.match(s) else s
        try:
            lost += yaml.load("bdf: %s\n" % v, Loader=loader)["bdf"] != s
        except yaml.YAMLError:
            lost += 1
    assert lost > len(sample) // 2


@pytest.mark.parametrize("cdev", [False, True])
@pytest.mark.parametrize("kind", [b"a/b", E.kind_of(22), E.kind_of(63)])
@pytest.mark.parametrize("fmt", E.FMTS)
def test_typed_parse_restatement(fmt, kind, cdev):
    """pyref_vf_vgpu_cdi.parse reads the C oracle's documents back exactly and returns the expected verdicts on the
    damaged corpus; whatever it accepts, the oracle writes byte for byte."""
    recs, docs = VC.damaged(fmt, kind, cdev)
    verdict = {}
    for name, doc in docs:
        st, got = PV.parse(fmt, doc, kind, cdev)
        verdict[name] = st
        if st == PV.OK:
            assert E.oracle_doc("typed_cdev" if cdev else "typed", fmt, kind, got) == doc, name
    assert verdict["clean"] == PV.OK and verdict["zero_devices"] == PV.OK
    assert PV.parse(fmt, docs[0][1], kind, cdev)[1].tobytes() == recs.tobytes()
    named = [k for k in verdict if not k.startswith(("flip", "truncate")) and k not in ("clean", "zero_devices")]
    for name in named:
        want = PV.OK if name == "duplicated_fragment" or (name == "duplicated_last" and fmt == E.FMT_YAML) else PV.E_INVALID
        assert verdict[name] == want, name
    cuts = set(VC.CP.boundaries(fmt, docs[0][1])[1:-1]) if fmt == E.FMT_YAML else set()
    for k, v in verdict.items():
        if k.startswith("truncate@"):
            assert v == (PV.OK if int(k[9:]) in cuts else PV.E_INVALID), k
    assert sum(v == PV.E_INVALID for v in verdict.values()) > 100
    assert PV.parse(fmt, docs[0][1], b"example.com/other", cdev)[0] == PV.E_INVALID
    assert PV.parse(fmt, docs[0][1], b"no-slash", cdev)[0] == PV.E_UNSUPPORTED
    assert PV.parse(fmt, docs[0][1], kind, not cdev)[0] == PV.E_INVALID


@pytest.mark.parametrize("fmt", E.FMTS)
def test_typed_parse_restatement_reads_widest_and_mixed(fmt):
    for cdev in (False, True):
        layout = "typed_cdev" if cdev else "typed"
        for recs in (E.widest(layout, 5), E.mixed(layout, 300, 3), E.narrowest(layout, 20)):
            for kind in (b"a/b", E.kind_of(63)):
                st, got = PV.parse(fmt, E.oracle_doc(layout, fmt, kind, recs), kind, cdev)
                assert st == PV.OK and got.tobytes() == recs.tobytes()


@pytest.mark.parametrize("layout", E.LAYOUTS)
def test_generators_place_what_they_promise(layout):
    """start_at / end_at / sweep (the GPU phase sweep's documents) for one format and kind: the C oracle and the
    restatement agree, starts and ends fall where asked, and the sweep puts a widest start at every offset of a tile."""
    fmt, kind = E.FMT_JSON, E.kind_of(63)
    w = E.width(layout, fmt, kind)
    for off in (PT - HALO[layout], PT - 1, PT, PT + 16):
        recs, doc, k = E.start_at(layout, fmt, kind, off)
        assert E.fragments(fmt, doc)[k] == w and doc == E.pyref_doc(layout, fmt, kind, recs)
    for end in (PT - HALO[layout] - 16, PT, PT + 31):
        recs, doc = E.end_at(layout, fmt, kind, end)
        assert len(doc) == end
    recs, doc = E.sweep(layout, fmt, kind)
    s, f = E.starts(fmt, doc), E.fragments(fmt, doc)
    assert {a % PT for a, n in zip(s, f) if n == w} == set(range(PT))
