"""GPU tests of kxpu_vf_vgpu_drift against the C oracle (tests/vf_vgpu_health_oracle.c) and the Python restatement:
seeded inputs up to 2^20 records and groups, every current-type text edge, empty and one-member groups, drifted members
that are not the first, shared members, and every refusal with nothing written."""
import numpy as np
import pytest

import pyref_vf_vgpu_health as P
import vf_vgpu_health_oracle as O
from kxpu_b200 import binding as B
from test_vf_vgpu_health import EDGES, rec

pytestmark = pytest.mark.gpu


def _eq(got, want):
    assert want is not None
    assert {k: v.tolist() for k, v in got.items()} == want


def _seeded(n, n_groups, seed, drift_every=64):
    rng = np.random.default_rng(seed)
    recs = np.zeros(n, B.VFVGPUREC_DTYPE)
    was = rng.choice(np.array([557, 558, 559, 4294967295], np.uint32), n)
    texts = {int(t): np.frombuffer((b"%d\n" % t).ljust(16, b"\0"), np.uint8) for t in (557, 558, 559, 4294967295)}
    for t, row in texts.items():
        m = was == t
        recs["cur_txt"][m] = row
        recs["cur_len"][m] = len(b"%d\n" % t)
    recs["flags"] = B.VT_READ
    d = np.flatnonzero(rng.random(n) < 1.0 / drift_every)  # about 1 in 64 drifted: cleared, changed or unreadable
    kind = rng.integers(0, 3, len(d))
    for i, k in zip(d, kind):
        txt = [b"0\n", b"560\n", b"0560\n"][k]
        recs["cur_txt"][i] = np.frombuffer(txt.ljust(16, b"\0"), np.uint8)
        recs["cur_len"][i] = len(txt)
    recs["flags"][d[kind == 2][::2]] |= B.VT_CUR_ERR
    sizes = rng.integers(0, 3, n_groups)  # empty, one- and two-member groups
    goff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    gmem = rng.integers(0, n, int(goff[-1])).astype(np.uint32)
    return recs, was, goff, gmem


@pytest.mark.parametrize("n", [1, 255, 256, 257, 4097, 1 << 20])
def test_seeded_against_oracle(kx, n):
    recs, was, goff, gmem = _seeded(n, n, 15 + n)
    want = O.vf_vgpu_drift(recs, was, goff, gmem)
    _eq(kx.vf_vgpu_drift(recs, was, goff, gmem), want)
    if n <= 4097:
        assert P.vf_vgpu_drift(recs, was, goff.tolist(), gmem.tolist()) == want


def test_text_edges(kx):
    recs = np.concatenate([rec(t) for t, _, _, _ in EDGES])
    was = [w for _, w, _, _ in EDGES]
    n = len(EDGES)
    goff, gmem = np.arange(n + 1, dtype=np.uint32), np.arange(n, dtype=np.uint32)
    got = kx.vf_vgpu_drift(recs, was, goff, gmem)
    assert got["status_now"].tolist() == [s for _, _, s, _ in EDGES]
    assert got["type_now"].tolist() == [t for _, _, _, t in EDGES]
    _eq(got, O.vf_vgpu_drift(recs, was, goff, gmem))


def test_group_shapes(kx):
    """empty groups, one-member groups, a late drifted member in a group of more than 32 members (past the first lane
    round), shared members, and records no group names"""
    n = 200
    recs = np.concatenate([rec(b"557\n")] * n)
    was = np.full(n, 557, np.uint32)
    recs["cur_txt"][150] = np.frombuffer(b"0\n".ljust(16, b"\0"), np.uint8)
    recs["cur_len"][150] = 2
    recs["flags"][170] |= B.VT_CUR_ERR
    groups = [[], [0], [150], list(range(100)) + [150, 170], [], list(range(140, 180)), [170, 150], [199]]
    goff = np.concatenate([[0], np.cumsum([len(g) for g in groups])]).astype(np.uint32)
    gmem = np.array([m for g in groups for m in g], np.uint32)
    got = kx.vf_vgpu_drift(recs, was, goff, gmem)
    assert got["group_first"].tolist() == [P.STEADY, P.STEADY, 0, 100, P.STEADY, 10, 0, P.STEADY]
    _eq(got, O.vf_vgpu_drift(recs, was, goff, gmem))


def test_no_records_or_no_groups(kx):
    recs = np.concatenate([rec(b"0\n"), rec(b"557\n")])
    _eq(kx.vf_vgpu_drift(recs, [557, 557], [0], []), O.vf_vgpu_drift(recs, [557, 557], [0], []))
    _eq(kx.vf_vgpu_drift(recs[:0], [], [0, 0, 0], []), dict(type_now=[], status_now=[], group_first=[P.STEADY] * 2))


def _raw(kx, recs, was, goff, gmem, now, st, first, n=None, G=None):
    n = 2 if n is None else n
    G = 2 if G is None else G
    p = lambda a: None if a is None else a.ctypes.data
    return kx.L.kxpu_vf_vgpu_drift(kx.ctx, p(recs), p(was), n, p(goff), p(gmem), G, p(now), p(st), p(first))


def test_refusals_write_nothing(kx):
    recs = np.concatenate([rec(b"0\n"), rec(b"558\n")])
    was = np.array([557, 557], np.uint32)
    goff, gmem = np.array([0, 1, 2], np.uint32), np.array([0, 1], np.uint32)

    def outs():
        return np.full(2, 7, np.uint32), np.full(2, 9, np.uint8), np.full(2, 11, np.uint32)

    cases = [
        (dict(recs=None), B.E_INVALID), (dict(was=None), B.E_INVALID), (dict(now=None), B.E_INVALID),
        (dict(st=None), B.E_INVALID), (dict(goff=None), B.E_INVALID), (dict(gmem=None), B.E_INVALID),
        (dict(first=None), B.E_INVALID), (dict(goff=np.array([0, 2, 1], np.uint32)), B.E_INVALID),
        (dict(gmem=np.array([0, 2], np.uint32)), B.E_INVALID), (dict(n=1 << 28), B.E_UNSUPPORTED),
        (dict(G=1 << 28), B.E_UNSUPPORTED),
    ]
    for over, rc in cases:
        now, st, first = outs()
        a = dict(recs=recs, was=was, goff=goff, gmem=gmem, now=now, st=st, first=first)
        a.update(over)
        assert _raw(kx, **a) == rc, over
        assert now.tolist() == [7, 7] and st.tolist() == [9, 9] and first.tolist() == [11, 11], over
    assert kx.L.kxpu_vf_vgpu_drift(None, recs.ctypes.data, was.ctypes.data, 2, goff.ctypes.data, gmem.ctypes.data, 2,
                                   *[o.ctypes.data for o in outs()]) == B.E_INVALID
    now, st, first = outs()
    assert _raw(kx, recs, was, goff, gmem, now, st, first) == B.KXPU_OK
    assert st.tolist() == [P.CLEARED, P.CHANGED] and now.tolist() == [0, 558] and first.tolist() == [0, 0]


def test_one_launch_timed_under_classify(kx):
    recs, was, goff, gmem = _seeded(4096, 4096, 3)
    before = kx.launch_count()
    kx.vf_vgpu_drift(recs, was, goff, gmem)
    assert kx.launch_count() - before == 1
    assert kx.timings()[B.T_CLASSIFY] > 0
