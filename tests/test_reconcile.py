"""CPU tests of the rediscovery index rule (include/kxpu.h, ABI v6): the C oracle (oracle/kxpu_reconcile_oracle.c)
against the independent dict-based restatement (tests/pyref_reconcile.py) under a fuzz, both identities, every
invalid case, and the rediscovery workload's shape."""
import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pyref_reconcile as P
from kxpu_b200 import workloads as W
from kxpu_b200.binding import SNAPREC_DTYPE
from oracle import reconcile_oracle as RO

KEYS = [b"0000:00:00.0", b"0000:00:00.1", b"0000:01:00.0", b"0000:02:00.0", b"0000:0a:00.0",
        b"8a6d5b2e-6f7a-4b2c-9d1e-0123456789ab", b"x" * 39, b"k"]


def snap(entries):
    a = np.zeros(len(entries), SNAPREC_DTYPE)
    for i, e in enumerate(entries):
        a[i] = e
    return a


def same(got, want):
    assert (got is None) == (want is None)
    if got is None:
        return
    assert list(got["index"]) == list(want["index"])
    assert list(got["cur_state"]) == list(want["cur_state"])
    assert list(got["prev_state"]) == list(want["prev_state"])
    assert got["counts"] == want["counts"]


@st.composite
def pairs(draw):
    """prev / cur over a small key pool, so that kept, changed, new, retired and (sometimes) duplicates all occur."""
    def entries(n, with_index):
        return [(draw(st.sampled_from(KEYS)), draw(st.integers(0, 3)), draw(st.integers(0, 2)),
                 draw(st.sampled_from([0, 1, 0xFFFFFFFFFFFFFFFF])), draw(st.integers(0, 20)) if with_index else 0)
                for _ in range(n)]
    prev = entries(draw(st.integers(0, 6)), True)
    if draw(st.booleans()):  # mostly distinct keys
        seen = set()
        prev = [e for e in prev if not (e[0] in seen or seen.add(e[0]))]
    cur = entries(draw(st.integers(0, 6)), False)
    if draw(st.booleans()):
        seen = set()
        cur = [e for e in cur if not (e[0] in seen or seen.add(e[0]))]
    next_index = draw(st.one_of(st.integers(0, 24), st.just((1 << 64) - 3)))
    return prev, cur, next_index


@settings(max_examples=400, deadline=None)
@given(pairs())
def test_oracle_equals_pyref(p):
    prev, cur, next_index = p
    same(RO.reconcile(snap(prev), snap(cur), next_index), P.reconcile(prev, cur, next_index))


def test_workload_oracle_equals_pyref():
    prev, cur, ni = W.reconcile_pair(4, 1 << 12)
    same(RO.reconcile(prev, cur, ni), P.reconcile(P.rows(prev), P.rows(cur), ni))
    prev, cur, ni = W.reconcile_pair(5, 1 << 12, mdev=True)
    same(RO.reconcile(prev, cur, ni), P.reconcile(P.rows(prev), P.rows(cur), ni))


@pytest.mark.parametrize("mdev", [False, True])
def test_workload_shape(mdev):
    n = 1 << 14
    prev, cur, ni = W.reconcile_pair(3, n, mdev=mdev)
    assert ni == n and list(prev["index"]) == list(range(n))
    assert list(prev["key"]) == sorted(prev["key"]) and list(cur["key"]) == sorted(cur["key"])
    c = RO.reconcile(prev, cur, ni)["counts"]
    assert c["n_retired"] == n // 20 and c["n_new"] == n // 20
    assert c["n_changed"] == 3 * (n // 100)
    assert c["next_index_out"] == ni + c["n_new"] + c["n_changed"]


def test_identity_fresh_walk_is_walk_order():
    prev, cur, _ = W.reconcile_pair(6, 1 << 10)
    r = RO.reconcile(snap([]), cur, 0)
    assert list(r["index"]) == list(range(len(cur)))
    assert set(r["cur_state"].tolist()) == {P.RC_NEW}
    assert r["counts"]["next_index_out"] == len(cur)


def test_identity_reconcile_of_own_output_keeps_everything():
    prev, cur, ni = W.reconcile_pair(7, 1 << 10, mdev=True)
    r = RO.reconcile(prev, cur, ni)
    again = cur.copy()
    again["index"] = r["index"]
    nxt = r["counts"]["next_index_out"]
    r2 = RO.reconcile(again, cur, nxt)
    assert list(r2["index"]) == list(r["index"])
    assert set(r2["cur_state"].tolist()) == {P.RC_KEPT} and set(r2["prev_state"].tolist()) == {P.RC_KEPT}
    assert r2["counts"]["next_index_out"] == nxt


def test_identity_matches_classify_busindex(oracle, oracle_rows):
    """n_prev = 0, next_index = 0 over the accepted cfg3 records in walk order gives their busIndex."""
    recs = W.cfg3_records(oracle_rows["key"], n=1 << 12)
    acc = oracle.classify(recs)["accept_index"]
    cur = W.snapshot_of_records(recs, acc)
    r = RO.reconcile(snap([]), cur, 0)
    assert np.array_equal(r["index"], cur["index"])


def invalid_cases():
    ok = (b"0000:00:00.0", 1, 0, 5, 0)
    ok2 = (b"0000:00:01.0", 2, 0, 5, 1)
    return {
        "dup_prev": ([ok, (ok[0], 3, 1, 1, 1)], [ok], 2),
        "dup_cur": ([ok], [ok2, ok2], 2),
        "empty_key_prev": ([(b"", 1, 0, 0, 0)], [ok], 2),
        "empty_key_cur": ([ok], [(b"", 1, 0, 0, 0)], 2),
        "nul_inside_prev": ([(b"ab\0cd", 1, 0, 0, 0)], [], 2),
        "nul_inside_cur": ([], [(b"0000\0:00.0", 1, 0, 0, 0)], 2),
        "index_at_next": ([ok2], [ok], 1),
        "index_above_next": ([(ok[0], 1, 0, 5, 9)], [ok], 3),
        "overflow": ([], [ok, ok2], (1 << 64) - 1),
    }


@pytest.mark.parametrize("case", list(invalid_cases()))
def test_invalid_inputs(case):
    prev, cur, ni = invalid_cases()[case]
    assert P.reconcile(prev, cur, ni) is None
    assert RO.reconcile(snap(prev), snap(cur), ni) is None


def test_key_of_39_bytes_and_full_64bit_tag_are_valid():
    k = b"y" * 39
    r = RO.reconcile(snap([(k, 0, 0, 0xFFFFFFFFFFFFFFFF, 3)]), snap([(k, 0, 0, 0xFFFFFFFFFFFFFFFF, 0)]), 4)
    assert list(r["index"]) == [3] and r["counts"]["n_kept"] == 1
