"""CPU tests of the drift rule of kxpu_vf_vgpu_drift: the C oracle and the Python restatement agree with each other and
with hand-written answers at every edge of the current-type text, on the group fold and on the refusals."""
import numpy as np
import pytest

import pyref_vf_vgpu_health as P
import vf_vgpu_health_oracle as O
from kxpu_b200.binding import VFVGPUREC_DTYPE, VT_CUR_ERR, VT_READ


def rec(text, flags=VT_READ, length=None):
    r = np.zeros(1, VFVGPUREC_DTYPE)
    r["cur_txt"][0][:min(len(text), 16)] = np.frombuffer(text[:16], np.uint8)
    r["cur_len"] = min(len(text), 17) if length is None else length
    r["flags"] = flags
    return r


# (file text, the walk's type, status, type now)
EDGES = [
    (b"557\n", 557, P.SAME, 557),
    (b"557", 557, P.SAME, 557),
    (b"0", 557, P.CLEARED, 0),
    (b"0\n", 557, P.CLEARED, 0),
    (b"0\n", 0, P.SAME, 0),
    (b"558\n", 557, P.CHANGED, 558),
    (b"557\n", 0, P.CHANGED, 557),
    (b"557\n\n", 557, P.BAD, 0),       # one trailing '\n' only
    (b"557\r\n", 557, P.BAD, 0),
    (b"557\r", 557, P.BAD, 0),
    (b"0557\n", 557, P.BAD, 0),        # a leading zero
    (b"00\n", 0, P.BAD, 0),
    (b"", 557, P.BAD, 0),
    (b"\n", 557, P.BAD, 0),
    (b" 557\n", 557, P.BAD, 0),
    (b"+557\n", 557, P.BAD, 0),
    (b"4294967295\n", 4294967295, P.SAME, 4294967295),
    (b"4294967295", 557, P.CHANGED, 4294967295),
    (b"4294967296\n", 557, P.BAD, 0),
    (b"99999999999\n", 557, P.BAD, 0),  # eleven digits
    (b"1" + b"\0" * 14 + b"\n", 1, P.BAD, 0),   # 16 bytes
    (b"1" + b"\0" * 15 + b"\n", 1, P.BAD, 0),   # 17 bytes: longer than the record holds
]


@pytest.mark.parametrize("text,was,status,now", EDGES)
def test_text_edges(text, was, status, now):
    want = dict(type_now=[now], status_now=[status], group_first=[P.STEADY if status == P.SAME else 0])
    for impl in (O, P):
        assert impl.vf_vgpu_drift(rec(text), [was], [0, 1], [0]) == want, impl.__name__


def test_sixteen_digit_texts():
    """a 16-byte text of digits is too long for a type ID; cur_len 17 is refused whatever the bytes hold"""
    for impl in (O, P):
        assert impl.vf_vgpu_drift(rec(b"1" * 16), [1], [0, 1], [0])["status_now"] == [P.BAD]
        assert impl.vf_vgpu_drift(rec(b"557\n", length=17), [557], [0, 1], [0])["status_now"] == [P.BAD]


def test_read_error_and_unread():
    recs = np.concatenate([rec(b"557\n", VT_READ | VT_CUR_ERR), rec(b"558\n", 0), rec(b"", 0)])
    want = dict(type_now=[0, 557, 9], status_now=[P.BAD, P.SAME, P.SAME], group_first=[0, P.STEADY])
    for impl in (O, P):
        assert impl.vf_vgpu_drift(recs, [557, 557, 9], [0, 1, 3], [0, 1, 2]) == want


def test_groups():
    """empty groups, one-member groups, a drifted member that is not the first, members shared between groups"""
    recs = np.concatenate([rec(b"557\n"), rec(b"0\n"), rec(b"558\n"), rec(b"557\n")])
    was = [557, 557, 557, 557]
    goff = [0, 0, 1, 2, 5, 5, 8]
    gmem = [0, 1, 3, 0, 2, 3, 3, 1]
    want = dict(type_now=[557, 0, 558, 557], status_now=[P.SAME, P.CLEARED, P.CHANGED, P.SAME],
                group_first=[P.STEADY, P.STEADY, 0, 2, P.STEADY, 2])
    for impl in (O, P):
        assert impl.vf_vgpu_drift(recs, was, goff, gmem) == want


def test_refusals():
    recs = np.concatenate([rec(b"557\n"), rec(b"557\n")])
    for impl in (O, P):
        assert impl.vf_vgpu_drift(recs, [557, 557], [0, 2, 1], [0, 1]) is None  # decreasing
        assert impl.vf_vgpu_drift(recs, [557, 557], [0, 2], [0, 2]) is None     # member >= n
        assert impl.vf_vgpu_drift(recs[:0], [], [0], []) == dict(type_now=[], status_now=[], group_first=[])


def test_oracle_against_pyref_seeded():
    rng = np.random.default_rng(15)
    texts = [b"0", b"0\n", b"557\n", b"558\n", b"4294967295\n", b"4294967296\n", b"0557\n", b"557\r\n", b"x\n", b""]
    n = 4096
    recs = np.zeros(n, VFVGPUREC_DTYPE)
    for i in range(n):
        t = texts[rng.integers(len(texts))] if rng.random() < 0.9 else bytes(rng.integers(0, 256, rng.integers(0, 18),
                                                                                           dtype=np.uint8))
        recs[i] = rec(t, int(rng.choice([VT_READ, VT_READ, VT_READ | VT_CUR_ERR, 0])))[0]
    was = rng.choice([0, 557, 558, 4294967295], n).astype(np.uint32)
    sizes = rng.integers(0, 5, 1500)
    goff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    gmem = rng.integers(0, n, int(goff[-1])).astype(np.uint32)
    assert O.vf_vgpu_drift(recs, was, goff, gmem) == P.vf_vgpu_drift(recs, was, goff.tolist(), gmem.tolist())
