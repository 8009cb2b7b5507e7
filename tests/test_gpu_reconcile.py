"""GPU tests of kxpu_reconcile (include/kxpu.h, ABI v6) against the CPU oracle (oracle/kxpu_reconcile_oracle.c)."""
import numpy as np
import pytest

import kxpu_b200 as K
from kxpu_b200.binding import E_INVALID, REJECTED, SNAPREC_DTYPE, reconcile_outputs
from oracle import reconcile_oracle as RO

pytestmark = pytest.mark.gpu


def same(got, want):
    for k in ("index", "cur_state", "prev_state"):
        assert np.array_equal(got[k], want[k]), k
    assert got["counts"] == want["counts"]


@pytest.mark.parametrize("mdev", [False, True])
def test_reconcile_pair_2_20(kx, workloads, mdev):
    prev, cur, ni = workloads.reconcile_pair(3, 1 << 20, mdev=mdev)
    got = kx.reconcile(prev, cur, ni)
    same(got, RO.reconcile(prev, cur, ni))
    c = got["counts"]
    assert c["n_kept"] and c["n_new"] and c["n_changed"] and c["n_retired"]


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 5000, 77777])
def test_sizes_around_the_tile(kx, workloads, n):
    prev, cur, ni = workloads.reconcile_pair(n, max(n, 20), mdev=bool(n & 1))
    cur = cur[:n]
    same(kx.reconcile(prev, cur, ni), RO.reconcile(prev, cur, ni))


def test_keys_differing_in_one_byte(kx):
    """39-byte keys that differ only in their last byte, or only past a shared 32-byte prefix: the byte compare on a hash
    hit must tell them apart."""
    rng = np.random.default_rng(1)
    n = 1 << 16
    base = np.frombuffer(b"q" * 39, np.uint8)
    keys = np.tile(base, (n, 1))
    keys[:, 38] = 33 + (np.arange(n) % 90)
    keys[:, 33] = 33 + (np.arange(n) // 90) % 90
    keys[:, 35] = 33 + (np.arange(n) // 8100)
    prev = np.zeros(n, SNAPREC_DTYPE)
    prev["key"] = keys.view("S39").reshape(n)
    prev["iommu_group"] = rng.integers(0, 50, n)
    prev["index"] = rng.permutation(2 * n)[:n]
    cur = prev[rng.permutation(n)[: n - 100]].copy()
    cur["klass"][::7] = 1
    same(kx.reconcile(prev, cur, 2 * n), RO.reconcile(prev, cur, 2 * n))


def test_identities_equal_classify_busindex_cfg3(kx, workloads, oracle_rows):
    recs = workloads.cfg3_records(oracle_rows["key"])
    acc = kx.classify(recs)["accept_index"]
    cur = workloads.snapshot_of_records(recs, acc)
    fresh = kx.reconcile(np.zeros(0, SNAPREC_DTYPE), cur, 0)
    assert np.array_equal(fresh["index"], acc[acc != REJECTED].astype(np.uint64))
    assert fresh["counts"]["next_index_out"] == len(cur) and (fresh["cur_state"] == 1).all()
    prev = cur.copy()
    prev["index"] = fresh["index"]
    again = kx.reconcile(prev, cur, len(cur))
    assert np.array_equal(again["index"], fresh["index"])
    assert (again["cur_state"] == 0).all() and (again["prev_state"] == 0).all()
    assert again["counts"] == dict(n_kept=len(cur), n_new=0, n_changed=0, n_retired=0, next_index_out=len(cur))


def test_empty_lists(kx, workloads):
    prev, cur, ni = workloads.reconcile_pair(2, 3000)
    empty = np.zeros(0, SNAPREC_DTYPE)
    same(kx.reconcile(prev, empty, ni), RO.reconcile(prev, empty, ni))
    r = kx.reconcile(empty, empty, 17)
    assert r["counts"] == dict(n_kept=0, n_new=0, n_changed=0, n_retired=0, next_index_out=17)


@pytest.mark.parametrize("where", ["cur", "prev", "both"])
def test_duplicates_are_invalid_and_leave_outputs_untouched(kx, workloads, where):
    prev, cur, ni = workloads.reconcile_pair(8, 1 << 18, mdev=where == "prev")
    if where in ("cur", "both"):
        cur[5000]["key"] = cur[90000]["key"]
    if where in ("prev", "both"):
        prev[123456]["key"] = prev[7]["key"]
    assert RO.reconcile(prev, cur, ni) is None
    out = reconcile_outputs(len(prev), len(cur), fill=0xA5A5A5A5A5A5A5A5)
    counts0 = out["counts"].copy()
    with pytest.raises(K.KxpuError) as e:
        kx.reconcile_raw(prev, cur, ni, out)
    assert e.value.status == E_INVALID and "duplicate" in str(e.value)
    assert (out["index"] == 0xA5A5A5A5A5A5A5A5).all() and (out["cur_state"] == 0xA5).all()
    assert (out["prev_state"] == 0xA5).all() and out["counts"].tobytes() == counts0.tobytes()


@pytest.mark.parametrize("case", ["empty_key", "nul_inside", "prev_index", "overflow"])
def test_other_invalid_inputs(kx, workloads, case):
    prev, cur, ni = workloads.reconcile_pair(9, 4096)
    if case == "empty_key":
        cur[100]["key"] = b""
    elif case == "nul_inside":
        k = bytearray(bytes(prev[200]["key"]).ljust(40, b"\0"))
        k[20] = ord("z")
        prev.view(np.uint8).reshape(-1, 64)[200, :40] = np.frombuffer(bytes(k), np.uint8)
    elif case == "prev_index":
        prev[300]["index"] = ni
    else:
        ni = (1 << 64) - 10
    assert RO.reconcile(prev, cur, ni) is None
    out = reconcile_outputs(len(prev), len(cur), fill=0x5A)
    with pytest.raises(K.KxpuError) as e:
        kx.reconcile_raw(prev, cur, ni, out)
    assert e.value.status == E_INVALID
    assert (out["index"] == 0x5A).all() and (out["cur_state"] == 0x5A).all() and (out["prev_state"] == 0x5A).all()
