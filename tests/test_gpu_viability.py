"""GPU tests of kxpu_classify_viable (include/kxpu.h, ABI v8) against the CPU oracle (oracle/kxpu_viab_oracle.c), and
the identities with kxpu_classify_rules / kxpu_classify_topo."""
import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import viab_cases as VC
from oracle import viab_oracle as VO

pytestmark = pytest.mark.gpu
KEYS = ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups", "dev_rule")


def assert_viable(kx, rules, recs):
    """The call with and without group_numa: bitwise the oracle's blockers, and every other output bitwise
    kxpu_classify_rules' / kxpu_classify_topo's on the same records."""
    want = VO.classify_viable(rules, recs)
    for topo in (False, True):
        got = kx.classify_viable(rules, recs, topo=topo)
        assert np.array_equal(got["group_blocker"], want["group_blocker"])
        plain = kx.classify_topo(rules, recs) if topo else kx.classify_rules(rules, recs)
        for k in KEYS + (("group_numa",) if topo else ()):
            assert np.array_equal(got[k], plain[k]), k
        assert got["n_accepted"] == plain["n_accepted"] and got["n_devids"] == plain["n_devids"]
    return want


def test_classify_viable_2_20(kx, workloads):
    recs = workloads.viab_records(n=1 << 20)
    n0 = kx.launch_count()
    got = kx.classify_viable(workloads.VIAB_RULES, recs)
    n1 = kx.launch_count()
    kx.classify_rules(workloads.VIAB_RULES, recs)
    assert kx.launch_count() - n1 == n1 - n0  # no added launch
    want = assert_viable(kx, workloads.VIAB_RULES, recs)
    assert np.array_equal(got["group_blocker"], want["group_blocker"])
    gb = want["group_blocker"]
    assert (gb == VC.VIABLE).any() and (gb != VC.VIABLE).sum() > 10000


@pytest.mark.parametrize("name", sorted(VC.HAND))
def test_hand_cases(kx, name):
    recs, want = VC.HAND[name]
    assert_viable(kx, VC.NV, recs)
    got = kx.classify_viable(VC.NV, recs)
    assert [(int(g), int(b)) for g, b in zip(got["group_ids"], got["group_blocker"])] == want


def test_blocker_of_group_all_ones_is_unsupported(kx):
    import kxpu_b200 as K
    recs = VC.arr(VC.gpu(0, 1), VC.host(1, 0xFFFFFFFF))
    with pytest.raises(K.KxpuError) as e:
        kx.classify_viable(VC.NV, recs)
    assert e.value.status == K.binding.E_UNSUPPORTED
    # the same record is no error for the calls that ignore the flag
    assert kx.classify_rules(VC.NV, recs)["n_groups"] == 1


def test_invalid_arguments(kx):
    import ctypes as C
    import kxpu_b200 as K
    L = kx.L
    recs = VC.arr(VC.gpu(0, 1))
    ra = K.binding.rules_array(VC.NV)
    out = K.binding.ClassifyOut()
    # group_blocker is required when n > 0; the rule list is checked as for kxpu_classify_rules
    assert L.kxpu_classify_viable(kx.ctx, ra.ctypes.data, 1, recs.ctypes.data, 1, C.byref(out), None, None, None) == -1
    buf = np.zeros(4, np.uint32)
    assert L.kxpu_classify_viable(kx.ctx, ra.ctypes.data, 0, recs.ctypes.data, 1, C.byref(out), None, None,
                                  buf.ctypes.data) == -1
    assert L.kxpu_classify_viable(kx.ctx, None, 1, recs.ctypes.data, 1, C.byref(out), None, None, buf.ctypes.data) == -1


def test_device_id_growth_retry(kx, workloads):
    """200 000 distinct device ids overflow the first 2^17-slot device-id table; the rerun must find the blockers again
    from a reset table."""
    from kxpu_b200.binding import DEVREC_DTYPE
    m = 200000
    n = 2 * m
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    recs["bdf"] = workloads.enumerate_bdfs(n).view("S16").reshape(n)
    recs["vendor_txt"][0::2] = np.frombuffer(b"0x10de\n\0", np.uint8)
    recs["vendor_txt"][1::2] = np.frombuffer(b"0x144d\n\0", np.uint8)
    recs["device_txt"][0::2] = np.frombuffer(b"".join(b"0x%05x\n" % k for k in range(m)), np.uint8).reshape(m, 8)
    recs["device_txt"][1::2] = np.frombuffer(b"0xa80a\n\0", np.uint8)
    recs["vendor_len"], recs["device_len"] = 7, 8
    recs["device_len"][1::2] = 7
    recs["driver"][0::2] = b"vfio-pci"
    recs["driver"][1::2] = b"nvme"
    k = np.arange(m, dtype=np.int64)
    recs["iommu_group"][0::2] = k
    # behind GPU k: a blocker of its own group (k % 3 == 0), of a group without candidates (k % 3 == 1), or none
    recs["iommu_group"][1::2] = np.where(k % 3 == 1, m + k, k)
    recs["flags"][1::2] = np.where(k % 3 == 2, 0, VC.BLOCKS)
    want = assert_viable(kx, VC.NV, recs)
    assert want["n_devids"] == m > (1 << 17)
    assert np.array_equal(want["group_blocker"], np.where(k % 3 == 0, 2 * k + 1, VC.VIABLE).astype(np.uint32))


def test_existing_calls_ignore_the_flag(kx, workloads, oracle_rows):
    """The same records with and without KXPU_REC_BLOCKS give bitwise the same outputs through every other call."""
    recs = workloads.viab_records(n=1 << 18)
    bare = recs.copy()
    bare["flags"] &= ~np.uint8(VC.BLOCKS)
    rules = workloads.VIAB_RULES
    for fn in (kx.classify, lambda r: kx.classify_rules(rules, r), lambda r: kx.classify_topo(rules, r)):
        a, b = fn(recs), fn(bare)
        for key in a:
            assert np.array_equal(np.asarray(a[key]), np.asarray(b[key])), key
    got = kx.classify_viable(rules, bare)
    assert (got["group_blocker"] == VC.VIABLE).all()


@settings(max_examples=150, deadline=None)
@given(VC.viab_recs(), st.sampled_from([VC.NV, VC.TWO]))
def test_fuzz(kx, recs, rules):
    assert_viable(kx, rules, recs)
