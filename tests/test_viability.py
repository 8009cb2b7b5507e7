"""CPU tests of IOMMU group viability (include/kxpu.h, ABI v8): the C oracle (oracle/kxpu_viab_oracle.c) against the
independent Python restatement (tests/pyref_viab.py), and the identities with the any-vendor and topology checkers."""
import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pyref_viab as P
import viab_cases as VC
from oracle import topo_oracle as TO
from oracle import viab_oracle as VO
from oracle import xpu_oracle as XO

KEYS = ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups", "dev_rule")


def _pairs(res):
    return [(int(g), int(b)) for g, b in zip(res["group_ids"], res["group_blocker"])]


@pytest.mark.parametrize("name", sorted(VC.HAND))
def test_hand_cases(name):
    recs, want = VC.HAND[name]
    res = VO.classify_viable(VC.NV, recs)
    assert _pairs(res) == want
    assert P.viability(VC.NV, recs) == want


@settings(max_examples=300, deadline=None)
@given(VC.viab_recs(), st.sampled_from([VC.NV, VC.TWO]), st.booleans())
def test_oracle_equals_pyref(recs, rules, topo):
    res = VO.classify_viable(rules, recs, topo=topo)
    assert _pairs(res) == P.viability(rules, recs)
    want = TO.classify_topo(rules, recs) if topo else XO.classify_rules(rules, recs)
    for k in KEYS + (("group_numa",) if topo else ()):
        assert np.array_equal(res[k], want[k]), k


@settings(max_examples=100, deadline=None)
@given(VC.viab_recs(), st.sampled_from([VC.NV, VC.TWO]))
def test_without_the_flag_every_group_is_viable(recs, rules):
    recs = recs.copy()
    recs["flags"] &= ~np.uint8(VC.BLOCKS)
    res = VO.classify_viable(rules, recs)
    assert (res["group_blocker"] == VO.VIABLE).all()
    want = XO.classify_rules(rules, recs)
    for k in KEYS:
        assert np.array_equal(res[k], want[k]), k


def test_blocker_of_group_all_ones_is_unsupported():
    recs = VC.arr(VC.gpu(0, 1), VC.host(1, 0xFFFFFFFF))
    assert VO.classify_viable(VC.NV, recs) == -7
    assert P.viability(VC.NV, recs) == "unsupported"
    # a directory or a candidate with the flag is not a blocker, so its group is not looked at
    recs = VC.arr(VC.gpu(0, 1), VC.rec(b"0000:01:00.0", 0xFFFFFFFF, driver=b"", flags=VC.IS_DIR | VC.BLOCKS))
    assert _pairs(VO.classify_viable(VC.NV, recs)) == [(1, VC.VIABLE)]


def test_invalid_rule_list():
    assert VO.classify_viable([], VC.arr(VC.gpu(0, 1))) == -1
    assert VO.classify_viable([(b"10de", b"vfio-pci")] * 2, VC.arr(VC.gpu(0, 1))) == -1


def test_workload(workloads):
    recs = workloads.viab_records(n=1 << 14)
    res = VO.classify_viable(workloads.VIAB_RULES, recs)
    assert _pairs(res) == P.viability(workloads.VIAB_RULES, recs)
    gb = res["group_blocker"]
    first = res["group_members"][res["group_off"][:-1]]
    blocked = gb != VO.VIABLE
    # every shape the workload promises: blockers in front of and behind the first member, viable groups, and
    # blocker-only groups that produce nothing
    assert (gb[blocked] < first[blocked]).any() and (gb[blocked] > first[blocked]).any() and (~blocked).any()
    blocker_groups = set(recs["iommu_group"][(recs["flags"] & VC.BLOCKS) != 0].tolist())
    assert blocker_groups - set(res["group_ids"].tolist())
