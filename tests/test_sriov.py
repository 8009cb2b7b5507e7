"""CPU tests of the SR-IOV calls (include/kxpu.h, additions to ABI v14): the C checker (tests/sriov_oracle.c) against the
independent Python restatement (tests/pyref_sriov.py) on the hand cases, every sriov_numvfs shape and under hypothesis;
their forest against the C PCIe oracle when no record has a PF; the depth limit of a VF's chain; the invalid inputs; and
the header and binding surface."""
import os
import re

import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pyref_pcie as PP
import pyref_sriov as P
import sriov_cases as SC
import sriov_oracle as SO
from conftest import ROOT
from oracle import pcie_oracle as PO
from oracle import xpu_oracle as XO
from kxpu_b200 import binding as B


def _csr(recs, rules=SC.NV):
    res = XO.classify_rules(rules, recs)
    return res["group_ids"], res["group_off"], res["group_members"]


def _both(rules, recs, srs, off, mem):
    got, want = SO.sriov(rules, recs, srs, off, mem), P.sriov(rules, recs, srs, off, mem)
    assert got == want
    return got


@pytest.mark.parametrize("name", sorted(SC.HAND))
def test_hand_cases(name):
    (recs, srs), pf_of, numvfs, groups = SC.HAND[name]
    gids, off, mem = _csr(recs)
    got = _both(SC.NV, recs, srs, off, mem)
    assert got["pf_of"] == pf_of and got["numvfs"] == numvfs
    assert dict(zip([int(g) for g in gids], got["group_sriov"])) == groups


@pytest.mark.parametrize("txt,want", SC.NUMVFS)
def test_numvfs_shapes(txt, want):
    s = SC.sr(numvfs=txt)
    assert P.numvfs(s["numvfs_txt"], int(s["numvfs_len"])) == want
    recs, srs = SC.walk(SC.fn(b"0000:01:00.0", 1, numvfs=txt))
    _, off, mem = _csr(recs)
    assert SO.sriov(SC.NV, recs, srs, off, mem)["numvfs"] == [want]


@settings(max_examples=300, deadline=None)
@given(SC.sriov_walks(), st.sampled_from([SC.NV, SC.VC.TWO]))
def test_oracle_equals_pyref(w, rules):
    recs, srs = w
    _, off, mem = _csr(recs, rules)
    _both(rules, recs, srs, off, mem)


@settings(max_examples=300, deadline=None)
@given(SC.sriov_walks())
def test_restatement_meets_each_rule(w):
    """Every output checked against its sentence in the header, record by record."""
    recs, srs = w
    gids, off, mem = _csr(recs)
    got = P.sriov(SC.NV, recs, srs, off, mem)
    names = [bytes(r["bdf"]).rstrip(b"\0") for r in recs]
    for i, s in enumerate(srs):
        pf = bytes(s["physfn"]).rstrip(b"\0")
        ok = P.canonical(pf) and not int(s["flags"]) & SC.PHYSFN_ERR and pf in names and names.index(pf) != i
        assert got["pf_of"][i] == (names.index(pf) if ok else SC.NO_PF)
    for g in range(len(gids)):
        members = [int(m) for m in mem[off[g]:off[g + 1]]]
        block = [i for i in members if got["numvfs"][i] > 0 or (
            got["pf_of"][i] != SC.NO_PF and bytes(recs[got["pf_of"][i]]["driver"]).rstrip(b"\0") == b"vfio-pci"
            and not int(recs[got["pf_of"][i]]["flags"]) & 0x02)]
        assert got["group_sriov"][g] == (min(block) if block else SC.VIABLE)


def test_invalid_csr():
    (recs, srs), *_ = SC.HAND["pf_on_vfio_with_vfs"]
    _, off, mem = _csr(recs)
    assert SO.sriov(SC.NV, recs, srs, np.array([0, 2, 1, 3], np.uint32), mem) is None
    assert SO.sriov(SC.NV, recs, srs, off, np.array([0, 1, 3], np.uint32)) is None


@settings(max_examples=300, deadline=None)
@given(SC.forests())
def test_tree_oracle_equals_pyref(f):
    recs, paths, off, mem, pf_of = f
    assert SO.tree(recs, paths, off, mem, pf_of) == P.tree(recs, paths, off, mem, pf_of)


@settings(max_examples=300, deadline=None)
@given(SC.forests())
def test_tree_without_pfs_is_the_pcie_tree(f):
    recs, paths, off, mem, _ = f
    want = PO.tree(recs, paths, off, mem)
    none = np.full(len(recs), SC.NO_PF, np.uint32)
    for got in (P.tree(recs, paths, off, mem, none), SO.tree(recs, paths, off, mem, none)):
        for k in ("group_node", "key", "parent", "depth"):
            assert got[k] == [int(x) for x in want[k]], k


@settings(max_examples=300, deadline=None)
@given(SC.forests())
def test_tree_places_vfs_under_their_pf(f):
    recs, paths, off, mem, pf_of = f
    got = P.tree(recs, paths, off, mem, pf_of)
    for g in range(len(off) - 1):
        members = [int(m) for m in mem[off[g]:off[g + 1]]]
        if len(members) != 1 or pf_of[members[0]] == SC.NO_PF:
            continue
        p = int(pf_of[members[0]])
        pc = PP.record_chain(recs[p], paths[p])
        if 0 < len(pc) < PP.MAX_DEPTH:  # the group's node is the PF's node, at the PF's depth
            v = got["group_node"][g]
            assert got["depth"][v] == len(pc) and got["key"][v] == PP.component_key(bytes(recs[p]["bdf"]).decode())[0]


def test_tree_depth_limit():
    # a PF chain of 7 keys: the VF's chain is 8 keys, the PF's node is its parent
    recs, paths, off, mem, pf_of = SC.deep(7)
    t = P.tree(recs, paths, off, mem, pf_of)
    assert SO.tree(recs, paths, off, mem, pf_of) == t
    assert t["depth"][t["group_node"][1]] == 7 and t["parent"][t["group_node"][1]] == t["group_node"][0]
    # a PF chain of 8 keys: 9 would not fit, so the VF keeps its own chain (the PF's siblings' parent)
    recs, paths, off, mem, pf_of = SC.deep(8)
    t = P.tree(recs, paths, off, mem, pf_of)
    assert SO.tree(recs, paths, off, mem, pf_of) == t
    assert t["group_node"][1] == t["group_node"][0]
    assert t == P.tree(recs, paths, off, mem, np.full(2, SC.NO_PF, np.uint32))


def test_tree_invalid_pf_of():
    recs, paths, off, mem, _ = SC.deep(2)
    bad = np.array([SC.NO_PF, 2], np.uint32)
    assert P.tree(recs, paths, off, mem, bad) is None and SO.tree(recs, paths, off, mem, bad) is None


def test_header_and_binding():
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert re.search(r"#define KXPU_ABI_VERSION 14\b", hdr)
    for sym in ("kxpu_sriov", "kxpu_pcie_tree_sriov"):
        assert re.search(r"\b%s\s*\(" % sym, hdr) and sym in B.ABI_SYMBOLS
    assert "kxpu_sriovrec;" in hdr and B.SRIOVREC_DTYPE.itemsize == 32
    assert B.SRIOVREC_DTYPE.fields["numvfs_len"][1] == 24 and B.SRIOVREC_DTYPE.fields["flags"][1] == 25
    assert hdr.count("[assumed]") >= 4
