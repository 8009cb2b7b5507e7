"""CPU tests of kxpu_reset_check (include/kxpu.h, an addition to ABI v14): the C checker (tests/reset_oracle.c) against
the independent Python restatement (tests/pyref_reset.py) on the hand-worked forests, every reset_method text edge and
under hypothesis; each output against its sentence in the header; the invalid CSRs; and the header and binding
surface."""
import os
import re

import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pyref_pcie as PP
import pyref_reset as P
import reset_cases as RC
import reset_oracle as RO
from conftest import ROOT
from oracle import xpu_oracle as XO
from kxpu_b200 import binding as B


def _csr(recs, rules=RC.NV):
    res = XO.classify_rules(rules, recs)
    return res["group_ids"], res["group_off"], res["group_members"]


def _both(rules, recs, paths, rrs, allow, off, mem):
    got, want = RO.reset_check(rules, recs, paths, rrs, allow, off, mem), P.reset_check(rules, recs, paths, rrs, allow, off, mem)
    assert got == want
    return got


@pytest.mark.parametrize("name", sorted(RC.HAND))
def test_hand_forests(name):
    (recs, paths, rrs), allow, methods, verdict, groups = RC.HAND[name]
    gids, off, mem = _csr(recs)
    got = _both(RC.NV, recs, paths, rrs, allow, off, mem)
    assert got["methods"] == methods and got["set_verdict"] == verdict
    assert dict(zip([int(g) for g in gids], got["group_reset"])) == groups


@pytest.mark.parametrize("txt,flags,want", RC.TEXTS)
def test_reset_method_texts(txt, flags, want):
    s = RC.rr(txt, flags)
    assert P.methods(bytes(s["txt"]), int(s["len"]), int(s["flags"])) == want
    recs, paths, rrs = RC.walk(RC.fn(b"0000:00:05.0", 1, ["pci0000:00"], method=txt, rflags=flags))
    _, off, mem = _csr(recs)
    for allow in RC.ALLOWS:
        got = _both(RC.NV, recs, paths, rrs, allow, off, mem)
        assert got["methods"] == [want]
        fn = bool(want & allow) or (bool(want & RC.UNNAMED) and allow == RC.ALL)  # a root bus: no set reset
        assert got["group_reset"] == [RC.VIABLE if fn else 0]


def test_text_lengths_at_the_limit():
    assert len(RC._T64) == B.RESET_FILE_MAX and len(RC._T65) == B.RESET_FILE_MAX + 1
    assert RC.rr(RC._T65)["len"] == B.RESET_FILE_MAX + 1 and RC.rr(b"x" * 300)["len"] == B.RESET_FILE_MAX + 1


@settings(max_examples=300, deadline=None)
@given(RC.reset_walks(), st.sampled_from(RC.ALLOWS), st.sampled_from([RC.NV, [(b"10de", b"vfio-pci"), (b"1002", b"nvme")]]))
def test_oracle_equals_pyref(w, allow, rules):
    recs, paths, rrs = w
    _, off, mem = _csr(recs, rules)
    _both(rules, recs, paths, rrs, allow, off, mem)


@settings(max_examples=300, deadline=None)
@given(RC.reset_walks(), st.sampled_from(RC.ALLOWS))
def test_restatement_meets_each_rule(w, allow):
    """Every verdict checked against its sentence in the header: the named record keeps the set from being closed."""
    recs, paths, rrs = w
    gids, off, mem = _csr(recs)
    got = P.reset_check(RC.NV, recs, paths, rrs, allow, off, mem)
    chains = [PP.record_chain(recs[i], paths[i]) for i in range(len(recs))]
    for i, v in enumerate(got["set_verdict"]):
        if not chains[i]:
            assert v == RC.NO_PATH
        elif chains[i][-1] >> 63:
            assert v == RC.ROOT_BUS
        elif v != RC.SET_OK:
            assert chains[i][-1] in chains[v]  # below the same bridge
            r = recs[v]
            bound = bytes(r["driver"]).rstrip(b"\0") == b"vfio-pci" and not int(r["flags"]) & 0x16
            assert not bound or int(r["iommu_group"]) != int(recs[i]["iommu_group"])
    for g in range(len(gids)):
        for i in (int(x) for x in mem[off[g]:off[g + 1]]):
            if i < got["group_reset"][g]:
                assert P.function_reset(got["methods"][i], allow) or got["set_verdict"][i] == RC.SET_OK


def test_invalid_csr():
    (recs, paths, rrs), *_ = RC.HAND["three_groups_under_one_port"]
    _, off, mem = _csr(recs)
    assert RO.reset_check(RC.NV, recs, paths, rrs, RC.ALL, np.array([0, 2, 1, 4], np.uint32), mem) is None
    assert RO.reset_check(RC.NV, recs, paths, rrs, RC.ALL, off, np.array([0, 1, 2, 4], np.uint32)) is None
    assert P.reset_check(RC.NV, recs, paths, rrs, RC.ALL, off, np.array([0, 1, 2, 4], np.uint32)) is None


def test_header_and_binding():
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert re.search(r"#define KXPU_ABI_VERSION 14\b", hdr)
    assert re.search(r"\bkxpu_reset_check\s*\(", hdr) and "kxpu_reset_check" in B.ABI_SYMBOLS
    assert "kxpu_resetrec;" in hdr and B.RESETREC_DTYPE.itemsize == 80
    assert B.RESETREC_DTYPE.fields["len"][1] == 64 and B.RESETREC_DTYPE.fields["flags"][1] == 65
    for k, name in enumerate(B.RESET_METHODS):
        assert re.search(r"#define KXPU_RM_%s\s+0x%02xu" % (name.upper(), 1 << k), hdr, re.I), name
    start = hdr.index("resets between tenants")
    assert hdr[start:hdr.index("kxpu_reset_check(kxpu_ctx")].count("[assumed]") >= 4
