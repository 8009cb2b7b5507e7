"""CPU tests of the vGPU-on-VF calls (include/kxpu.h, additions to ABI v14): the C checker (tests/vf_vgpu_oracle.c, and
the C classify oracles on rewritten records) against the independent Python restatement (tests/pyref_vf_vgpu.py) on the
hand cases, every current_vgpu_type shape and under hypothesis; the restatement against the header's sentences; and the
header and binding surface."""
import os
import re

import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pyref_vf_vgpu as P
import vf_vgpu_cases as VV
import vf_vgpu_oracle as VO
from conftest import ROOT
from oracle import xpu_oracle as XO
from kxpu_b200 import binding as B


def _both_types(recs, tables):
    got, want = VO.vf_vgpu_types(recs, tables), P.vf_vgpu_types(recs, tables)
    assert got == want
    return got


@pytest.mark.parametrize("name", sorted(VV.HAND))
def test_hand_cases(name):
    tables, curs, want = VV.HAND[name]
    got = _both_types(VV.vts(*[VV.vt(c) for c in curs]), tables)
    assert list(zip(got["status"], got["type_id"])) == [(s, t) for s, t, _ in want]
    for row, (_, _, k) in zip(got["keys"], want):
        assert row == VV.key(k).tobytes()


@pytest.mark.parametrize("case", range(len(VV.CURRENT)))
def test_current_shapes(case):
    (cur, flags), want = VV.CURRENT[case]
    got = _both_types(VV.vts(VV.vt(cur, flags)), [b"557 : A\n"])
    assert (got["status"][0], got["type_id"][0]) == want


@settings(max_examples=300, deadline=None)
@given(VV.type_inputs())
def test_types_oracle_equals_pyref(inp):
    tables, recs = inp
    got = _both_types(recs, tables)
    for row, s in zip(got["keys"], got["status"]):
        assert (row != bytes(48)) == (s == VV.NAMED)
        assert row[40:47] == bytes(7)  # nothing but the key and its length lives in a row


def test_decreasing_table_offsets():
    assert VO.vf_vgpu_types(VV.vts(VV.vt(b"557")), (b"557 : A\n", [0, 8, 4])) is None


def _both_classify(recs, keys, mask, topo, viable):
    got = VO.classify_vf_vgpu(VV.RULES, mask, recs, keys, topo=topo, viable=viable)
    want = P.classify_vf_vgpu(VV.RULES, mask, recs, [k.tobytes() for k in keys], topo=topo, viable=viable)
    assert set(got) == set(want)
    for k in want:
        g = [int(x) for x in got[k]] if isinstance(want[k], list) else got[k]
        assert g == want[k], k
    return want


def _hand_walk():
    recs = np.array([VV.dev(b"0000:03:00.0", 30),                                 # the PF: no key, no candidate
                     VV.dev(b"0000:03:00.4", 31), VV.dev(b"0000:03:00.5", 32),    # type A
                     VV.dev(b"0000:03:00.6", 33),                                 # type B
                     VV.dev(b"0000:03:00.7", 34),                                 # free
                     VV.dev(b"0000:04:00.0", 40, driver=b"vfio-pci"),             # passthrough
                     VV.dev(b"0000:03:01.0", 35)], XO.DEVREC_DTYPE)               # type A again
    keys = np.array([VV.key(k) for k in (b"", b"A", b"A", b"B", b"", b"", b"A")], B.VGPUKEY_DTYPE)
    return recs, keys


@pytest.mark.parametrize("topo,viable", [(False, False), (True, False), (False, True), (True, True)])
def test_classify_hand_walk(topo, viable):
    recs, keys = _hand_walk()
    got = _both_classify(recs, keys, VV.VGPU_BIT, topo, viable)
    assert got["group_ids"] == [31, 32, 33, 40, 35]
    assert got["dev_ids"][:2] == [1, 3] and got["dev_rule"] == [2, 2, 0]
    assert [got["dev_groups"][got["dev_off"][d]:got["dev_off"][d + 1]] for d in range(3)] == [[31, 32, 35], [33], [40]]


@settings(max_examples=300, deadline=None)
@given(VV.classify_inputs(), st.sampled_from([0, VV.VGPU_BIT, 1 | VV.VGPU_BIT, 7]), st.booleans(), st.booleans())
def test_classify_oracle_equals_pyref(inp, mask, topo, viable):
    recs, keys = inp
    _both_classify(recs, keys, mask, topo, viable)


def test_header_and_binding():
    h = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    for sym in ("kxpu_vf_vgpu_types", "kxpu_classify_vf_vgpu"):
        assert re.search(r"int32_t %s\(" % sym, h) and sym in B.ABI_SYMBOLS
    block = h[h.index("vGPUs on SR-IOV virtual functions"):h.index("runtime rediscovery (ABI v6)")]
    assert block.count("[assumed]") == 5
    assert B.VFVGPUREC_DTYPE.itemsize == 32 and B.VGPUKEY_DTYPE.itemsize == 48
    assert (B.VT_READ, B.VT_CUR_ERR, B.VT_NONE, B.VT_NAMED, B.VT_UNNAMED, B.VT_BAD) == (1, 2, 0, 1, 2, 3)
    blob, toff = B.vgpu_tables([b"ab", b"", b"c"])
    assert blob.tobytes() == b"abc" and toff.tolist() == [0, 2, 2, 3]
