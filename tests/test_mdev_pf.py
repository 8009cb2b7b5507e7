"""CPU tests of the calls for mdev vGPUs on SR-IOV VFs (kxpu_mdev_pf and kxpu_dra_slices_mdev_pf, include/kxpu.h,
additions to ABI v14): the C oracle (tests/mdev_pf_oracle.c) against the Python restatement (tests/pyref_mdev_pf.py) on
hand cases -- non-canonical and flagged links, a PF outside the walk, a link to the mdev's own parent, duplicate
addresses -- and under hypothesis; the slices on the golden cfg1 line, with every attribute present or absent at the
slice seams, every domain refusal, the all-empty-physfn pool giving the mdev layout's bytes, and the kxpu_dramdevpf
layout."""
import json
import os
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import dra_mdev_cases as MC
import dra_taint_cases as TC
import mdev_pf_cases as PC
import mdev_pf_oracle as MO
import pyref_dra_mdev as PM
import pyref_dra_taint as PT
import pyref_mdev_pf as PR
from conftest import ROOT
from test_dra import LONG_DRIVER, LONG_NAME, check_schema

NO_PF = PC.NO_PF
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_mdev_pf_cfg1.jsonl")
ATTRS = ["iommuGroup", "mdevType", "numaNode", "parentAddress", "parentDeviceID", "parentVendorID", "physfnAddress",
         "physfnDeviceID", "productName", "resource.kubernetes.io/pcieRoot", "uuid"]


def join(recs, m, s):
    got = MO.mdev_pf(recs, m, s)
    assert got == PR.mdev_pf(recs, m, s)
    return got


def both(driver, pool, node, gen, devs, taints=(), since=None):
    got = MO.dra_slices_mdev_pf(driver, pool, node, gen, devs, taints, since)
    want = PR.slices(driver, pool, node, gen, devs, taints, since)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == want[1]
    else:
        assert got == want
    return got


def lines(blob):
    return [json.loads(x) for x in blob.split(b"\n")[:-1]]


# ---------------------------------------------------------------- kxpu_mdev_pf

WALK = [b"0000:41:00.0", b"0000:41:00.4", b"0000:41:00.5", b"0000:c1:00.0", b"0000:41:00.0", b"0000:81:00.0"]


@pytest.mark.parametrize("parent,physfn,flags,want", [
    (b"0000:41:00.4", b"0000:41:00.0", 0, 0),           # a VF's PF; the first of its two records
    (b"0000:41:00.5", b"0000:41:00.0", 0, 0),
    (b"0000:c1:00.0", b"", 0, NO_PF),                   # an mdev on a PF: no link
    (b"0000:41:00.4", b"0000:41:00.0", PC.SR_PHYSFN_ERR, NO_PF),  # a failed read
    (b"0000:41:00.4", b"0000:41:00.0\n", 0, NO_PF),     # not canonical
    (b"0000:41:00.4", b"0000:41:00.8", 0, NO_PF),
    (b"0000:41:00.4", b"0000:41:20.0", 0, NO_PF),       # device above 1f
    (b"0000:41:00.4", b"0000:41:0A.0", 0, NO_PF),       # uppercase
    (b"0000:41:00.4", b"41:00.0", 0, NO_PF),            # no domain
    (b"0000:41:00.4", b"0000:e1:00.0", 0, NO_PF),       # a PF outside the walk
    (b"0000:81:00.0", b"0000:81:00.0", 0, NO_PF),       # a link to its own parent, which is in the walk
    (b"0000:41:00.4", b"0000:81:00.0", 0, 5),
    (b"0000:41:00.4", b"0000:c1:00.0", 0, 3),
])
def test_join_hand_cases(parent, physfn, flags, want):
    m, s = PC.mdevs([(parent, physfn, flags)])
    assert join(PC.walk(WALK), m, s) == [want]


def test_join_lowest_index_and_edges():
    walk = PC.walk([b"0000:41:00.1", b"0000:41:00.0", b"junk", b"0000:41:00.0", b"0000:41:00.0"])
    m, s = PC.mdevs([(b"0000:41:00.1", b"0000:41:00.0", 0), (b"0000:41:00.2", b"junk", 0),
                     (b"0000:41:00.0", b"0000:41:00.1", 0)])
    assert join(walk, m, s) == [1, NO_PF, 0]
    assert join(PC.walk([]), m, s) == [NO_PF] * 3  # no PCI records
    assert join(walk, *PC.mdevs([])) == []
    # full 16-byte fields without a NUL never match a canonical address
    m, s = PC.mdevs([(b"0000:41:00.2", b"0000:41:00.0abcd", 0)])
    assert join(walk, m, s) == [NO_PF]


def test_join_workload_small():
    from kxpu_b200 import workloads as W
    recs, m, s, want = W.mdev_pf_walk(1 << 12, 1 << 7, 1 << 12, seed=3)
    assert join(recs, m, s) == want.tolist()
    assert 0 < int((want == NO_PF).sum()) < len(want)


_addr = st.one_of(st.sampled_from(WALK + [b"0000:e1:00.0", b"", b"0000:41:00.4"]), st.binary(max_size=16),
                  st.tuples(st.integers(0, 3), st.integers(0, 0x1f), st.integers(0, 7)).map(
                      lambda t: b"0000:4%d:%02x.%d" % t))


@settings(max_examples=300, deadline=None)
@given(st.lists(_addr, max_size=40), st.lists(st.tuples(_addr, _addr, st.sampled_from([0, 0, 1, 2])), max_size=60))
def test_join_fuzz(walk, pairs):
    join(PC.walk([w[:16] for w in walk]), *PC.mdevs([(p[:15], f[:16], fl) for p, f, fl in pairs]))


# ---------------------------------------------------------------- kxpu_dra_slices_mdev_pf

def test_golden_cfg1():
    want = open(GOLDEN, "rb").read()
    c = PC.CFG1
    blob, offs = both(c["driver"], c["pool"], c["node"], c["gen"], PC.cfg1())
    assert blob == want and list(offs) == [0, len(want)]
    devs = check_schema(blob, offs, 2)[0]["spec"]["devices"]
    a0, a1 = devs[0]["attributes"], devs[1]["attributes"]
    assert a0["physfnAddress"] == {"string": "0000:41:00.0"} and a0["physfnDeviceID"] == {"string": "2330"}
    assert a0["parentAddress"] == {"string": "0000:41:00.4"} and "parentDeviceID" not in a0
    assert a0["productName"] == {"string": "GH100_H100_SXM5_80GB"}
    assert "physfnAddress" not in a1 and "physfnDeviceID" not in a1


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000])
def test_sizes_mixed(n):
    devs = PC.random_devs(n, seed=n)
    devs["dev"]["iommu_group"] = np.arange(n)
    check_schema(*both("vgpu.nvidia.com", "node-a", "node-a", 7, devs), n)


@pytest.mark.parametrize("table", [PC.TAINTS1, PC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129])
def test_sizes_tainted(table, n):
    devs = PC.random_devs(n, seed=100 + n)
    since = np.stack([TC.since_pattern(n, "some", seed=t) for t in range(len(table))], axis=1) if n else \
        np.zeros((0, len(table)), np.int64)
    if len(table) == 3:
        since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    blob, offs = both("vgpu.nvidia.com", "node-a", "node-a", 3, devs, table, since)
    assert len(lines(blob)) == max(1, -(-n // 64))


@pytest.mark.parametrize("per", [64, 128])
def test_every_attribute_at_the_seams(per):
    """around each slice edge, one device per combination of the optional attributes"""
    n = 3 * per + 2
    devs = PC.random_devs(n, seed=per, all_attrs=True)
    for i in range(n):
        k = i % 32
        d = devs[i]["dev"]
        if k & 1: d["numa_mask"] = 0
        if k & 2: d["device"] = b""
        if k & 4: d["product_len"] = 0
        if k & 8: d["pcie_root"] = b""
        if k & 16: devs[i]["physfn"], devs[i]["physfn_device"] = b"", b""
        elif k & 1: devs[i]["physfn_device"] = b""
    since = None if per == 128 else np.where(np.arange(n)[:, None] % 3 == 0, 5, -1).astype(np.int64)
    table = PC.TAINTS1 if per == 64 else ()
    blob, offs = both("d", "p", "n", 1, devs, table, since)
    seen = set()
    for o in lines(blob):
        for dv in o["spec"]["devices"]:
            seen.add(tuple(a in dv["attributes"] for a in ATTRS))
    assert len(seen) == 32  # 16 of the mdev attributes, times physfn present (its id with it or not) or absent


@pytest.mark.parametrize("n", [0, 1, 64, 65, 128, 129, 300])
@pytest.mark.parametrize("taints", ["null", "1"])
def test_empty_physfn_is_the_mdev_layout(n, taints):
    """with every physfn empty the bytes are the mdev layout's (its untainted and one-taint statements; the GPU tests
    compare whole taint tables against kxpu_dra_slices_mdev_taints)"""
    devs = PC.random_devs(n, seed=n, no_physfn=True)
    if taints == "null":
        blob, want = both("d", "p", "n", 1, devs), PM.slices("d", "p", "n", 1, devs["dev"])
    else:
        since = np.where(np.arange(n) % 5 == 0, 9, -1).astype(np.int64)
        blob = both("d", "p", "n", 1, devs, PC.TAINTS1, since.reshape(n, 1))
        want = PT.slices_mdev("d", "p", "n", 1, devs["dev"], *PC.TAINTS1[0], since)
    assert blob[0] == want[0] and list(blob[1]) == list(want[1])


def test_longest_fields():
    devs = PC.random_devs(300, seed=5, all_attrs=True)
    blob, offs = both(LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1, devs)
    for o in check_schema(blob, offs, 300, unique=False):
        for d in o["spec"]["devices"]:
            assert list(d["attributes"]) == ATTRS
            assert len(d["attributes"]["physfnAddress"]["string"]) == 16
            assert len(d["attributes"]["physfnDeviceID"]["string"]) == 6


@pytest.mark.parametrize("why,field,value", PC.BAD)
def test_out_of_domain(why, field, value):
    devs = np.concatenate([PC.cfg1(), PC.bad_rec(field, value)])
    assert both("d", "p", "n", 1, devs) == (-7, why)
    assert both("d", "p", "n", 1, devs, PC.TAINTS1, np.full((3, 1), -1, np.int64)) == (-7, why)


def test_physfn_device_without_physfn():
    assert both("d", "p", "n", 1, PC.bad_rec("physfn_device", b"2330", physfn=b"")) == (-7, "physfn_device")


@pytest.mark.parametrize("why,field,value", MC.BAD)
def test_out_of_domain_dev(why, field, value):
    """the dev's refusals are the mdev layout's, in its order"""
    r = PC.rec()
    r["dev"] = MC.bad_rec(field, value)
    assert both("d", "p", "n", 1, np.concatenate([PC.cfg1(), r])) == (-7, why)


@pytest.mark.parametrize("args", [("d" * 64, "p", "n", 1), ("Vfio", "p", "n", 1), ("d", "p", "n.", 1), ("d", "p", "n", 1 << 63)])
def test_invalid_arguments(args):
    assert both(*args, PC.cfg1()) == -1


@pytest.mark.parametrize("key,value,effect", TC.INVALID)
def test_invalid_taint_arguments(key, value, effect):
    assert both("d", "p", "n", 1, PC.cfg1(), [(key, value, effect)], np.zeros((2, 1), np.int64)) == -1


def test_since_and_duplicate():
    devs = PC.cfg1()
    assert both("d", "p", "n", 1, devs, PC.TAINTS3, np.array([[-1, -1, -1], [TC.SINCE_MAX + 1, -1, -1]])) == \
        (-7, "taint_since")
    assert both("d", "p", "n", 1, devs, PC.TAINTS3, np.array([[-1, 5, 6], [-1, -1, -1]])) == (-7, "taint_duplicate")


def test_layout_matches_header(tmp_path):
    """offsetof / sizeof / alignof of kxpu_dramdevpf in include/kxpu.h == the binding's dtype"""
    from kxpu_b200.binding import DRAMDEVPF_DTYPE as D
    src = tmp_path / "layout.c"
    fields = list(D.names)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu", '
                   'sizeof(kxpu_dramdevpf), _Alignof(kxpu_dramdevpf));%sreturn 0;}\n'
                   % (os.path.join(ROOT, "include", "kxpu.h"),
                      "".join('printf(" %%zu", offsetof(kxpu_dramdevpf, %s));' % f for f in fields)))
    exe = tmp_path / "layout"
    subprocess.check_call([os.environ.get("CC", "gcc"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [240, 8] + [D.fields[f][1] for f in fields]


def test_header_declares_the_calls():
    import kxpu_b200.binding as B
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    for sym in ("kxpu_mdev_pf", "kxpu_dra_slices_mdev_pf"):
        assert "int32_t %s(" % sym in hdr and sym in B.ABI_SYMBOLS


@st.composite
def _rec(draw):
    valid = draw(st.booleans())
    r = PC.random_devs(1, seed=draw(st.integers(0, 1 << 20)))
    addr = st.text("0123456789abcdef:.", max_size=16).map(str.encode)
    dev = st.text("0123456789abcdef", max_size=6).map(str.encode)
    if not valid:
        addr, dev = st.one_of(addr, st.binary(max_size=16)), st.one_of(dev, st.binary(max_size=8))
    pf = draw(addr)[:16]
    r["physfn"], r["physfn_device"] = pf, (draw(dev)[:8] if pf or not valid else b"")
    if not valid and draw(st.booleans()):
        r["dev"]["iommu_group"] = draw(st.sampled_from([0, 0xFFFFFFFF]))
    return r


_since = st.one_of(st.integers(-(1 << 63), -1), st.integers(0, TC.SINCE_MAX), st.just(TC.SINCE_MAX + 1))


@settings(max_examples=200, deadline=None)
@given(st.lists(_rec(), max_size=150), st.sampled_from(["null", "1", "3"]), st.data())
def test_fuzz_oracle_vs_pyref(recs, table, data):
    devs = np.concatenate(recs) if recs else np.zeros(0, PC.DRAMDEVPF_DTYPE)
    taints = {"null": PC.TAINTS3, "1": PC.TAINTS1, "3": PC.TAINTS3}[table]
    since = None
    if table != "null":
        since = np.array(data.draw(st.lists(_since, min_size=len(devs) * len(taints), max_size=len(devs) * len(taints))),
                         np.int64).reshape(len(devs), len(taints))
    both("vgpu.nvidia.com", "node-a", "node-a", 2, devs, taints, since)
