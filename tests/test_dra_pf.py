"""CPU tests of kxpu_dra_slices_pf (include/kxpu.h, an addition to ABI v14): the C oracle (tests/dra_pf_oracle.c)
against the Python restatement (tests/pyref_dra_pf.py) on the golden cfg1 line, at the slice seams with every attribute
present or absent, with 1- and 3-entry taint tables and under hypothesis; every domain refusal in the stated flag order;
the all-empty-physfn pool giving kxpu_dra_slices_taints' bytes (oracle/aer_oracle.py); and the kxpu_dradevpf layout."""
import json
import os
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import dra_cases as DC
import dra_pf_cases as PC
import dra_pf_oracle as PO
import dra_taint_cases as TC
import pyref_dra_pf as PR
from conftest import ROOT
from oracle import aer_oracle as AO
from test_dra import LONG_DRIVER, LONG_NAME, check_schema

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_pf_cfg1.jsonl")
ATTRS = ["deviceID", "iommuGroup", "numaNode", "pciAddress", "physfnAddress", "physfnDeviceID", "productName",
         "resource.kubernetes.io/pcieRoot", "vendorID"]


def both(driver, pool, node, gen, devs, taints=(), since=None):
    got = PO.dra_slices_pf(driver, pool, node, gen, devs, taints, since)
    want = PR.slices(driver, pool, node, gen, devs, taints, since)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == want[1]
    else:
        assert got == want
    return got


def lines(blob):
    return [json.loads(x) for x in blob.split(b"\n")[:-1]]


def since_for(table, n, seed=0):
    """one column per entry; the two pcie-aer entries (same key and effect) never on one device"""
    if n == 0:
        return np.zeros((0, len(table)), np.int64)
    since = np.stack([TC.since_pattern(n, "some", seed=seed + t) for t in range(len(table))], axis=1)
    if len(table) == 3:
        since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    return since


def test_golden_cfg1():
    want = open(GOLDEN, "rb").read()
    c = PC.CFG1
    blob, offs = both(c["driver"], c["pool"], c["node"], c["gen"], PC.cfg1())
    assert blob == want and list(offs) == [0, len(want)]
    devs = check_schema(blob, offs, 2)[0]["spec"]["devices"]
    a0, a1 = devs[0]["attributes"], devs[1]["attributes"]
    assert a0["physfnAddress"] == {"string": "0000:4d:00.0"} and a0["physfnDeviceID"] == {"string": "56c0"}
    assert a0["pciAddress"] == {"string": "0000:4d:00.1"}
    assert "physfnAddress" not in a1 and "physfnDeviceID" not in a1


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000])
def test_sizes_mixed(n):
    devs = PC.random_devs(n, seed=n)
    devs["dev"]["iommu_group"] = np.arange(n)
    check_schema(*both("vfio.example.com", "node-a", "node-a", 7, devs), n)


@pytest.mark.parametrize("table", [PC.TAINTS1, PC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129])
def test_sizes_tainted(table, n):
    devs = PC.random_devs(n, seed=100 + n)
    blob, offs = both("vfio.example.com", "node-a", "node-a", 3, devs, table, since_for(table, n))
    assert len(lines(blob)) == max(1, -(-n // 64))


@pytest.mark.parametrize("per", [64, 128])
def test_every_attribute_at_the_seams(per):
    """around each slice edge, one device per combination of the optional attributes"""
    n = 3 * per + 2
    devs = PC.random_devs(n, seed=per, all_attrs=True)
    for i in range(n):
        k = i % 16
        d = devs[i]["dev"]
        if k & 1: d["numa_mask"] = 0
        if k & 2: d["product_len"] = 0
        if k & 4: d["pcie_root"] = b""
        if k & 8: devs[i]["physfn"], devs[i]["physfn_device"] = b"", b""
        elif k & 1: devs[i]["physfn_device"] = b""
    since = None if per == 128 else np.where(np.arange(n)[:, None] % 3 == 0, 5, -1).astype(np.int64)
    table = PC.TAINTS1 if per == 64 else ()
    blob, offs = both("d", "p", "n", 1, devs, table, since)
    seen = set()
    for o in lines(blob):
        for dv in o["spec"]["devices"]:
            seen.add(tuple(a in dv["attributes"] for a in ATTRS))
    assert len(seen) == 16  # 8 of the PCI attributes, times physfn present (its id with it or not) or absent


@pytest.mark.parametrize("n", [0, 1, 3, 64, 65, 128, 129, 300])
@pytest.mark.parametrize("table", [None, PC.TAINTS1, PC.TAINTS3], ids=["null", "1", "3"])
def test_empty_physfn_is_the_taint_list_layout(n, table):
    """with every physfn empty both checkers give the existing taint-list checker's bytes for the devs"""
    devs = PC.random_devs(n, seed=n, no_physfn=True)
    taints = table or PC.TAINTS3
    since = None if table is None else since_for(table, n, seed=n)
    blob = both("d", "p", "n", 1, devs, taints if table else (), since)
    want = AO.dra_slices_taints("d", "p", "n", 1, devs["dev"], taints, since)
    assert blob[0] == want[0] and list(blob[1]) == list(want[1])


@pytest.mark.parametrize("n", [1, 3])
def test_non_vf_records_are_the_taint_list_layout(n):
    """a 1- or 3-entry pool of functions that are no VF, untainted and tainted"""
    devs = np.concatenate([PC.rec(group=g, bdf=b"0000:c%d:00.0" % g) for g in range(1, n + 1)])
    for table, since in ((None, None), (PC.TAINTS3, np.array([[5, -1, -1], [-1, 6, -1], [-1, -1, 7]])[:n])):
        got = both("d", "p", "n", 1, devs, table or (), since)
        want = AO.dra_slices_taints("d", "p", "n", 1, devs["dev"], table or PC.TAINTS3, since)
        assert got[0] == want[0] and list(got[1]) == list(want[1])


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
    assert both("d", "p", "n", 1, PC.bad_rec("physfn_device", b"56c0", physfn=b"")) == (-7, "physfn_device")


@pytest.mark.parametrize("why,field,value", DC.BAD)
def test_out_of_domain_dev(why, field, value):
    """the dev's refusals are kxpu_dra_slices', in its order, before the two new rules"""
    r = PC.bad_rec("physfn_device", b"1234567")  # breaks the last rule too
    r["dev"] = DC.bad_rec(field, value)
    assert both("d", "p", "n", 1, np.concatenate([PC.cfg1(), r])) == (-7, why)


def test_flag_order_of_the_new_rules():
    """a record that breaks both new rules reports physfn"""
    r = PC.bad_rec("physfn", b"0000:4D:00.0")
    r["physfn_device"] = b"56C0"
    assert both("d", "p", "n", 1, r) == (-7, "physfn")


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
    """offsetof / sizeof / alignof of kxpu_dradevpf in include/kxpu.h == the binding's dtype"""
    from kxpu_b200.binding import DRADEVPF_DTYPE as D
    src = tmp_path / "layout.c"
    fields = list(D.names)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu", '
                   'sizeof(kxpu_dradevpf), _Alignof(kxpu_dradevpf));%sreturn 0;}\n'
                   % (os.path.join(ROOT, "include", "kxpu.h"),
                      "".join('printf(" %%zu", offsetof(kxpu_dradevpf, %s));' % f for f in fields)))
    exe = tmp_path / "layout"
    subprocess.check_call([os.environ.get("CC", "gcc"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [160, 8] + [D.fields[f][1] for f in fields]


def test_header_declares_the_call():
    import kxpu_b200.binding as B
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert "int32_t kxpu_dra_slices_pf(" in hdr and "kxpu_dra_slices_pf" in B.ABI_SYMBOLS


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
    devs = np.concatenate(recs) if recs else np.zeros(0, PC.DRADEVPF_DTYPE)
    taints = {"null": PC.TAINTS3, "1": PC.TAINTS1, "3": PC.TAINTS3}[table]
    since = None
    if table != "null":
        since = np.array(data.draw(st.lists(_since, min_size=len(devs) * len(taints), max_size=len(devs) * len(taints))),
                         np.int64).reshape(len(devs), len(taints))
    both("vfio.example.com", "node-a", "node-a", 2, devs, taints, since)
