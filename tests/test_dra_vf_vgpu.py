"""CPU tests of the DRA ResourceSlices of vGPUs on SR-IOV VFs (kxpu_dra_slices_vf_vgpu, include/kxpu.h, addition to ABI
v14): the C oracle (tests/dra_vf_vgpu_oracle.c) against the Python restatement (tests/pyref_dra_vf_vgpu.py) on hand
cases and under a hypothesis fuzz with taint tables of one and three entries and with taint_since NULL, the golden cfg1
line, the resource.k8s.io/v1 limits on every line, every domain refusal, the taint refusals, and the kxpu_dravfvgpu
layout."""
import json
import os
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import dra_taint_cases as TC
import dra_vf_vgpu_cases as VC
import dra_vf_vgpu_oracle as VO
import pyref_dra_vf_vgpu as PR
from conftest import ROOT
from test_dra import LONG_DRIVER, LONG_NAME, check_schema

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_vf_vgpu_cfg1.jsonl")
ATTRS = ["iommuGroup", "numaNode", "parentAddress", "parentDeviceID", "parentVendorID", "pciAddress", "productName",
         "resource.kubernetes.io/pcieRoot", "vgpuType", "vgpuTypeID"]


def both(driver, pool, node, gen, devs, taints=(), since=None):
    got = VO.dra_slices_vf_vgpu(driver, pool, node, gen, devs, taints, since)
    want = PR.slices(driver, pool, node, gen, devs, taints, since)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == want[1]
    else:
        assert got == want
    return got


def lines(blob):
    return [json.loads(x) for x in blob.split(b"\n")[:-1]]


def test_golden_cfg1():
    want = open(GOLDEN, "rb").read()
    blob, offs = both(**VC.CFG1, devs=VC.cfg1())
    assert blob == want and list(offs) == [0, len(want)]
    attrs = check_schema(blob, offs, 1)[0]["spec"]["devices"][0]["attributes"]
    assert list(attrs) == ATTRS
    assert attrs["parentDeviceID"] == {"string": "2330"} and attrs["productName"] == {"string": "GH100_H100_SXM5_80GB"}
    assert attrs["vgpuTypeID"] == {"int": 1058}


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000])
def test_sizes_mixed(n):
    devs = VC.random_devs(n, seed=n)
    devs["iommu_group"] = np.arange(n)  # unique names across the pool
    blob, offs = both("vgpu-vf.nvidia.com", "node-a", "node-a", 7, devs)
    objs = check_schema(blob, offs, n)
    if n == 0:
        assert objs[0]["spec"]["devices"] == []


@pytest.mark.parametrize("table", [VC.TAINTS1, VC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("kind", ["none", "some", "all"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 128, 129])
def test_sizes_tainted(table, kind, n):
    devs = VC.random_devs(n, seed=100 + n)
    since = np.stack([TC.since_pattern(n, kind, seed=t) for t in range(len(table))], axis=1) if n else \
        np.zeros((0, len(table)), np.int64)
    if len(table) == 3:  # the two AER entries share key and effect: a device carries at most one of them
        since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    blob, offs = both("vgpu-vf.nvidia.com", "node-a", "node-a", 3, devs, table, since)
    objs = lines(blob)
    assert len(objs) == len(offs) - 1 == max(1, -(-n // 64))
    tainted = sum(1 for o in objs for d in o["spec"]["devices"] if "taints" in d)
    assert tainted == int((since >= 0).any(axis=1).sum())


@pytest.mark.parametrize("n", [0, 1, 128, 129, 300])
def test_null_since_is_the_untainted_bytes(n):
    devs = VC.random_devs(n, seed=n)
    blob, offs = both("d", "p", "n", 1, devs, VC.TAINTS3, None)
    want, woffs = both("d", "p", "n", 1, devs)
    assert blob == want and np.array_equal(offs, woffs)


def test_timestamp_edges():
    devs = VC.random_devs(len(TC.EDGES), seed=1)
    since = TC.since_pattern(len(devs), "edges").reshape(-1, 1)
    blob, _ = both("d", "p", "n", 1, devs, VC.TAINTS1, since)
    got = [d["taints"][0]["timeAdded"] for d in lines(blob)[0]["spec"]["devices"]]
    assert got == [TC.EDGES[int(t)] for t in since[:, 0]]


def test_longest_fields():
    devs = VC.random_devs(300, seed=5, all_attrs=True)
    devs["iommu_group"] = 4294967294 - np.arange(300)
    blob, offs = both(LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1, devs)
    for o in check_schema(blob, offs, 300):
        for d in o["spec"]["devices"]:
            assert list(d["attributes"]) == ATTRS
            assert len(d["attributes"]["vgpuType"]["string"]) == 40


def test_optional_attributes():
    devs = np.concatenate([VC.rec(group=g, numa=m, device=dv, product=p, root=r) for g, (m, dv, p, r) in enumerate(
        [(0, b"", b"", b""), (1, b"2330", b"X", b"pci0000:00"), (1 << 63, b"", b"A" * 63, b""),
         (3, b"abcdef", b"B" * 64, b"pci10000:e0"), (1 << 5, b"1", b"", b"pci0000:c0")])])
    blob, offs = both("a", "b", "c", 0, devs)
    attrs = [d["attributes"] for d in check_schema(blob, offs, len(devs))[0]["spec"]["devices"]]
    assert list(attrs[0]) == ["iommuGroup", "parentAddress", "parentVendorID", "pciAddress", "vgpuType", "vgpuTypeID"]
    assert attrs[1]["numaNode"] == {"int": 0} and attrs[2]["numaNode"] == {"int": 63} and "numaNode" not in attrs[3]
    assert attrs[1]["parentDeviceID"] == {"string": "2330"} and "parentDeviceID" not in attrs[2]
    assert attrs[2]["productName"]["string"] == "A" * 63 and attrs[3]["productName"]["string"] == "B" * 64
    assert attrs[4]["resource.kubernetes.io/pcieRoot"] == {"string": "pci0000:c0"}


def test_full_width_fields():
    """a 40-byte key and 16-byte addresses fill their fields without a NUL; bytes past product_len are ignored"""
    r = VC.rec(type_key=b"T" * 40, bdf=b"0123456789abcdef", parent=b"fedcba9876543210", product=b"AB  \"\n", product_len=2,
               type_id=4294967295)
    blob, _ = both("d", "p", "n", 1, r)
    assert b'"vgpuType":{"string":"' + b"T" * 40 + b'"}' in blob and b'"productName":{"string":"AB"}' in blob
    assert b'"pciAddress":{"string":"0123456789abcdef"}' in blob
    assert b'"parentAddress":{"string":"fedcba9876543210"}' in blob and b'"vgpuTypeID":{"int":4294967295}' in blob


@pytest.mark.parametrize("args", [
    ("d" * 64, "p", "n", 1), ("Vfio", "p", "n", 1), ("a..b", "p", "n", 1), ("", "p", "n", 1),
    ("d", LONG_NAME + "x", "n", 1), ("d", "p", "n.", 1), ("d", "p", "n", 1 << 63)])
def test_invalid_arguments(args):
    assert both(*args, VC.cfg1()) == -1


@pytest.mark.parametrize("key,value,effect", TC.INVALID)
def test_invalid_taint_arguments(key, value, effect):
    assert both("d", "p", "n", 1, VC.cfg1(), [(key, value, effect)], np.zeros((1, 1), np.int64)) == -1


def test_invalid_taint_table_sizes():
    assert VO.dra_slices_vf_vgpu("d", "p", "n", 1, VC.cfg1(), [], np.zeros(0, np.int64)) == -1
    five = [("k%d" % t, "", "NoSchedule") for t in range(5)]
    assert VO.dra_slices_vf_vgpu("d", "p", "n", 1, VC.cfg1(), five, np.zeros((1, 5), np.int64)) == -1


@pytest.mark.parametrize("why,field,value", VC.BAD)
def test_out_of_domain(why, field, value):
    devs = np.concatenate([VC.cfg1(), VC.bad_rec(field, value)])
    assert both("d", "p", "n", 1, devs) == (-7, why)
    assert both("d", "p", "n", 1, devs, VC.TAINTS1, np.full((2, 1), -1, np.int64)) == (-7, why)


@pytest.mark.parametrize("t", [TC.SINCE_MAX + 1, 1 << 40, (1 << 63) - 1])
def test_since_above_year_9999(t):
    since = np.array([[-1, -1, -1], [-1, -1, t]], np.int64)
    assert both("d", "p", "n", 1, np.concatenate([VC.cfg1(), VC.cfg1()]), VC.TAINTS3, since) == (-7, "taint_since")


def test_duplicate_taint():
    since = np.array([[5, 6, 7]], np.int64)  # both AER entries on one device: same key and effect
    assert both("d", "p", "n", 1, VC.cfg1(), VC.TAINTS3, since) == (-7, "taint_duplicate")
    since = np.array([[5, -1, 7]], np.int64)
    blob, _ = both("d", "p", "n", 1, VC.cfg1(), VC.TAINTS3, since)
    assert [t["value"] for t in lines(blob)[0]["spec"]["devices"][0]["taints"]] == ["vfio-device-missing", "nonfatal"]


def test_layout_matches_header(tmp_path):
    """offsetof / sizeof / alignof of kxpu_dravfvgpu in include/kxpu.h == the binding's dtype"""
    from kxpu_b200.binding import DRAVFVGPU_DTYPE as D
    src = tmp_path / "layout.c"
    fields = list(D.names)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu", '
                   'sizeof(kxpu_dravfvgpu), _Alignof(kxpu_dravfvgpu));%sreturn 0;}\n'
                   % (os.path.join(ROOT, "include", "kxpu.h"),
                      "".join('printf(" %%zu", offsetof(kxpu_dravfvgpu, %s));' % f for f in fields)))
    exe = tmp_path / "layout"
    subprocess.check_call([os.environ.get("CC", "gcc"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [192, 8] + [D.fields[f][1] for f in fields]


def test_header_declares_the_call():
    import kxpu_b200.binding as B
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert "int32_t kxpu_dra_slices_vf_vgpu(" in hdr and "kxpu_dra_slices_vf_vgpu" in B.ABI_SYMBOLS


_names = st.sampled_from(["a", "node-a", "x.y-z", LONG_NAME, "A", "a..b"])
_field = st.binary(max_size=16)


@st.composite
def _rec(draw):
    valid = draw(st.booleans())
    hexs = st.text("0123456789abcdef", min_size=1, max_size=6).map(str.encode)
    dev = st.text("0123456789abcdef", max_size=6).map(str.encode)
    name = st.text("ABCxyz019_.-", max_size=64).map(str.encode)
    key = st.text("ABCxyz019_.-", min_size=1, max_size=40).map(str.encode)
    addr = st.text("0123456789abcdef:.", min_size=1, max_size=16).map(str.encode)
    root = st.one_of(st.just(b""), st.text("0123456789abcdef:", min_size=1, max_size=13).map(lambda s: b"pci" + s.encode()))
    numa = st.one_of(st.just(0), st.integers(0, 63).map(lambda k: 1 << k), st.integers(0, (1 << 64) - 1))
    group = st.integers(0, 0xFFFFFFFE) if valid else st.integers(0, 0xFFFFFFFF)
    tid = st.integers(1, 0xFFFFFFFF) if valid else st.integers(0, 0xFFFFFFFF)
    bdf, parent = addr, addr
    if not valid:
        hexs, dev, name, root = _field, _field, st.binary(max_size=64), st.one_of(root, _field)
        key, bdf, parent = st.one_of(key, st.binary(max_size=40)), st.one_of(addr, _field), st.one_of(addr, _field)
    r = VC.rec(group=draw(group), type_key=draw(key)[:40], type_id=draw(tid), bdf=draw(bdf)[:16], parent=draw(parent)[:16],
               root=draw(root)[:16], vendor=draw(hexs)[:8], device=draw(dev)[:8], product=draw(name), numa=draw(numa))
    if not valid and draw(st.booleans()):
        r["product_len"] = draw(st.integers(0, 255))
    return r


_since = st.one_of(st.integers(-(1 << 63), -1), st.integers(0, TC.SINCE_MAX), st.just(TC.SINCE_MAX + 1))


@settings(max_examples=300, deadline=None)
@given(st.lists(_rec(), max_size=200), _names, _names, st.integers(0, (1 << 64) - 1),
       st.sampled_from(["null", "1", "3"]), st.data())
def test_fuzz_oracle_vs_pyref(recs, driver, node, gen, table, data):
    devs = np.concatenate(recs) if recs else np.zeros(0, VC.rec().dtype)
    taints, since = {"null": (VC.TAINTS3, None), "1": (VC.TAINTS1, None), "3": (VC.TAINTS3, None)}[table]
    if table != "null":
        since = np.array(data.draw(st.lists(_since, min_size=len(devs) * len(taints), max_size=len(devs) * len(taints))),
                         np.int64).reshape(len(devs), len(taints))
    got = both(driver, "pool", node, gen, devs, taints, since)
    if isinstance(got, tuple) and isinstance(got[0], bytes) and since is None:
        objs = check_schema(got[0], got[1], len(devs), unique=False)
        assert sum(len(o["spec"]["devices"]) for o in objs) == len(devs)
