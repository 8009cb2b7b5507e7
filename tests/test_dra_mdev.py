"""CPU tests of the vGPU DRA ResourceSlices (kxpu_dra_slices_mdev, include/kxpu.h ABI v10): the C oracle
(oracle/kxpu_dra_mdev_oracle.c) against the Python restatement (tests/pyref_dra_mdev.py) on hand cases and under a
hypothesis fuzz, the golden cfg1 line, the resource.k8s.io/v1 limits on every line, every domain refusal, and the
kxpu_dramdev layout."""
import os
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import dra_mdev_cases as MC
import pyref_dra_mdev as PR
from oracle import dra_mdev_oracle as DO
from test_dra import LONG_DRIVER, LONG_NAME, check_schema

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_mdev_cfg1.jsonl")


def both(driver, pool, node, gen, devs):
    got, want = DO.dra_slices_mdev(driver, pool, node, gen, devs), PR.slices(driver, pool, node, gen, devs)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == want[1]
    else:
        assert got == want
    return got


def test_golden_cfg1():
    want = open(GOLDEN, "rb").read()
    blob, offs = both(**MC.CFG1, devs=MC.cfg1())
    assert blob == want and list(offs) == [0, len(want)]
    attrs = check_schema(blob, offs, 1)[0]["spec"]["devices"][0]["attributes"]
    assert list(attrs) == ["iommuGroup", "mdevType", "numaNode", "parentAddress", "parentDeviceID", "parentVendorID",
                           "productName", "resource.kubernetes.io/pcieRoot", "uuid"]


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000])
def test_sizes_mixed(n):
    devs = MC.random_devs(n, seed=n)
    devs["iommu_group"] = np.arange(n)  # unique names across the pool
    blob, offs = both("vgpu.nvidia.com", "node-a", "node-a", 7, devs)
    objs = check_schema(blob, offs, n)
    if n == 0:
        assert objs[0]["spec"]["devices"] == []


def test_longest_fields():
    devs = MC.random_devs(300, seed=5, all_attrs=True)
    devs["iommu_group"] = 4294967294 - np.arange(300)
    blob, offs = both(LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1, devs)
    for o in check_schema(blob, offs, 300):
        for d in o["spec"]["devices"]:
            assert len(d["attributes"]) == 9


def test_optional_attributes():
    devs = np.concatenate([MC.rec(group=g, numa=m, device=dv, product=p, root=r) for g, (m, dv, p, r) in enumerate(
        [(0, b"", b"", b""), (1, b"2330", b"X", b"pci0000:00"), (1 << 63, b"", b"A" * 63, b""),
         (3, b"abcdef", b"B" * 64, b"pci10000:e0"), (1 << 5, b"1", b"", b"pci0000:c0")])])
    blob, offs = both("a", "b", "c", 0, devs)
    attrs = [d["attributes"] for d in check_schema(blob, offs, len(devs))[0]["spec"]["devices"]]
    assert list(attrs[0]) == ["iommuGroup", "mdevType", "parentAddress", "parentVendorID", "uuid"]
    assert attrs[1]["numaNode"] == {"int": 0} and attrs[2]["numaNode"] == {"int": 63} and "numaNode" not in attrs[3]
    assert attrs[1]["parentDeviceID"] == {"string": "2330"} and "parentDeviceID" not in attrs[2]
    assert attrs[2]["productName"]["string"] == "A" * 63 and attrs[3]["productName"]["string"] == "B" * 64
    assert attrs[4]["resource.kubernetes.io/pcieRoot"] == {"string": "pci0000:c0"}


@pytest.mark.parametrize("args", [
    ("d" * 64, "p", "n", 1), ("Vfio", "p", "n", 1), ("a..b", "p", "n", 1), ("", "p", "n", 1),
    ("d", LONG_NAME + "x", "n", 1), ("d", "p", "n.", 1), ("d", "p", "n", 1 << 63)])
def test_invalid_arguments(args):
    assert both(*args, MC.cfg1()) == -1


@pytest.mark.parametrize("why,field,value", MC.BAD)
def test_out_of_domain(why, field, value):
    devs = np.concatenate([MC.cfg1(), MC.bad_rec(field, value)])
    assert both("d", "p", "n", 1, devs) == (-7, why)


def test_full_width_fields():
    """a 40-byte type and a 16-byte parent fill their fields without a NUL; bytes past product_len are ignored"""
    r = MC.rec(mdev_type=b"T" * 40, parent=b"0123456789abcdef", product=b"AB  \"\n", product_len=2)
    blob, _ = both("d", "p", "n", 1, r)
    assert b'"mdevType":{"string":"' + b"T" * 40 + b'"}' in blob and b'"productName":{"string":"AB"}' in blob
    assert b'"parentAddress":{"string":"0123456789abcdef"}' in blob


def test_layout_matches_header(tmp_path):
    """offsetof / sizeof / alignof of kxpu_dramdev in include/kxpu.h == the dtypes of the binding and the checker"""
    import kxpu_b200.binding as B
    assert B.DRAMDEV_DTYPE == DO.DRAMDEV_DTYPE
    src = tmp_path / "layout.c"
    fields = list(DO.DRAMDEV_DTYPE.names)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu", sizeof(kxpu_dramdev), '
                   '_Alignof(kxpu_dramdev));%sreturn 0;}\n'
                   % (os.path.join(os.path.dirname(DO._HERE), "include", "kxpu.h"),
                      "".join('printf(" %%zu", offsetof(kxpu_dramdev, %s));' % f for f in fields)))
    exe = tmp_path / "layout"
    subprocess.check_call([os.environ.get("CC", "gcc"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [208, 8] + [DO.DRAMDEV_DTYPE.fields[f][1] for f in fields]


_names = st.sampled_from(["a", "node-a", "x.y-z", LONG_NAME, "A", "a..b"])
_field = st.binary(max_size=16)


@st.composite
def _rec(draw):
    valid = draw(st.booleans())
    hexs = st.text("0123456789abcdef", min_size=1, max_size=6).map(str.encode)
    dev = st.text("0123456789abcdef", max_size=6).map(str.encode)
    name = st.text("ABCxyz019_.-", max_size=64).map(str.encode)
    mtype = st.text("ABCxyz019_.-", min_size=1, max_size=40).map(str.encode)
    uuid = st.sampled_from([MC.UUID, b"00000000-0000-0000-0000-000000000000", b"ffffffff-ffff-ffff-ffff-ffffffffffff"])
    parent = st.text("0123456789abcdef:.", min_size=1, max_size=16).map(str.encode)
    root = st.one_of(st.just(b""), st.text("0123456789abcdef:", min_size=1, max_size=13).map(lambda s: b"pci" + s.encode()))
    numa = st.one_of(st.just(0), st.integers(0, 63).map(lambda k: 1 << k), st.integers(0, (1 << 64) - 1))
    group = st.integers(0, 0xFFFFFFFE) if valid else st.integers(0, 0xFFFFFFFF)
    if not valid:
        hexs, dev, name, parent, root = _field, _field, st.binary(max_size=64), _field, st.one_of(root, _field)
        mtype, uuid = st.one_of(mtype, st.binary(max_size=40)), st.one_of(uuid, st.binary(min_size=36, max_size=36))
    r = MC.rec(group=draw(group), mdev_type=draw(mtype)[:40], uuid=draw(uuid)[:36], parent=draw(parent)[:16],
               root=draw(root)[:16], vendor=draw(hexs)[:8], device=draw(dev)[:8], product=draw(name), numa=draw(numa))
    if not valid and draw(st.booleans()):
        r["product_len"] = draw(st.integers(0, 255))
    return r


@settings(max_examples=300, deadline=None)
@given(st.lists(_rec(), max_size=300), _names, _names, st.integers(0, (1 << 64) - 1))
def test_fuzz_oracle_vs_pyref(recs, driver, node, gen):
    devs = np.concatenate(recs) if recs else np.zeros(0, DO.DRAMDEV_DTYPE)
    got = both(driver, "pool", node, gen, devs)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        objs = check_schema(got[0], got[1], len(devs), unique=False)
        assert sum(len(o["spec"]["devices"]) for o in objs) == len(devs)
