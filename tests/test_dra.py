"""CPU tests of the DRA ResourceSlices (kxpu_dra_slices, include/kxpu.h ABI v9): the C oracle
(oracle/kxpu_dra_oracle.c) against the Python restatement (tests/pyref_dra.py) on hand cases and under a hypothesis
fuzz, the golden cfg1 line, a schema check of every line from the resource.k8s.io/v1 limits as include/kxpu.h states
them, and the kxpu_dradev layout."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import dra_cases as DC
import pyref_dra as PR
from oracle import dra_oracle as DO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_cfg1.jsonl")
LONG_DRIVER = "d" * 63
LONG_NAME = ".".join(["a" * 63] * 3 + ["b" * 61])  # 253 bytes, labels of at most 63
assert len(LONG_NAME) == 253
_DNS_LABEL = re.compile(r"[a-z0-9]([-a-z0-9]{0,61}[a-z0-9])?\Z")
_C_IDENT = re.compile(r"[A-Za-z_][A-Za-z0-9_]{0,31}\Z")


def check_schema(blob, offs, n, unique=True):
    """every line a ResourceSlice within the v1 limits (include/kxpu.h [assumed] list); returns the parsed objects.
    unique=False: the input may repeat a group, so names are not checked for uniqueness"""
    assert offs[0] == 0 and offs[-1] == len(blob)
    lines = blob.split(b"\n")
    assert lines[-1] == b""
    lines = lines[:-1]
    assert len(lines) == len(offs) - 1 == max(1, -(-n // 128))
    objs, names, gens = [], set(), set()
    for s, line in enumerate(lines):
        assert blob[offs[s]:offs[s + 1]] == line + b"\n"
        o = json.loads(line)
        assert list(o) == ["kind", "apiVersion", "metadata", "spec"]
        assert o["kind"] == "ResourceSlice" and o["apiVersion"] == "resource.k8s.io/v1"
        spec = o["spec"]
        assert list(spec) == ["driver", "pool", "nodeName", "devices"]
        assert list(spec["pool"]) == ["name", "generation", "resourceSliceCount"]
        assert spec["pool"]["resourceSliceCount"] == len(lines)
        gens.add(spec["pool"]["generation"])
        assert len(spec["devices"]) <= 128
        for d in spec["devices"]:
            assert list(d) == ["name", "attributes"]
            assert _DNS_LABEL.match(d["name"]) and (not unique or d["name"] not in names)
            names.add(d["name"])
            attrs = d["attributes"]
            assert len(attrs) <= 32 and list(attrs) == sorted(attrs)
            for k, v in attrs.items():
                assert _C_IDENT.match(k) or k == "resource.kubernetes.io/pcieRoot"
                assert len(v) == 1 and list(v)[0] in ("int", "bool", "string", "version")
                if "string" in v:
                    assert len(v["string"].encode()) <= 64
        objs.append(o)
    assert len(gens) == 1
    return objs


def both(driver, pool, node, gen, devs):
    got, want = DO.dra_slices(driver, pool, node, gen, devs), PR.slices(driver, pool, node, gen, devs)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == want[1]
    else:
        assert got == want
    return got


def test_golden_cfg1():
    want = open(GOLDEN, "rb").read()
    blob, offs = both(**DC.CFG1, devs=DC.cfg1())
    assert blob == want and list(offs) == [0, len(want)]
    check_schema(blob, offs, 1)


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000])
def test_sizes_mixed(n):
    devs = DC.random_devs(n, seed=n)
    devs["iommu_group"] = np.arange(n)  # unique names across the pool
    blob, offs = both("vfio.nvidia.com", "node-a", "node-a", 7, devs)
    objs = check_schema(blob, offs, n)
    if n == 0:
        assert objs[0]["spec"]["devices"] == []


def test_optional_attributes():
    devs = np.concatenate([DC.rec(group=g, numa=m, product=p, root=r) for g, (m, p, r) in enumerate(
        [(0, b"", b""), (1, b"X", b"pci0000:00"), (1 << 63, b"A" * 63, b""), (3, b"B" * 64, b"pci10000:e0"),
         (1 << 5, b"", b"pci0000:c0")])])
    blob, offs = both("a", "b", "c", 0, devs)
    attrs = [d["attributes"] for d in check_schema(blob, offs, len(devs))[0]["spec"]["devices"]]
    assert "numaNode" not in attrs[0] and "productName" not in attrs[0] and "resource.kubernetes.io/pcieRoot" not in attrs[0]
    assert attrs[1]["numaNode"] == {"int": 0} and attrs[2]["numaNode"] == {"int": 63} and "numaNode" not in attrs[3]
    assert attrs[2]["productName"]["string"] == "A" * 63 and attrs[3]["productName"]["string"] == "B" * 64
    assert attrs[4]["resource.kubernetes.io/pcieRoot"] == {"string": "pci0000:c0"}


def test_groups_and_long_names():
    devs = np.concatenate([DC.rec(group=0), DC.rec(group=4294967294)])
    blob, offs = both(LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1, devs)
    o = check_schema(blob, offs, 2)[0]
    assert [d["name"] for d in o["spec"]["devices"]] == ["vfio0", "vfio4294967294"]
    assert o["spec"]["pool"]["generation"] == (1 << 63) - 1


@pytest.mark.parametrize("args", [
    ("d" * 64, "p", "n", 1), ("Vfio", "p", "n", 1), ("a..b", "p", "n", 1), ("-a", "p", "n", 1), ("a-", "p", "n", 1),
    ("", "p", "n", 1), ("a_b", "p", "n", 1), ("d", LONG_NAME + "x", "n", 1), ("d", "p", LONG_NAME + "x", 1),
    ("d", "a" * 64, "n", 1), ("d", "p", "n.", 1), ("d", "p", "n", 1 << 63)])
def test_invalid_arguments(args):
    assert both(*args, DC.cfg1()) == -1


@pytest.mark.parametrize("why,field,value", DC.BAD)
def test_out_of_domain(why, field, value):
    devs = np.concatenate([DC.cfg1(), DC.bad_rec(field, value)])
    assert both("d", "p", "n", 1, devs) == (-7, why)


def test_bytes_past_product_len_ignored():
    r = DC.rec(product=b"AB  \"\n", product_len=2)
    blob, _ = both("d", "p", "n", 1, r)
    assert b'"productName":{"string":"AB"}' in blob


def test_layout_matches_header(tmp_path):
    """offsetof / sizeof of kxpu_dradev in include/kxpu.h == the dtypes of the binding and the checker"""
    import kxpu_b200.binding as B
    assert B.DRADEV_DTYPE == DO.DRADEV_DTYPE
    src = tmp_path / "layout.c"
    fields = [f for f in DO.DRADEV_DTYPE.names]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu", sizeof(kxpu_dradev));%s'
                   'return 0;}\n' % (os.path.join(os.path.dirname(DO._HERE), "include", "kxpu.h"),
                                     "".join('printf(" %%zu", offsetof(kxpu_dradev, %s));' % f for f in fields)))
    exe = tmp_path / "layout"
    subprocess.check_call([os.environ.get("CC", "gcc"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [DO.DRADEV_DTYPE.itemsize] + [DO.DRADEV_DTYPE.fields[f][1] for f in fields]


_names = st.sampled_from(["a", "node-a", "x.y-z", LONG_NAME, "A", "a..b", "a" * 64])
_field = st.binary(max_size=16)


@st.composite
def _rec(draw):
    valid = draw(st.booleans())
    hexs = st.text("0123456789abcdef", min_size=1, max_size=6).map(str.encode)
    prod = st.text("ABCxyz019_.-", max_size=64).map(str.encode)
    bdf = st.text("0123456789abcdef:.", min_size=1, max_size=16).map(str.encode)
    root = st.one_of(st.just(b""), st.text("0123456789abcdef:", min_size=1, max_size=13).map(lambda s: b"pci" + s.encode()))
    numa = st.one_of(st.just(0), st.integers(0, 63).map(lambda k: 1 << k), st.integers(0, (1 << 64) - 1))
    group = st.integers(0, 0xFFFFFFFE) if valid else st.integers(0, 0xFFFFFFFF)
    if not valid:
        hexs, prod, bdf, root = _field, st.binary(max_size=64), _field, st.one_of(root, _field)
    p = draw(prod)
    r = DC.rec(group=draw(group), bdf=draw(bdf)[:16], vendor=draw(hexs)[:8], device=draw(hexs)[:8], product=p,
               root=draw(root)[:16], numa=draw(numa))
    if not valid and draw(st.booleans()):
        r["product_len"] = draw(st.integers(0, 255))
    return r


@settings(max_examples=300, deadline=None)
@given(st.lists(_rec(), max_size=300), _names, _names, st.integers(0, (1 << 64) - 1))
def test_fuzz_oracle_vs_pyref(recs, driver, node, gen):
    devs = np.concatenate(recs) if recs else np.zeros(0, DO.DRADEV_DTYPE)
    got = both(driver, "pool", node, gen, devs)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        objs = check_schema(got[0], got[1], len(devs), unique=False)
        assert sum(len(o["spec"]["devices"]) for o in objs) == len(devs)
