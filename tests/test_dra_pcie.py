"""CPU tests of kxpu_pcie_ports and kxpu_dra_slices_pcie (include/kxpu.h, additions to ABI v14): the C checker
(tests/dra_pcie_oracle.c) against the Python restatement (tests/pyref_dra_pcie.py) on the rule's hand cases, on seeded
walks and under hypothesis; the slices on the golden cfg1 line, at the slice seams, with 1- and 3-entry taint tables,
at every position of the two names, with 16-byte addresses, and with every key absent against kxpu_dra_slices_pf's and
kxpu_dra_slices_taints' checkers; every refusal; and the kxpu_dradevpcie layout."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import dra_pcie_cases as CC
import dra_pcie_oracle as CO
import dra_pf_cases as PC
import dra_pf_oracle as PO
import pyref_dra_pcie as PR
from conftest import ROOT
from oracle import aer_oracle as AO
from test_dra_pf import since_for

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_pcie_cfg1.jsonl")
NINE = ["deviceID", "iommuGroup", "numaNode", "pciAddress", "physfnAddress", "physfnDeviceID", "productName",
        "resource.kubernetes.io/pcieRoot", "vendorID"]


_QUALIFIED = re.compile(r"(([a-z0-9]([-a-z0-9]*[a-z0-9])?\.)*[a-z0-9]([-a-z0-9]*[a-z0-9])?/)?[A-Za-z_][A-Za-z0-9_]{0,31}\Z")


def check_schema(blob, offs, n, per=128):
    """test_dra.check_schema's slice checks, attribute names qualified by a domain allowed"""
    ls = blob.split(b"\n")
    assert ls[-1] == b"" and len(ls) - 1 == len(offs) - 1 == max(1, -(-n // per))
    objs = []
    for s, line in enumerate(ls[:-1]):
        assert blob[offs[s]:offs[s + 1]] == line + b"\n"
        o = json.loads(line)
        assert list(o) == ["kind", "apiVersion", "metadata", "spec"] and o["spec"]["pool"]["resourceSliceCount"] == len(ls) - 1
        for d in o["spec"]["devices"]:
            attrs = d["attributes"]
            assert list(d) == ["name", "attributes"] and len(attrs) <= 32 and list(attrs) == sorted(attrs)
            for k, v in attrs.items():
                assert _QUALIFIED.match(k) and len(k.split("/")[0]) <= 63, k
                assert len(v) == 1 and list(v)[0] in ("int", "string") and len(v.get("string", "").encode()) <= 64
        objs.append(o)
    return objs


def ports_both(walk):
    got, want = CO.pcie_ports(*walk), PR.pcie_ports(*walk)
    if isinstance(want, int):
        assert got == want
        return got
    assert list(got[0]) == want[0] and list(got[1]) == want[1]
    return want


def both(driver, pool, node, gen, domain, devs, taints=(), since=None):
    got = CO.dra_slices_pcie(driver, pool, node, gen, domain, devs, taints, since)
    want = PR.slices(driver, pool, node, gen, domain, devs, taints, since)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == want[1]
    else:
        assert got == want
    return got


def lines(blob):
    return [json.loads(x) for x in blob.split(b"\n")[:-1]]


@pytest.mark.parametrize("case", CC.HAND, ids=[c[0] for c in CC.HAND])
def test_rule_hand_cases(case):
    _, groups, want = case
    rp, sw = ports_both(CC.walk(groups))
    assert (rp, sw) == tuple(CC.expected(want))


@pytest.mark.parametrize("seed", range(8))
def test_rule_seeded_walks(seed):
    rp, sw = ports_both(CC.random_walk(400, seed))
    assert any(k != CC.NO for k in sw) and any(k == CC.NO for k in rp)


@settings(max_examples=60, deadline=None)
@given(st.integers(0, 60), st.integers(0, 2 ** 32 - 1), st.floats(0, 0.5), st.integers(1, 5))
def test_rule_hypothesis(groups, seed, unknown, members):
    ports_both(CC.random_walk(groups, seed, unknown, members))


def test_rule_refusals():
    recs, paths, off, mem = CC.walk([[("0000:01:00.0", None)], [("0000:02:00.0", None)]])
    assert ports_both((recs, paths, np.array([0, 2, 1], np.uint32), mem)) == -1  # offsets decrease
    assert ports_both((recs, paths, off, np.array([0, 2], np.uint32))) == -1     # a member >= n


def test_rule_vf_keeps_its_own_path():
    """the plain chains: a VF gets the ports its own path gives, which are its PF's (no placement below the PF)"""
    _, groups, want = CC.HAND[6]  # vf_beside_pf
    rp, sw = PR.pcie_ports(*CC.walk(groups))
    assert rp[1] == rp[2] and sw[1] == sw[2]


def test_golden_cfg1():
    want = open(GOLDEN, "rb").read()
    blob, offs = both("vfio.example.com", "node-a", "node-a", 1, CC.DOMAIN, CC.cfg1())
    assert blob == want and list(offs) == [0, len(want)]
    devs = check_schema(blob, offs, 4)[0]["spec"]["devices"]
    a = [d["attributes"] for d in devs]
    rp, sw = CC.DOMAIN + "/pcieRootPort", CC.DOMAIN + "/pcieSwitch"
    assert a[0][rp] == a[1][rp] == {"string": "0000:c0:01.0"} and a[0][sw] == a[1][sw] == {"string": "0000:c1:00.0"}
    assert a[2][rp] == {"string": "10000:e0:1d.0"} and sw not in a[2]
    assert rp not in a[3] and sw not in a[3]
    assert list(a[1]) == sorted(a[1])


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 1000])
def test_sizes_mixed(n):
    devs = CC.random_devs(n, seed=n)
    devs["pf"]["dev"]["iommu_group"] = np.arange(n)
    check_schema(*both("vfio.example.com", "node-a", "node-a", 7, CC.DOMAIN, devs), n)


@pytest.mark.parametrize("table", [PC.TAINTS1, PC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129])
def test_sizes_tainted(table, n):
    devs = CC.random_devs(n, seed=100 + n)
    blob, offs = both("vfio.example.com", "node-a", "node-a", 3, CC.DOMAIN, devs, table, since_for(table, n))
    assert len(lines(blob)) == max(1, -(-n // 64))


@pytest.mark.parametrize("pos", [p for p in range(10) if CC.POSITIONS[p]])
def test_every_position(pos):
    dom = CC.POSITIONS[pos]
    assert sum(k < dom + "/pcieRootPort" for k in NINE) == pos
    devs = CC.random_devs(200, seed=pos, all_attrs=pos % 2 == 0)
    for table, since in (((), None), (PC.TAINTS3, since_for(PC.TAINTS3, 200))):
        blob, _ = both("d", "p", "n", 1, dom, devs, table, since)
        for o in lines(blob):
            for d in o["spec"]["devices"]:
                keys = list(d["attributes"])
                assert keys == sorted(keys)
                if dom + "/pcieRootPort" in keys:
                    assert sum(k in NINE for k in keys[:keys.index(dom + "/pcieRootPort")]) == \
                        sum(k < dom for k in keys if k in NINE)


def test_no_domain_between_physfn_keys():
    """position 5 cannot occur: a lowercase domain that starts "physfn" sorts before physfnAddress or after
    physfnDeviceID"""
    for c in "-.0123456789abcdefghijklmnopqrstuvwxyz/":
        k = "physfn" + c
        assert not ("physfnAddress" < k < "physfnDeviceID")


@pytest.mark.parametrize("n", [1, 64, 65, 129])
def test_long_vmd_addresses(n):
    devs = CC.random_devs(n, seed=5, long_addr=True, all_attrs=True)
    blob, _ = both("d", "p", "n", 1, CC.DOMAIN, devs)
    for o in lines(blob):
        for d in o["spec"]["devices"]:
            assert len(d["attributes"][CC.DOMAIN + "/pcieRootPort"]["string"]) == 16


@pytest.mark.parametrize("n", [0, 1, 3, 64, 65, 128, 129, 300])
@pytest.mark.parametrize("table", [None, PC.TAINTS1, PC.TAINTS3], ids=["null", "1", "3"])
@pytest.mark.parametrize("dom", [CC.DOMAIN, "a.io", "w.io"])
def test_no_keys_is_the_pf_layout(n, table, dom):
    devs = CC.random_devs(n, seed=n, no_keys=True)
    since = None if table is None else since_for(table, n, seed=n)
    got = both("d", "p", "n", 1, dom, devs, table or (), since)
    want = PO.dra_slices_pf("d", "p", "n", 1, devs["pf"], table or (), since)
    assert got[0] == want[0] and list(got[1]) == list(want[1])
    devs = CC.random_devs(n, seed=n, no_keys=True, no_physfn=True)
    got = both("d", "p", "n", 1, dom, devs, table or (), since)
    want = AO.dra_slices_taints("d", "p", "n", 1, devs["pf"]["dev"], table or PC.TAINTS3, since)
    assert got[0] == want[0] and list(got[1]) == list(want[1])


@pytest.mark.parametrize("dom", CC.BAD_DOMAINS)
def test_bad_domain(dom):
    assert both("d", "p", "n", 1, dom, CC.cfg1()) == -1


@pytest.mark.parametrize("dom", CC.GOOD_DOMAINS)
def test_good_domain(dom):
    assert isinstance(both("d", "p", "n", 1, dom, CC.cfg1())[0], bytes)


@pytest.mark.parametrize("case", CC.BAD_KEYS)
def test_bad_keys(case):
    why, rp, sw = case
    devs = CC.cfg1()
    devs[2]["root_port"], devs[2]["pcie_switch"] = rp, sw
    assert both("d", "p", "n", 1, CC.DOMAIN, devs) == (-7, why)


def test_pf_rules_come_first():
    devs = CC.cfg1()
    devs[1]["pf"]["physfn"] = b"0000:C4:00.0"
    devs[1]["root_port"] = 1 << 63
    assert both("d", "p", "n", 1, CC.DOMAIN, devs) == (-7, "physfn")


@settings(max_examples=40, deadline=None)
@given(st.integers(0, 200), st.integers(0, 2 ** 31), st.sampled_from([None, 1, 3]),
       st.sampled_from([CC.DOMAIN] + [p for p in CC.POSITIONS if p]))
def test_hypothesis(n, seed, nt, dom):
    devs = CC.random_devs(n, seed)
    table = {None: (), 1: PC.TAINTS1, 3: PC.TAINTS3}[nt]
    both("d", "p", "n", 1, dom, devs, table, None if nt is None else since_for(table, n, seed=seed % 97))


def test_layout():
    src = r'''
#include <stddef.h>
#include <stdio.h>
#include "kxpu.h"
int main(void) {
    printf("%zu %zu %zu %zu %llx\n", sizeof(kxpu_dradevpcie), _Alignof(kxpu_dradevpcie),
           offsetof(kxpu_dradevpcie, root_port), offsetof(kxpu_dradevpcie, pcie_switch), KXPU_PCIE_NO_KEY);
    return 0;
}
'''
    import tempfile
    d = tempfile.mkdtemp()
    with open(os.path.join(d, "l.c"), "w") as f:
        f.write(src)
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "l"), os.path.join(d, "l.c")])
    out = subprocess.check_output([os.path.join(d, "l")]).decode().split()
    assert out == ["176", "8", "160", "168", "ffffffffffffffff"]
    from kxpu_b200.binding import DRADEVPCIE_DTYPE
    assert DRADEVPCIE_DTYPE.itemsize == 176 and DRADEVPCIE_DTYPE.fields["root_port"][1] == 160
