"""CPU tests of PCIe root ports and switches of vGPUs in DRA (include/kxpu.h, additions to ABI v14) on the Python
restatement (tests/pyref_vgpu_pcie.py): the vGPU rule on its hand cases, its invariant against kxpu_pcie_ports' rule on
the parents' own records, the names' positions among each layout's keys and the ones no lowercase domain reaches, the
bytes with every key absent against the mdev-PF and VF-vGPU restatements, and the hand-written golden lines."""
import os

import numpy as np

import pytest
from hypothesis import given, settings, strategies as st

import dra_vgpu_pcie_oracle as CO
import pyref_dra_pcie as PP
import pyref_dra_vf_vgpu as PV
import pyref_mdev_pf as PM
import pyref_vgpu_pcie as R
import vgpu_pcie_cases as CC

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("case", CC.HAND, ids=[c[0] for c in CC.HAND])
def test_rule_hand_cases(case):
    _, rows, groups, want = case
    assert R.pcie_ports_mdev(*CC.hand_walk(rows, groups)) == tuple(CC.expected(want))


@settings(max_examples=40, deadline=None)
@given(st.integers(0, 200), st.integers(0, 2 ** 31), st.integers(1, 4))
def test_rule_is_the_parents_ports(n, seed, per_group):
    mwalk, pwalk = CC.random_walk(n, seed, unknown=0, per_group=per_group)
    assert R.pcie_ports_mdev(*mwalk) == PP.pcie_ports(*pwalk)


@pytest.mark.parametrize("keys,positions", [(CC.MDEV_KEYS, CC.MDEV_POSITIONS), (CC.VF_KEYS, CC.VF_POSITIONS)])
def test_positions(keys, positions):
    assert len(positions) == len(keys) + 1
    for p, dom in enumerate(positions):
        if dom is not None:
            assert CC.position(keys, dom) == p
            continue
        # unreachable: the two neighbours first differ in an uppercase byte of each, so no lowercase name sorts
        # between them
        a, b = keys[p - 1], keys[p]
        t = next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), None)
        if t is None:  # a is a prefix of b: a name between them starts with a, which holds an uppercase byte
            assert b.startswith(a) and any(c.isupper() for c in a)
        else:
            assert a[t].isupper() and b[t].isupper()


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129])
@pytest.mark.parametrize("taints", [0, 1, 3])
def test_no_keys_give_the_parent_layouts_bytes(n, taints):
    tab = [("d.io/k%d" % t, "", "NoSchedule") for t in range(taints)]
    since = None if not taints else [[(i * 7 + t) % 3 - 1 for t in range(taints)] for i in range(n)]
    m = CC.random_mdev_devs(n, n, no_keys=True)
    assert R.slices("mdev", "d.io", "p", "n", 3, CC.DOMAIN, m, tab, since) == PM.slices("d.io", "p", "n", 3, m["pf"], tab,
                                                                                     since)
    v = CC.random_vf_devs(n, n, no_keys=True)
    assert R.slices("vf_vgpu", "d.io", "p", "n", 3, CC.DOMAIN, v, tab, since) == PV.slices("d.io", "p", "n", 3, v["dev"],
                                                                                        tab, since)


@pytest.mark.parametrize("layout,cfg,name", [("mdev", CC.mdev_cfg1, "dra_mdev_pcie_cfg1.jsonl"),
                                             ("vf_vgpu", CC.vf_cfg1, "dra_vf_vgpu_pcie_cfg1.jsonl")])
def test_golden(layout, cfg, name):
    want = open(os.path.join(GOLDEN, name), "rb").read()
    assert R.slices(layout, "vgpu.example.com", "node-a", "node-a", 1, CC.DOMAIN, cfg())[0] == want
    assert CO.slices(layout, "vgpu.example.com", "node-a", "node-a", 1, CC.DOMAIN, cfg())[0] == want


def test_refusals():
    m = CC.mdev_cfg1()
    for dom in [None, "", "Pcie.example.com", "kubernetes.io", "x.k8s.io", "a" * 64]:
        assert R.slices("mdev", "d.io", "p", "n", 1, dom, m) == -1
    bad = CC.mdev_cfg1()
    bad["root_port"][1], bad["pcie_switch"][1] = CC.NO, CC.fkey("0000:01:00.0")
    assert R.slices("mdev", "d.io", "p", "n", 1, CC.DOMAIN, bad) == (-7, "port_orphan")
    bad = CC.vf_cfg1()
    bad["root_port"][0] = 1 << 63 | 0x8000
    assert R.slices("vf_vgpu", "d.io", "p", "n", 1, CC.DOMAIN, bad) == (-7, "port_key")


# ------------------------------------------------------------------ the C checker against the Python restatement


@pytest.mark.parametrize("case", CC.HAND, ids=[c[0] for c in CC.HAND])
def test_c_rule_hand_cases(case):
    _, rows, groups, want = case
    rp, sw = CO.pcie_ports_mdev(*CC.hand_walk(rows, groups))
    assert (list(rp), list(sw)) == tuple(CC.expected(want))


@settings(max_examples=40, deadline=None)
@given(st.integers(0, 300), st.integers(0, 2 ** 31), st.floats(0, 0.3), st.integers(1, 5))
def test_c_rule_agrees(n, seed, unknown, per_group):
    walk, _ = CC.random_walk(n, seed, unknown, per_group)
    rp, sw = CO.pcie_ports_mdev(*walk)
    assert (list(rp), list(sw)) == R.pcie_ports_mdev(*walk)


@settings(max_examples=30, deadline=None)
@given(st.sampled_from(["mdev", "vf_vgpu"]), st.integers(0, 200), st.integers(0, 2 ** 31), st.integers(0, 3),
       st.sampled_from(CC.MDEV_POSITIONS[:4] + CC.VF_POSITIONS[5:]), st.booleans())
def test_c_slices_agree(layout, n, seed, nt, dom, long_addr):
    dom = dom or "x.io"
    devs = CC.random_mdev_devs(n, seed, long_addr=long_addr) if layout == "mdev" else \
        CC.random_vf_devs(n, seed, long_addr=long_addr)
    tab = [("d.io/k%d" % t, "", "NoSchedule") for t in range(nt)]
    since = None if not nt else np.where(np.random.default_rng(seed).random((n, nt)) < 0.3, 1767225600, -1)
    got = CO.slices(layout, "d.io", "p", "n", 2, dom, devs, tab, since)
    want = R.slices(layout, "d.io", "p", "n", 2, dom, devs, tab, since)
    assert got[0] == want[0] and list(got[1]) == list(want[1])


@pytest.mark.parametrize("layout,cfg", [("mdev", CC.mdev_cfg1), ("vf_vgpu", CC.vf_cfg1)])
def test_c_refusals(layout, cfg):
    bad = cfg()
    bad["root_port"][0], bad["pcie_switch"][0] = CC.NO, CC.fkey("0000:01:00.0")
    assert CO.slices(layout, "d.io", "p", "n", 1, CC.DOMAIN, bad) == (-7, "port_orphan")
    assert CO.slices(layout, "d.io", "p", "n", 1, "k8s.io", cfg()) == -1
