"""GPU tests of the PCIe topology calls (include/kxpu.h, ABI v7) against the CPU oracle (oracle/kxpu_pcie_oracle.c),
and of kxpu_preferred_allocation after its kernels were generalised to serve both calls."""
import numpy as np
import pytest

import pcie_example as EX
from oracle import pcie_oracle as PO
from oracle import topo_oracle as TO

pytestmark = pytest.mark.gpu
NO = PO.NO_NODE


def _same_tree(got, want):
    for k in ("group_node", "key", "parent", "depth"):
        assert np.array_equal(got[k], want[k]), k


@pytest.mark.parametrize("group_max", [1, 4])
def test_tree_2_20(kx, workloads, group_max):
    recs, paths, off, mem = workloads.pcie_walk(1 << 20, seed=21 + group_max, group_max=group_max)
    got = kx.pcie_tree(recs, paths, off, mem)
    _same_tree(got, PO.tree(recs, paths, off, mem))
    assert (got["group_node"] == NO).any() and len(np.unique(got["depth"])) == 8


def test_tree_example_and_edges(kx):
    recs, paths, off, mem = EX.records()
    _same_tree(kx.pcie_tree(recs, paths, off, mem), PO.tree(recs, paths, off, mem))
    empty = kx.pcie_tree(recs, paths, np.zeros(1, np.uint32), np.zeros(0, np.uint32))
    assert len(empty["key"]) == 0 and len(empty["group_node"]) == 0
    import kxpu_b200 as K
    for o, m in ((np.array([0, 2, 1, 8], np.uint32), mem), (off, np.array([0, 1, 2, 3, 4, 5, 6, 8], np.uint32))):
        with pytest.raises(K.KxpuError) as e:
            kx.pcie_tree(recs, paths, o, m)
        assert e.value.status == K.binding.E_INVALID


def _forest(kx, workloads, n, seed):
    """n devices, one group each, of a walk over n + n / 8 records (4 % of which are in no group)"""
    recs, paths, off, mem = workloads.pcie_walk(n + n // 8, seed=seed, group_max=1)
    t = kx.pcie_tree(recs, paths, off, mem)
    assert len(t["group_node"]) >= n
    return t["group_node"][:n].copy(), t["parent"], t["depth"]


def test_example_answers(kx):
    recs, paths, off, mem = EX.records()
    t = kx.pcie_tree(recs, paths, off, mem)
    got = kx.preferred_allocation_pcie(EX.DEV_NUMA, t["group_node"], t["parent"], t["depth"], EX.requests())
    assert got == EX.answers()


def test_alloc_warp_shape(kx, workloads):
    dev_node, parent, depth = _forest(kx, workloads, 4096, seed=31)
    dev_numa = workloads.topo_dev_numa(len(dev_node), nodes=4)
    reqs = workloads.topo_requests(dev_numa, n_req=4096, avail=16, size=8, must_max=2, seed=32)
    want = PO.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, reqs)
    assert kx.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, reqs) == want
    # local requests: the available devices of one bus (one switch), so that X is a deep node
    rng = np.random.default_rng(33)
    loc = []
    for _ in range(512):
        s = int(rng.integers(0, len(dev_node) - 300))
        av = (s + rng.permutation(256)[:int(rng.integers(1, 257))]).tolist()
        mu = av[:int(rng.integers(0, min(3, len(av)) + 1))]
        loc.append((av, mu, int(rng.integers(len(mu), len(av) + 1))))
    assert kx.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, loc) == \
        PO.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, loc)


def test_alloc_large_shape_2_20(kx, workloads):
    n = 1 << 20
    dev_node, parent, depth = _forest(kx, workloads, n, seed=41)
    dev_numa = workloads.topo_dev_numa(n, nodes=2)
    one = workloads.topo_requests(dev_numa, n_req=1, avail=n, size=n // 2, must_max=3, seed=42)
    assert kx.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, one) == \
        PO.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, one)
    part = workloads.topo_requests(dev_numa, n_req=3, avail=300000, size=1000, must_max=5, seed=43)
    assert kx.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, part) == \
        PO.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, part)
    # a large request inside one host bridge (64 buses = 16384 positions), a must-include device in it
    av = list(range(40000, 40000 + 16384))
    loc = [(av, [av[100]], 600), (av, [], 3), (av, [av[5], av[9000]], 20000 // 4)]
    assert kx.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, loc) == \
        PO.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, loc)


@pytest.mark.parametrize("avail", [16, 5000])
def test_alloc_identity_with_numa_rule(kx, workloads, avail):
    dev_node, parent, depth = _forest(kx, workloads, 1 << 14, seed=51)
    dev_numa = workloads.topo_dev_numa(len(dev_node), nodes=4)
    reqs = workloads.topo_requests(dev_numa, n_req=64 if avail == 16 else 2, avail=avail, size=avail // 2, must_max=2,
                                   seed=52)
    want = kx.preferred_allocation(dev_numa, reqs)
    assert want == TO.preferred_allocation(dev_numa, reqs)
    assert kx.preferred_allocation_pcie(dev_numa, None, parent, depth, reqs) == want
    none = np.full(len(dev_numa), NO, np.uint32)
    assert kx.preferred_allocation_pcie(dev_numa, none, parent, depth, reqs) == want


@pytest.mark.parametrize("big", [False, True])
def test_alloc_invalid_forest_writes_nothing(kx, big):
    import kxpu_b200 as K
    from kxpu_b200.binding import pref_requests
    n = 6000 if big else 8
    recs, paths, off, mem = EX.records()
    t = kx.pcie_tree(recs, paths, off, mem)
    good_node = np.full(n, NO, np.uint32)
    good_node[:8] = t["group_node"]
    cases = [(np.where(np.arange(n) == 3, 18, good_node).astype(np.uint32), t["parent"], t["depth"]),
             (good_node, np.where(np.arange(18) == 5, 7, t["parent"]).astype(np.uint32), t["depth"]),
             (good_node, t["parent"], np.where(np.arange(18) == 5, 2, t["depth"]).astype(np.uint8)),
             (good_node, np.where(np.arange(18) == 9, 0, t["parent"]).astype(np.uint32), t["depth"]),
             (good_node, t["parent"], np.where(np.arange(18) == 0, 8, t["depth"]).astype(np.uint8))]
    reqs = [(list(range(n)), [1], 4)]
    a = pref_requests(reqs)
    for dn, par, dep in cases:
        out = np.full(4, 0xABCD, np.uint32)
        with pytest.raises(K.KxpuError) as e:
            kx.preferred_allocation_pcie_raw(np.ones(n, np.uint64), dn, par, dep, a, out, np.zeros(2, np.uint32))
        assert e.value.status == K.binding.E_INVALID
        assert (out == 0xABCD).all()
    assert kx.preferred_allocation_pcie(np.ones(n, np.uint64), good_node, t["parent"], t["depth"], reqs) == \
        PO.preferred_allocation_pcie(np.ones(n, np.uint64), good_node, t["parent"], t["depth"], reqs)


def test_numa_rule_unchanged_by_generalisation(kx, workloads):
    """kxpu_preferred_allocation's answers after its kernels took the level parameter: both shapes against the
    NUMA oracle, with all-unknown and multi-node masks."""
    dev_numa = workloads.topo_dev_numa(1 << 16, nodes=4)
    reqs = workloads.topo_requests(dev_numa, n_req=2048, avail=200, size=100, must_max=4, seed=61)
    reqs += workloads.topo_requests(dev_numa, n_req=2, avail=20000, size=7000, must_max=4, seed=62)
    assert kx.preferred_allocation(dev_numa, reqs) == TO.preferred_allocation(dev_numa, reqs)
    zeros = np.zeros(len(dev_numa), np.uint64)
    assert kx.preferred_allocation(zeros, reqs) == TO.preferred_allocation(zeros, reqs)
