"""GPU tests of GetPreferredAllocation at its edges (csrc/topology.cu), against the C oracles
(oracle/kxpu_pcie_oracle.c, oracle/kxpu_topo_oracle.c) everywhere and the Python restatements where the sizes are
small:

  - every hand case of tests/pref_edge_cases.py in the one-warp shape as is, and in the large shape padded with null
    devices: both shapes must give the hand answer, with no oracle in between;
  - the shape boundary (255 .. 4097 available positions) alone and interleaved in one call, with out_off;
  - r on the tile seams of k_big_scatter at 4095 .. 3 * 4096 + 1 devices, with lca levels spread over the tiles;
  - k_pick over a forest larger than its first stage's threads, the winner in the last CTA's last stride;
  - several large PCIe requests in one call whose X, must-include set and lowest position differ;
  - the forests of kxpu_pcie_tree_mdev and kxpu_pcie_tree_sriov in both shapes;
  - identity with kxpu_preferred_allocation at the shape boundary and the seams;
  - the invalid requests of the large PCIe shape."""
import numpy as np
import pytest

import pref_edge_cases as E
import pyref_pcie as P
import pyref_topo as PT
from kxpu_b200.binding import E_INVALID, NO_PF, KxpuError, pref_requests
from oracle import pcie_oracle as PO
from oracle import topo_oracle as TO

pytestmark = pytest.mark.gpu
NO = E.NO


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def check_pcie(kx, numa, node, parent, depth, reqs, pyref=False):
    """The GPU answer of the PCIe call, equal to the C oracle's (and the Python restatement's)."""
    got = kx.preferred_allocation_pcie(numa, node, parent, depth, reqs)
    assert got == PO.preferred_allocation_pcie(numa, node, parent, depth, reqs)
    if pyref:
        assert got == P.preferred(numa, node, parent, depth, reqs)
    return got


def check_numa(kx, numa, parent, depth, reqs, pyref=False):
    """kxpu_preferred_allocation and the PCIe call without nodes (NULL, and every entry NO_NODE) give the NUMA
    oracle's answer."""
    want = TO.preferred_allocation(numa, reqs)
    assert kx.preferred_allocation(numa, reqs) == want
    assert kx.preferred_allocation_pcie(numa, None, parent, depth, reqs) == want
    assert kx.preferred_allocation_pcie(numa, np.full(len(numa), NO, np.uint32), parent, depth, reqs) == want
    if pyref:
        assert want == PT.preferred(numa, reqs)
    return want


# ---------------------------------------------------------------- the hand cases in both shapes
@pytest.mark.parametrize("name", sorted(E.HAND))
def test_hand_case_both_shapes(kx, name):
    c = E.HAND[name]
    assert max(len(r[0]) for r in c.requests) <= E.WARP_MAX
    warp = check_pcie(kx, c.dev_numa, c.dev_node, c.parent, c.depth, c.requests, pyref=True)
    assert warp == c.answers
    numa, node, padded = E.pad(c.dev_numa, c.dev_node, c.requests, 300, seed=len(name))
    assert min(len(r[0]) for r in padded) > E.WARP_MAX
    assert check_pcie(kx, numa, node, c.parent, c.depth, padded) == warp
    # both shapes in one call: the padded requests, each followed by its one-warp twin over the padded device list
    mixed = [r for pair in zip(padded, c.requests) for r in pair]
    assert kx.preferred_allocation_pcie(numa, node, c.parent, c.depth, mixed) == [a for a in c.answers for _ in (0, 1)]
    if c.numa:
        assert check_numa(kx, c.dev_numa, c.parent, c.depth, c.requests, pyref=True) == c.answers
        assert check_numa(kx, numa, c.parent, c.depth, padded) == c.answers


# ---------------------------------------------------------------- the shape boundary
BOUNDARY = [255, 256, 257, 258, 511, 4096, 4097]


def boundary_requests(n_devs, seed):
    """One request per size in BOUNDARY: available positions from one stretch of the walk (so that X is a node of the
    forest), up to two of them must-include, a random size."""
    rng = np.random.default_rng(seed)
    reqs = []
    for na in BOUNDARY:
        lo = int(rng.integers(0, n_devs - na))
        av = (lo + rng.permutation(min(n_devs - lo, na + na // 3))[:na]).astype(np.uint32)
        mu = av[:int(rng.integers(0, 3))]
        reqs.append((av, mu, int(rng.integers(len(mu), na + 1))))
    return reqs


@pytest.mark.parametrize("order", ["alone", "large_first", "large_middle", "large_last"])
def test_shape_boundary(kx, order):
    n = 2 * E.TILE + 1
    node, parent, depth = E.range_forest(n)
    numa = E.range_numa(n)
    reqs = boundary_requests(n, seed=7)
    small = [r for r in reqs if len(r[0]) <= E.WARP_MAX]
    large = [r for r in reqs if len(r[0]) > E.WARP_MAX]
    if order == "alone":
        for r in reqs:
            check_pcie(kx, numa, node, parent, depth, [r], pyref=len(r[0]) <= 511)
            check_numa(kx, numa, parent, depth, [r], pyref=len(r[0]) <= 511)
        return
    if order == "large_first":
        reqs = large + small
    elif order == "large_middle":
        reqs = small[:1] + large[:2] + small[1:] + large[2:] + small[:1]
    else:
        reqs = small + large
    check_pcie(kx, numa, node, parent, depth, reqs)
    check_numa(kx, numa, parent, depth, reqs)
    a = pref_requests(reqs)
    out = np.zeros(int(a["size"].sum()), np.uint32)
    out_off = np.full(len(reqs) + 1, 0xABCD, np.uint32)
    kx.preferred_allocation_pcie_raw(numa, node, parent, depth, a, out, out_off)
    assert out_off.tolist() == [0] + np.cumsum(a["size"]).tolist()


# ---------------------------------------------------------------- tile seams of k_big_scatter
@pytest.mark.parametrize("n_devs", [4095, 4096, 4097, 8191, 8192, 8193, 3 * 4096 + 1])
def test_tile_seams(kx, n_devs):
    """r = 0, r on the last candidate in front of a seam and on the first behind it, and r = every candidate, in one
    call (one look-back per request); the deep lca levels of the first must-include device lie in the last tile only,
    the shallow ones span tiles.  The same requests through kxpu_preferred_allocation and the PCIe call without
    nodes."""
    node, parent, depth = E.range_forest(n_devs)
    numa = E.range_numa(n_devs)
    mu = E.seam_must(n_devs, node)
    av = np.random.default_rng(n_devs).permutation(n_devs).astype(np.uint32)
    for nodes in (node, None):
        full = PO.preferred_allocation_pcie(numa, nodes, parent, depth, [(av, mu, n_devs)])[0]
        sizes = [len(mu), n_devs] + (E.seam_sizes(full, len(mu)) if n_devs > E.TILE else [])
        reqs = [(av, mu, s) for s in sizes]
        if nodes is None:
            got = check_numa(kx, numa, parent, depth, reqs)
        else:
            got = check_pcie(kx, numa, nodes, parent, depth, reqs)
        assert got == [full[:s] for s in sizes]
    # with no must-include device: one lca level, the bins alone cut the tiles
    reqs = [(av, [], s) for s in (0, 1, E.TILE - 1, E.TILE, E.TILE + 1, n_devs) if s <= n_devs]
    check_pcie(kx, numa, node, parent, depth, reqs)
    check_numa(kx, numa, parent, depth, reqs)


# ---------------------------------------------------------------- k_pick across CTAs
def test_pick_across_ctas(kx, sm_count):
    """A forest of 2 * T nodes, T = 2 * SMs * 256 the threads of k_pick's first stage, so every thread strides once.
    Nodes 5 and 2T - 1 (thread T - 1: the last CTA, its second stride) are depth-1 leaves of two devices under roots of
    three: equal avail, depth and ancestors, in different CTAs, and 2T - 1 holds the lower positions.  Decoys: a root of
    two devices (shallower), a root of three, a large root; null devices make the request large."""
    T = 2 * sm_count * 256
    nn = 2 * T
    parent = np.full(nn, NO, np.uint32)
    parent[5], parent[nn - 1] = 0, 1
    devs = {nn - 1: [3, 4], 5: [10, 11], 0: [12], 1: [13], nn - 2: [5, 6], T - 1: [0, 1, 2], T: list(range(14, 314))}
    n = 314
    node = np.full(n + 40, NO, np.uint32)
    for v, ps in devs.items():
        node[ps] = v
    numa = np.ones(len(node), np.uint64)
    depth = E.depths(parent)
    av = np.random.default_rng(3).permutation(len(node)).astype(np.uint32)
    reqs = [(av, [], 2), (av, [12], 2), (av, [], 3), (av, [13], 3), (av, [], 301), (av, [4], 1)]
    got = check_pcie(kx, numa, node, parent, depth, reqs, pyref=True)
    assert got[0] == [3, 4] and got[1] == [12, 10] and got[2] == [0, 1, 2] and got[3] == [13, 3, 4] and got[5] == [4]
    # the same forest through the one-warp shape
    small = [(np.array(sum(devs.values(), [])[:200], np.uint32), [], 2)]
    assert check_pcie(kx, numa, node, parent, depth, small, pyref=True) == [[3, 4]]


# ---------------------------------------------------------------- several large requests in one call
def back_to_back(n_devs):
    """Large requests over overlapping devices, each with a different X, must-include set and lowest position than the
    one before: a node count, must count or lowest position left over from the request in front changes an answer."""
    r = np.random.default_rng(11)

    def span(lo, hi):
        return r.permutation(np.arange(lo, hi)).astype(np.uint32)
    return [
        (span(0, 2048), [], 64),             # X = the first 64-position node with no device missing
        (span(192, 4096), [], 64),           # X = a later one: the first is not available any more
        (span(0, 6000), [5000, 5001], 100),  # X = the 512-position node holding both
        (span(3000, n_devs), [n_devs - 1], 3000),
        (span(0, 2048), [], 64),
        (span(100, 9000), [4200, 130, 8900], 700),
        (span(0, n_devs), [], n_devs // 2),
        (span(192, 4096), [200], 2),
    ]


def test_large_requests_back_to_back(kx):
    n = 3 * E.TILE + 1
    node, parent, depth = E.range_forest(n)
    numa = E.range_numa(n)
    reqs = back_to_back(n)
    got = check_pcie(kx, numa, node, parent, depth, reqs)
    assert got[4] == got[0] and got[1] != got[0]
    # each request alone, and the list reversed
    for r in reqs:
        check_pcie(kx, numa, node, parent, depth, [r])
    check_pcie(kx, numa, node, parent, depth, reqs[::-1])


# ---------------------------------------------------------------- forests of every producer
def producer_requests(dev_node, seed):
    """One-warp and large requests: the devices of a few nodes (a parent GPU's vGPUs, a PF and its VFs) with some
    must-include, and random positions."""
    rng = np.random.default_rng(seed)
    n = len(dev_node)
    reqs = []
    for na in (8, 16, 200, 256, 257, 1000, 5000):
        v = dev_node[int(rng.integers(0, n))]
        own = np.flatnonzero(dev_node == v) if v != NO else np.zeros(0, np.int64)
        rest = rng.permutation(n)[:na]
        av = np.unique(np.concatenate([own[:na // 2], rest]))[:na]
        av = av[rng.permutation(len(av))].astype(np.uint32)
        mu = av[np.isin(av, own)][:int(rng.integers(0, 3))]
        reqs.append((av, mu, int(rng.integers(len(mu), len(av) + 1))))
    reqs.append((rng.permutation(n).astype(np.uint32), [], n // 3))
    return reqs


@pytest.mark.parametrize("producer", ["mdev32", "mdev1", "sriov"])
def test_producer_forests(kx, workloads, producer):
    n = 1 << 14
    if producer.startswith("mdev"):
        recs, paths, off, mem, _, _ = workloads.pcie_mdev_walk(n, seed=5, per_gpu=int(producer[4:]))
        t = kx.pcie_tree_mdev(recs, paths, off, mem)
    else:
        recs, paths, off, mem = workloads.pcie_walk(n, seed=5, group_max=1)
        i = np.arange(n)
        pf_of = np.where(i & 7, i & ~7, NO_PF).astype(np.uint32)  # functions 1..7 of a device below function 0
        t = kx.pcie_tree(recs, paths, off, mem, pf_of)
        assert len(t["key"]) > len(kx.pcie_tree(recs, paths, off, mem)["key"])
    node = t["group_node"].copy()
    numa = workloads.topo_dev_numa(len(node), nodes=4)
    reqs = producer_requests(node, seed=len(producer))
    assert {len(r[0]) > E.WARP_MAX for r in reqs} == {False, True}
    check_pcie(kx, numa, node, t["parent"], t["depth"], reqs)
    check_pcie(kx, numa, node, t["parent"], t["depth"], [r for r in reqs if len(r[0]) <= E.WARP_MAX], pyref=True)


# ---------------------------------------------------------------- invalid requests of the large PCIe shape
INVALID = {
    "position_past_n_devs": lambda av, n: (np.append(av, n), [], 4),
    "duplicate_available": lambda av, n: (np.append(av, av[17]), [], 4),
    "duplicate_must": lambda av, n: (av, [av[3], av[9], av[3]], 4),
    "must_not_available": lambda av, n: (av[1:], [av[0]], 4),
}


@pytest.mark.parametrize("kind", sorted(INVALID))
def test_invalid_large_pcie_request(kx, kind):
    n = 2 * E.TILE + 1
    node, parent, depth = E.range_forest(n)
    numa = E.range_numa(n)
    av = np.random.default_rng(1).permutation(n)[:3000].astype(np.uint32)
    good = [(av[:100], av[:1], 10), (av, av[5:7], 500)]
    bad = INVALID[kind](av, n)
    assert len(bad[0]) > E.WARP_MAX
    reqs = good + [bad] + good
    assert PO.preferred_allocation_pcie(numa, node, parent, depth, reqs) is None
    a = pref_requests(reqs)
    out = np.full(int(a["size"].sum()), 0xABCD, np.uint32)
    with pytest.raises(KxpuError) as e:
        kx.preferred_allocation_pcie_raw(numa, node, parent, depth, a, out, np.zeros(len(reqs) + 1, np.uint32))
    assert e.value.status == E_INVALID
    assert (out == 0xABCD).all()
    check_pcie(kx, numa, node, parent, depth, good)
