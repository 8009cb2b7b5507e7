"""CPU tests of GetPreferredAllocation at its edges (tests/pref_edge_cases.py): every hand case gives its hand-written
answer in both C oracles (oracle/kxpu_pcie_oracle.c, oracle/kxpu_topo_oracle.c) and both Python restatements
(tests/pyref_pcie.py, tests/pyref_topo.py); padding a request with null devices keeps its answer on the oracles, for
both calls, so that the GPU tests can send every small case through the large shape; and the large-shape generators
put r on the tile seams they claim."""
import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pref_edge_cases as E
import pyref_pcie as P
import pyref_topo as PT
from oracle import pcie_oracle as PO
from oracle import topo_oracle as TO

NO = E.NO


@pytest.mark.parametrize("name", sorted(E.HAND))
def test_hand_case(name):
    c = E.HAND[name]
    assert PO.preferred_allocation_pcie(c.dev_numa, c.dev_node, c.parent, c.depth, c.requests) == c.answers
    assert P.preferred(c.dev_numa, c.dev_node, c.parent, c.depth, c.requests) == c.answers
    if c.numa:
        assert TO.preferred_allocation(c.dev_numa, c.requests) == c.answers
        assert PT.preferred(c.dev_numa, c.requests) == c.answers
        assert PO.preferred_allocation_pcie(c.dev_numa, None, c.parent, c.depth, c.requests) == c.answers


@pytest.mark.parametrize("name", sorted(E.HAND))
def test_hand_case_padded(name):
    c = E.HAND[name]
    numa, node, reqs = E.pad(c.dev_numa, c.dev_node, c.requests, 300, seed=len(name))
    assert all(len(r[0]) > E.WARP_MAX for r in reqs)
    assert PO.preferred_allocation_pcie(numa, node, c.parent, c.depth, reqs) == c.answers
    assert P.preferred(numa, node, c.parent, c.depth, reqs) == c.answers
    if c.numa:
        assert TO.preferred_allocation(numa, reqs) == c.answers


def test_hand_cases_isolate_their_term():
    """The cases that pin one term of the node key are built so that the term goes against the lowest position and
    against the node ids: the winning leaf holds the higher positions and the higher node id."""
    for name in ("depth_decides", "parent_decides", "grandparent_decides", "depth7_root_decides"):
        c = E.HAND[name]
        assert c.answers == [c.leaves[1]] and c.leaves[0] < c.leaves[1]
        assert int(c.dev_node[c.leaves[0][0]]) < int(c.dev_node[c.leaves[1][0]])
    assert int(E.HAND["depth7_root_decides"].depth.max()) == E.MAX_DEPTH - 1


@st.composite
def padded_cases(draw):
    """A random forest of up to 24 nodes (depth < 8), devices in it or in no node, masks with homes 0, 1, 63 and 64,
    up to four requests of up to 40 positions, and 1 .. 300 null devices."""
    nn = draw(st.integers(0, 24))
    parent, depth = [], []
    for v in range(nn):
        p = draw(st.integers(-1, v - 1))
        if p >= 0 and depth[p] >= E.MAX_DEPTH - 1:
            p = -1
        parent.append(NO if p < 0 else p)
        depth.append(0 if p < 0 else depth[p] + 1)
    n = draw(st.integers(1, 40))
    dev_node = [draw(st.integers(0, nn - 1)) if nn and draw(st.integers(0, 4)) else NO for _ in range(n)]
    dev_numa = [draw(st.sampled_from([0, 1, 2, 3, 1 << 63, (1 << 64) - 1])) for _ in range(n)]
    reqs = []
    for _ in range(draw(st.integers(1, 4))):
        av = draw(st.permutations(list(range(n))))[:draw(st.integers(0, n))]
        mu = draw(st.permutations(av))[:draw(st.integers(0, min(len(av), 3)))]
        reqs.append((av, mu, draw(st.integers(len(mu), len(av)))))
    return (np.array(dev_numa, np.uint64), np.array(dev_node, np.uint32), np.array(parent, np.uint32),
            np.array(depth, np.uint8), reqs, draw(st.integers(1, 300)), draw(st.integers(0, 1 << 16)))


@settings(max_examples=300, deadline=None)
@given(padded_cases())
def test_padding_keeps_the_answer(case):
    dev_numa, dev_node, parent, depth, reqs, n_pad, seed = case
    want = PO.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, reqs)
    assert want is not None
    numa, node, padded = E.pad(dev_numa, dev_node, reqs, n_pad, seed)
    assert PO.preferred_allocation_pcie(numa, node, parent, depth, padded) == want
    want_numa = TO.preferred_allocation(dev_numa, reqs)
    assert TO.preferred_allocation(numa, padded) == want_numa
    assert PO.preferred_allocation_pcie(numa, None, parent, depth, padded) == want_numa


@pytest.mark.parametrize("n_devs", [4095, 4096, 4097, 8191, 8192, 8193, 3 * 4096 + 1])
def test_seam_generators(n_devs):
    """range_forest is a valid forest with deep nodes inside one tile; seam_must leaves X = every device; the sizes of
    seam_sizes end r on the last candidate in front of a seam and on the first behind it, in both calls."""
    dev_node, parent, depth = E.range_forest(n_devs)
    assert P.forest_valid(dev_node, parent, depth) and int(depth.max()) == 3
    numa = E.range_numa(n_devs)
    mu = E.seam_must(n_devs, dev_node)
    av = np.random.default_rng(n_devs).permutation(n_devs).astype(np.uint32)
    for node in (dev_node, None):
        full = PO.preferred_allocation_pcie(numa, node, parent, depth, [(av, mu, n_devs)])[0]
        assert sorted(full) == list(range(n_devs))
        sizes = E.seam_sizes(full, len(mu)) if n_devs > E.TILE else []
        reqs = [(av, mu, s) for s in sizes + [len(mu)]]
        got = PO.preferred_allocation_pcie(numa, node, parent, depth, reqs)
        for (_, _, s), g in zip(reqs, got):
            assert g == full[:s]
        for k in range(0, len(sizes), 2):
            last, first = full[sizes[k] - 1], full[sizes[k + 1] - 1]
            assert last // E.TILE < first // E.TILE
    # the deep levels of the must-include device near the end: their candidates all lie in the last tile
    deep = int(dev_node[mu[0]])
    members = np.flatnonzero(dev_node == deep)
    if (n_devs - 1) % E.TILE:
        assert (members // E.TILE == (n_devs - 1) // E.TILE).all()
