"""CPU tests of the PCIe topology semantics (include/kxpu.h, ABI v7): the C oracle (oracle/kxpu_pcie_oracle.c) against
the independent Python restatement (tests/pyref_pcie.py) -- the path grammar, the forest of a walk and the
allocation rule with every invalid case -- the worked example, and the identity with the NUMA-only rule."""
import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pcie_example as EX
import pyref_pcie as P
from oracle import pcie_oracle as PO
from oracle import topo_oracle as TO
from oracle import xpu_oracle as XO
from kxpu_b200.binding import PCIPATH_DTYPE

NO = P.NO_NODE


def _one(bdf, path, length=None):
    rec = np.zeros(1, XO.DEVREC_DTYPE)
    rec[0]["bdf"] = bdf
    p = np.zeros(1, PCIPATH_DTYPE)
    p[0]["path"] = path[:120]
    p[0]["len"] = len(path) if length is None else length
    return rec, p


GOOD = b"pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0"


@pytest.mark.parametrize("path,bdf,chain_len", [
    (GOOD, b"0000:03:00.0", 4),
    (b"pci0000:00/0000:03:00.0", b"0000:03:00.0", 1),
    (b"0000:03:00.0", b"0000:03:00.0", 0),                                   # no host bridge
    (b"pci0000:00/0000:00:01.0/0000:03:00.0", b"0000:03:00.1", 0),           # last component is not the bdf
    (b"pci0000:00/0000:00:01.0/0000:03:00.0/", b"0000:03:00.0", 0),          # trailing '/'
    (b"pci0000:00//0000:03:00.0", b"0000:03:00.0", 0),                       # empty component
    (b"/pci0000:00/0000:03:00.0", b"0000:03:00.0", 0),
    (b"pci0000:00/0000:00:1F.0/0000:03:00.0", b"0000:03:00.0", 0),           # upper case
    (b"PCI0000:00/0000:03:00.0", b"0000:03:00.0", 0),
    (b"pci000:00/0000:03:00.0", b"0000:03:00.0", 0),                         # short domain
    (b"pci00000:00/0000:03:00.0", b"0000:03:00.0", 0),                       # 5 digits, leading 0
    (b"pci10000:e0/0000:03:00.0", b"0000:03:00.0", 1),                       # VMD domain
    (b"pci123456789:00/0000:03:00.0", b"0000:03:00.0", 0),                   # 9 digits
    (b"pci0000:00/0000:00:20.0/0000:03:00.0", b"0000:03:00.0", 0),           # dev > 1f
    (b"pci0000:00/0000:00:1f.8/0000:03:00.0", b"0000:03:00.0", 0),           # fn > 7
    (b"pci0000:00/0000:00:1f.7/0000:03:00.0", b"0000:03:00.0", 2),
    (b"pci0000:00/0000:00:0e.0/0000:00:0e.5/pci10000:e0/10000:e0:1d.0/10000:e1:00.0", b"10000:e1:00.0", 5),
    (b"pci0000:00/0000:0:01.0/0000:03:00.0", b"0000:03:00.0", 0),            # 1-digit bus
    (b"pci0000:00:0/0000:03:00.0", b"0000:03:00.0", 0),
])
def test_parse_cases(path, bdf, chain_len):
    rec, p = _one(bdf, path)
    got = PO.parse(rec, p)
    assert len(got) == chain_len
    assert got == P.record_chain(rec[0], p[0])


def test_parse_depth_8_and_9():
    mids = ["0000:%02x:00.0" % k for k in range(1, 10)]
    for levels, want in ((8, 8), (9, 0)):
        path = "/".join(["pci0000:00"] + mids[:levels - 1] + ["0000:f0:00.0"]).encode()
        rec, p = _one(b"0000:f0:00.0", path)
        assert len(PO.parse(rec, p)) == want == len(P.record_chain(rec[0], p[0]))
    rec, p = _one(b"0000:03:00.0", GOOD, length=0)
    assert PO.parse(rec, p) == []
    rec, p = _one(b"0000:03:00.0", GOOD, length=121)
    assert PO.parse(rec, p) == []
    rec, p = _one(b"0000:03:00.0", GOOD)
    assert PO.parse(rec, p) == [1 << 63, 0x0000_00_08, 0x01_00 | 0, 0x02_00]


_ALPHA = "0123456789abcdefABx:./pci"


@st.composite
def path_texts(draw):
    bdf = draw(st.sampled_from(["0000:03:00.0", "0000:03:00.1", "10000:e1:1f.7"]))
    comps = [draw(st.sampled_from(["pci0000:00", "pci10000:e0", "pci0000:0", "PCI0000:00", "pci0000:80"]))]
    for _ in range(draw(st.integers(0, 9))):
        comps.append(draw(st.one_of(
            st.sampled_from(["0000:00:01.0", "0000:01:00.0", "0000:00:1f.7", "0000:00:20.0", "0000:00:01.8",
                             "10000:e0:1d.0", "pci10000:e0", "0000:00:1F.0", "", "000:00:01.0"]),
            st.text(alphabet=_ALPHA, max_size=14))))
    comps.append(draw(st.sampled_from([bdf, bdf, "0000:03:00.2"])))
    text = "/".join(comps) + draw(st.sampled_from(["", "", "/"]))
    return bdf.encode(), text.encode("ascii")


@settings(max_examples=400, deadline=None)
@given(path_texts())
def test_parse_oracle_equals_pyref(case):
    bdf, text = case
    rec, p = _one(bdf, text, length=len(text) if len(text) <= 120 else 0)
    assert PO.parse(rec, p) == P.record_chain(rec[0], p[0])


# ---------------------------------------------------------------- the forest
@st.composite
def walks(draw):
    n = draw(st.integers(0, 24))
    hb = ["pci0000:00", "pci0000:80", "pci10000:e0"]
    mid = ["0000:00:01.0", "0000:00:02.0", "0000:01:00.0", "0000:02:00.0", "0000:02:01.0"]
    recs = np.zeros(n, XO.DEVREC_DTYPE)
    paths = np.zeros(n, PCIPATH_DTYPE)
    for i in range(n):
        bdf = "0000:%02x:00.0" % (0x10 + i)
        comps = [draw(st.sampled_from(hb))] + draw(st.lists(st.sampled_from(mid), max_size=8)) + [bdf]
        text = "/".join(comps).encode()
        recs[i]["bdf"] = bdf.encode()
        paths[i]["path"] = text[:120]
        paths[i]["len"] = draw(st.sampled_from([len(text), len(text), 0])) if len(text) <= 120 else 0
    # groups: a permutation of some records cut into runs
    order = draw(st.permutations(list(range(n))))
    keep = order[:draw(st.integers(0, n))]
    cuts = sorted(draw(st.lists(st.integers(0, len(keep)), max_size=6)))
    off = [0] + cuts + [len(keep)]
    return recs, paths, np.array(off, np.uint32), np.array(keep, np.uint32)


@settings(max_examples=300, deadline=None)
@given(walks())
def test_tree_oracle_equals_pyref(w):
    recs, paths, off, mem = w
    got = PO.tree(recs, paths, off, mem)
    want = P.tree(recs, paths, off, mem)
    for k in ("group_node", "key", "parent", "depth"):
        assert [int(x) for x in got[k]] == want[k], k
    for v, p in enumerate(want["parent"]):
        assert p == NO or p < v


def test_tree_invalid_csr():
    recs, paths, off, mem = EX.records()
    assert PO.tree(recs, paths, np.array([0, 2, 1, 8], np.uint32), mem) is None
    assert PO.tree(recs, paths, off, np.array([0, 1, 2, 3, 4, 5, 6, 8], np.uint32)) is None
    assert P.tree(recs, paths, np.array([0, 2, 1, 8], np.uint32), mem) is None


def test_example_tree():
    recs, paths, off, mem = EX.records()
    t = PO.tree(recs, paths, off, mem)
    assert len(t["key"]) == 18
    assert list(t["depth"][:9]) == [0, 1, 2, 3, 3, 1, 2, 3, 3]
    assert list(t["parent"][:5]) == [NO, 0, 1, 2, 2]
    assert t["key"][0] == 1 << 63 and t["key"][9] == (1 << 63) | (0x80 << 8)
    assert [int(x) for x in t["group_node"]] == [3, 4, 7, 8, 12, 13, 16, 17]


# ---------------------------------------------------------------- allocation
def test_example_answers():
    recs, paths, off, mem = EX.records()
    t = PO.tree(recs, paths, off, mem)
    reqs = EX.requests()
    want = EX.answers()
    assert PO.preferred_allocation_pcie(EX.DEV_NUMA, t["group_node"], t["parent"], t["depth"], reqs) == want
    assert P.preferred(EX.DEV_NUMA, t["group_node"], t["parent"], t["depth"], reqs) == want


@st.composite
def alloc_cases(draw):
    recs, paths, off, mem = draw(walks())
    t = P.tree(recs, paths, off, mem)
    G = len(off) - 1
    n = draw(st.integers(max(G, 1), G + 6))
    dev_node = [t["group_node"][draw(st.integers(0, G - 1))] if G and draw(st.booleans()) else NO for _ in range(n)]
    dev_numa = [draw(st.sampled_from([0, 1, 2, 3, 1 << 63])) for _ in range(n)]
    reqs = []
    for _ in range(draw(st.integers(1, 4))):
        av = draw(st.permutations(list(range(n))))[:draw(st.integers(0, n))]
        mu = draw(st.permutations(av))[:draw(st.integers(0, min(len(av), 3)))]
        reqs.append((av, mu, draw(st.integers(len(mu), len(av)))))
    return (np.array(dev_numa, np.uint64), np.array(dev_node, np.uint32), np.array(t["parent"], np.uint32),
            np.array(t["depth"], np.uint8), reqs)


@settings(max_examples=300, deadline=None)
@given(alloc_cases())
def test_alloc_oracle_equals_pyref(case):
    dev_numa, dev_node, parent, depth, reqs = case
    got = PO.preferred_allocation_pcie(dev_numa, dev_node, parent, depth, reqs)
    assert got == P.preferred(dev_numa, dev_node, parent, depth, reqs)


@settings(max_examples=150, deadline=None)
@given(alloc_cases())
def test_alloc_without_nodes_is_numa_rule(case):
    dev_numa, dev_node, parent, depth, reqs = case
    want = TO.preferred_allocation(dev_numa, reqs)
    assert PO.preferred_allocation_pcie(dev_numa, None, parent, depth, reqs) == want
    none = np.full(len(dev_numa), NO, np.uint32)
    assert PO.preferred_allocation_pcie(dev_numa, none, parent, depth, reqs) == want
    assert P.preferred(dev_numa, none, parent, depth, reqs) == want


INVALID_FORESTS = [
    ("node past n_nodes", [0, 18], None, None),
    ("parent not below", [0, 1], [NO, 2, 1], [0, 1, 2]),
    ("parent of itself", [0, 1], [NO, 1], [0, 1]),
    ("depth not parent + 1", [0, 1], [NO, 0, 0], [0, 2, 1]),
    ("root with depth", [0, 1], [NO, NO], [0, 1]),
    ("depth 8", [0, 1], [NO] + list(range(8)), list(range(9))),
]


@pytest.mark.parametrize("name,dev_node,parent,depth", INVALID_FORESTS, ids=[c[0] for c in INVALID_FORESTS])
def test_alloc_invalid_forest(name, dev_node, parent, depth):
    recs, paths, off, mem = EX.records()
    t = PO.tree(recs, paths, off, mem)
    parent = t["parent"] if parent is None else np.array(parent, np.uint32)
    depth = t["depth"] if depth is None else np.array(depth, np.uint8)
    reqs = [([0, 1], [], 1)]
    assert PO.preferred_allocation_pcie(np.ones(2, np.uint64), dev_node, parent, depth, reqs) is None
    assert P.preferred(np.ones(2, np.uint64), dev_node, parent, depth, reqs) is None


@pytest.mark.parametrize("req", [([0, 9], [], 1), ([0, 1, 1], [], 1), ([0, 1], [0, 0], 2), ([0, 1], [2], 1),
                                 ([0, 1, 2], [0, 1], 1), ([0, 1], [], 3)])
def test_alloc_invalid_requests(req):
    recs, paths, off, mem = EX.records()
    t = PO.tree(recs, paths, off, mem)
    reqs = [([0], [], 1), req]
    assert PO.preferred_allocation_pcie(EX.DEV_NUMA, t["group_node"], t["parent"], t["depth"], reqs) is None
    assert P.preferred(EX.DEV_NUMA, t["group_node"], t["parent"], t["depth"], reqs) is None


def test_workload_forest_mixes_cases(workloads):
    recs, paths, off, mem = workloads.pcie_walk(1 << 14, seed=3)
    t = PO.tree(recs, paths, off, mem)
    assert t is not None
    chains = [PO.parse(recs[i:i + 1], paths[i:i + 1]) for i in range(0, len(recs), 7)]
    lens = {len(c) for c in chains}
    assert 0 in lens and 4 in lens and 7 in lens  # unknown, plain, VMD
    assert (t["group_node"] == NO).any() and len(np.unique(t["depth"])) >= 5
