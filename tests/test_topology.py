"""CPU tests of the NUMA topology semantics (include/kxpu.h, ABI v5): the C oracle (oracle/kxpu_topo_oracle.c)
against the independent Python restatement (tests/pyref_topo.py), the wire bytes against the protobuf runtime, and
the allocation rule's invalid inputs."""
import numpy as np
import pytest
from hypothesis import given, settings
from hypothesis import strategies as st

import pyref_topo as P
from oracle import topo_oracle as TO
from oracle import xpu_oracle as XO

NV = [(b"10de", b"vfio-pci")]


def _rec(bdf, group, numa=None, vendor=b"0x10de\n", driver=b"vfio-pci", device=b"0x2330\n"):
    r = np.zeros(1, XO.DEVREC_DTYPE)[0]
    r["bdf"] = bdf
    r["vendor_txt"][:len(vendor)] = np.frombuffer(vendor, np.uint8)
    r["vendor_len"] = len(vendor)
    r["device_txt"][:len(device)] = np.frombuffer(device, np.uint8)
    r["device_len"] = len(device)
    r["driver"] = driver
    r["iommu_group"] = group
    if numa is not None:
        r["flags"] = 64
        r["reserved0"] = numa
    return r


# ---------------------------------------------------------------- group masks
@st.composite
def topo_recs(draw):
    n = draw(st.integers(0, 40))
    recs = np.zeros(n, XO.DEVREC_DTYPE)
    for i in range(n):
        numa = draw(st.one_of(st.none(), st.sampled_from([0, 1, 2, 63]), st.integers(0, 255)))
        drv = draw(st.sampled_from([b"vfio-pci", b"vfio-pci", b"nvidia"]))
        recs[i] = _rec(b"0000:%02x:00.0" % i, draw(st.integers(0, 6)), numa, driver=drv)
        if numa is not None and draw(st.booleans()) and numa >= 64:
            recs[i]["flags"] = 64  # flag with an out-of-range byte: unknown
    return recs


@settings(max_examples=200, deadline=None)
@given(topo_recs())
def test_group_masks_oracle_equals_pyref(recs):
    res = TO.classify_topo(NV, recs)
    want = XO.classify_rules(NV, recs)
    for k in ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups"):
        assert np.array_equal(res[k], want[k]), k
    assert np.array_equal(res["group_numa"], P.group_masks(recs, res))


def test_group_masks_edges():
    recs = np.array([_rec(b"0000:00:00.0", 7, 0), _rec(b"0000:00:00.1", 7, 63), _rec(b"0000:00:01.0", 8, None),
                     _rec(b"0000:00:02.0", 9, 5), _rec(b"0000:00:02.1", 9, 5, driver=b"nvidia")], XO.DEVREC_DTYPE)
    res = TO.classify_topo(NV, recs)
    assert list(res["group_ids"]) == [7, 8, 9]
    assert list(res["group_numa"]) == [1 | (1 << 63), 0, 1 << 5]  # the rejected function adds nothing


def test_mdev_group_masks_on_workload(workloads):
    recs = workloads.topo_mdev_records(n=1 << 14, nodes=4)
    res = TO.classify_topo(workloads.MDEV_RULES, recs, mdev=True)
    assert res["n_groups"] > 1000
    assert np.array_equal(res["group_numa"], P.group_masks(recs, res))
    pop = np.array([bin(int(m)).count("1") for m in res["group_numa"]])
    assert (pop == 0).any() and (pop > 1).any()


def test_pci_group_masks_on_workload(workloads, oracle_rows):
    recs = workloads.topo_records(oracle_rows["key"], n=1 << 15, nodes=4)
    res = TO.classify_topo(NV, recs)
    gm = res["group_numa"]
    assert np.array_equal(gm, P.group_masks(recs, res))
    pop = np.array([bin(int(m)).count("1") for m in gm])
    assert (pop == 0).any() and (pop > 1).any() and len(set(int(m) for m in gm if m)) >= 4


# ---------------------------------------------------------------- wire bytes
@settings(max_examples=200, deadline=None)
@given(st.lists(st.tuples(st.integers(0, 2**32 - 2), st.booleans(),
                          st.one_of(st.just(0), st.just(1), st.just(1 << 63), st.just(2**64 - 1),
                                    st.integers(0, 2**64 - 1))), max_size=20))
def test_wire_bytes_equal_protobuf_runtime(items):
    g = [i[0] for i in items]
    h = [i[1] for i in items]
    m = [i[2] for i in items]
    got = TO.lw_encode_topo(g, h, m)
    assert got == P.lw_bytes(g, h, m)
    assert P.lw_parse(got) == [(str(a), "Healthy" if b else "Unhealthy", [k for k in range(64) if (c >> k) & 1])
                               for a, b, c in items]


def test_wire_bytes_without_masks_are_lw_encode(oracle):
    g = [0, 7, 214, 4294967294]
    h = [1, 0, 1, 1]
    assert TO.lw_encode_topo(g, h, [0] * 4) == TO.lw_encode_topo(g, h) == oracle.lw_encode(np.array(g, np.uint32),
                                                                                           np.array(h, np.uint8))


def test_wire_bytes_long_device():
    b = TO.lw_encode_topo([4294967294], [0], [2**64 - 1])
    # Device: 0a + 2-byte length; topology: 1a + 2-byte length (254 bytes of nodes)
    assert b[0] == 0x0a and b[1] & 0x80 and len(b) == 283
    assert b.index(b"\x1a\xfe\x01") > 0 and b.endswith(b"\x0a\x02\x08\x3f")
    assert P.lw_parse(b) == [("4294967294", "Unhealthy", list(range(64)))]
    assert TO.lw_encode_topo([5], None, [1]) == b"\x0a\x10\x0a\x01\x35\x12\x07Healthy\x1a\x02\x0a\x00"


# ---------------------------------------------------------------- preferred allocation
@st.composite
def alloc_case(draw):
    n = draw(st.integers(1, 40))
    masks = draw(st.lists(st.one_of(st.just(0), st.sampled_from([1, 2, 4, 1 << 63, 3, 6, (1 << 63) | 1]),
                                    st.integers(0, 2**64 - 1)), min_size=n, max_size=n))
    reqs = []
    for _ in range(draw(st.integers(0, 6))):
        avail = draw(st.lists(st.integers(0, n - 1), unique=True, max_size=n))
        must = draw(st.lists(st.sampled_from(avail), unique=True)) if avail else []
        size = draw(st.integers(len(must), len(avail)))
        reqs.append((avail, must, size))
    return masks, reqs


@settings(max_examples=400, deadline=None)
@given(alloc_case())
def test_allocation_oracle_equals_pyref(case):
    masks, reqs = case
    assert TO.preferred_allocation(masks, reqs) == P.preferred(masks, reqs)


def test_allocation_rules_by_hand():
    # homes: 0 0 1 1 1 64 2
    masks = [1, 1, 2, 2, 6, 0, 4]
    # U first: the must-include device sits on node 0, which has fewer candidates than node 1
    assert P.preferred(masks, [([0, 1, 2, 3, 4, 5, 6], [0], 3)]) == [[0, 1, 2]]
    assert TO.preferred_allocation(masks, [([0, 1, 2, 3, 4, 5, 6], [0], 3)]) == [[0, 1, 2]]
    # no must-include: the largest bin first, ascending position; unknown last
    assert TO.preferred_allocation(masks, [([6, 5, 4, 3, 2, 1, 0], [], 7)]) == [[2, 3, 4, 0, 1, 6, 5]]
    # ties: equal counts -> lower node first; r = 0; size = |available|
    assert TO.preferred_allocation([1, 2, 1, 2], [([3, 2, 1, 0], [], 2), ([0, 1], [1], 1), ([1, 0], [], 2)]) == \
        [[0, 2], [1], [0, 1]]
    # all unknown: position order
    assert TO.preferred_allocation([0] * 5, [([4, 1, 3], [3], 2)]) == [[3, 1]]


@pytest.mark.parametrize("req", [
    ([0, 5], [], 1),          # position >= n_devs
    ([0, 1, 1], [], 1),       # duplicate in available
    ([0, 1], [0, 0], 2),      # duplicate in must-include
    ([0, 1], [2], 1),         # must-include not available
    ([0, 1, 2], [0, 1], 1),   # size < |must|
    ([0, 1], [], 3),          # size > |available|
])
def test_allocation_invalid(req):
    assert P.preferred([1, 1, 2, 2], [req]) is None
    assert TO.preferred_allocation([1, 1, 2, 2], [([0], [], 1), req]) is None
