"""GPU tests of the NUMA topology calls (include/kxpu.h, ABI v5) against the CPU oracle (oracle/kxpu_topo_oracle.c)."""
import numpy as np
import pytest

import pyref_topo as P
from oracle import topo_oracle as TO

pytestmark = pytest.mark.gpu
NV = [(b"10de", b"vfio-pci")]
KEYS = ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups", "dev_rule")


@pytest.mark.parametrize("nodes", [2, 4])
def test_classify_topo_pci_2_20(kx, workloads, oracle_rows, nodes):
    recs = workloads.topo_records(oracle_rows["key"], n=1 << 20, nodes=nodes)
    n0 = kx.launch_count()
    got = kx.classify_topo(NV, recs)
    n1 = kx.launch_count()
    plain = kx.classify_rules(NV, recs)
    assert kx.launch_count() - n1 == n1 - n0  # the mask costs no launch
    for k in KEYS:
        assert np.array_equal(got[k], plain[k]), k
    want = TO.classify_topo(NV, recs)
    assert np.array_equal(got["group_numa"], want["group_numa"])
    assert (got["group_numa"] == 0).any() and len(np.unique(got["group_numa"])) > nodes


def test_classify_topo_mdev_2_20(kx, workloads):
    recs = workloads.topo_mdev_records(n=1 << 20, nodes=4)
    got = kx.classify_topo(workloads.MDEV_RULES, recs, mdev=True)
    plain = kx.classify_mdev(workloads.MDEV_RULES, recs)
    for k in KEYS:
        assert np.array_equal(got[k], plain[k]), k
    want = TO.classify_topo(workloads.MDEV_RULES, recs, mdev=True)
    assert np.array_equal(got["group_numa"], want["group_numa"])


def test_numa_bytes_change_nothing_else(kx, workloads, oracle_rows):
    """Random numa_node bytes with KXPU_REC_NUMA set give bitwise the results of zeroed ones through every pre-v5 call."""
    rng = np.random.default_rng(3)
    recs = workloads.cfg3_records(oracle_rows["key"], n=1 << 18)
    noisy = recs.copy()
    noisy["reserved0"] = rng.integers(0, 256, len(recs), dtype=np.uint8)
    noisy["flags"] |= 64
    for fn in (kx.classify, lambda r: kx.classify_rules(workloads.XPU_RULES, r)):
        a, b = fn(recs), fn(noisy)
        for k in a:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    m = workloads.mdev_records(n=1 << 18)
    mn = m.copy()
    mn["reserved0"] = rng.integers(0, 256, len(m), dtype=np.uint8)
    mn["flags"] |= 64
    a, b = kx.classify_mdev(workloads.MDEV_RULES, m), kx.classify_mdev(workloads.MDEV_RULES, mn)
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    idx = np.arange(0, len(m), 97, dtype=np.uint32)
    assert kx.mdev_names(m, idx)[0] == kx.mdev_names(mn, idx)[0]
    assert np.array_equal(kx.mdev_names(m, idx)[1], kx.mdev_names(mn, idx)[1])


def test_lw_encode_topo_1m(kx):
    n = 1 << 20
    rng = np.random.default_rng(5)
    groups = rng.integers(0, 2**32 - 1, n, dtype=np.uint64).astype(np.uint32)
    healthy = (rng.random(n) < 0.9).astype(np.uint8)
    masks = np.where(rng.random(n) < 0.2, 0, np.uint64(1) << rng.integers(0, 4, n).astype(np.uint64)).astype(np.uint64)
    masks[::1000] = rng.integers(0, 2**63, n // 1000 + 1, dtype=np.uint64)[:len(masks[::1000])] | np.uint64(1)  # many nodes
    masks[7] = np.uint64(2**64 - 1)  # 64 nodes: Device of 283 bytes
    got = kx.lw_encode_topo(groups, healthy, masks)
    assert got == TO.lw_encode_topo(groups, healthy, masks)
    cut = len(TO.lw_encode_topo(groups[:100], healthy[:100], masks[:100]))  # the first 100 Devices parse back
    head = P.lw_parse(got[:cut])
    assert [d[0] for d in head] == [str(g) for g in groups[:100]] and head[7][2] == list(range(64))


def test_lw_encode_topo_zero_masks_equal_lw_encode(kx):
    n = 1 << 20
    rng = np.random.default_rng(6)
    groups = rng.integers(0, 2**32 - 1, n, dtype=np.uint64).astype(np.uint32)
    healthy = (rng.random(n) < 0.5).astype(np.uint8)
    ref = kx.lw_encode(groups, healthy)
    assert kx.lw_encode_topo(groups, healthy, np.zeros(n, np.uint64)) == ref
    assert kx.lw_encode_topo(groups, healthy, None) == ref
    assert kx.lw_encode_topo(groups[:5], None, [1, 0, 2**63, 6, 0]) == P.lw_bytes(groups[:5], None, [1, 0, 2**63, 6, 0])


def test_preferred_allocation_batch(kx, workloads):
    dev_numa = workloads.topo_dev_numa(4096, nodes=4)
    reqs = workloads.topo_requests(dev_numa, n_req=4096, avail=16, size=8, must_max=2)
    got = kx.preferred_allocation(dev_numa, reqs)
    assert got == TO.preferred_allocation(dev_numa, reqs)
    # warp-path edges: r = 0, size = |available|, 256 positions, all unknown
    perm = np.random.default_rng(8).permutation(4096)[:256].tolist()
    edge = [(list(range(10)), [3, 1], 2), (list(range(9, -1, -1)), [], 10), (perm, perm[:2], 100), ([4000, 4001, 4002], [], 2)]
    zeros = np.zeros(4096, np.uint64)
    assert kx.preferred_allocation(dev_numa, edge) == TO.preferred_allocation(dev_numa, edge)
    assert kx.preferred_allocation(zeros, edge) == TO.preferred_allocation(zeros, edge)


def test_preferred_allocation_fuzz(kx):
    rng = np.random.default_rng(12)
    for trial in range(20):
        n = int(rng.integers(1, 600))
        choices = np.array([0, 1, 2, 4, 1 << 63, 3, 6, (1 << 63) | 1], np.uint64)
        dev_numa = choices[rng.integers(0, len(choices), n)]
        reqs = []
        for _ in range(int(rng.integers(1, 40))):
            na = int(rng.integers(0, min(n, 400) + 1))
            av = rng.permutation(n)[:na]
            mu = av[rng.permutation(na)[:int(rng.integers(0, min(na, 4) + 1))]]
            reqs.append((av.tolist(), mu.tolist(), int(rng.integers(len(mu), na + 1))))
        assert kx.preferred_allocation(dev_numa, reqs) == TO.preferred_allocation(dev_numa, reqs), trial


def test_preferred_allocation_one_request_2_20(kx, workloads):
    n = 1 << 20
    dev_numa = workloads.topo_dev_numa(n, nodes=4)
    reqs = workloads.topo_requests(dev_numa, n_req=1, avail=n, size=n // 2, must_max=3, seed=10)
    got = kx.preferred_allocation(dev_numa, reqs)
    assert got == TO.preferred_allocation(dev_numa, reqs)
    part = workloads.topo_requests(dev_numa, n_req=3, avail=300000, size=1000, must_max=5, seed=13)
    assert kx.preferred_allocation(dev_numa, part) == TO.preferred_allocation(dev_numa, part)


@pytest.mark.parametrize("req", [([0, 5000], [], 1), ([0, 1, 1], [], 1), ([0, 1], [0, 0], 2), ([0, 1], [2], 1),
                                 ([0, 1, 2], [0, 1], 1), ([0, 1], [], 3)])
def test_preferred_allocation_invalid(kx, req):
    import kxpu_b200 as K
    dev_numa = np.ones(4096, np.uint64)
    with pytest.raises(K.KxpuError) as e:
        kx.preferred_allocation(dev_numa, [([0], [], 1), req])
    assert e.value.status == K.binding.E_INVALID


@pytest.mark.parametrize("req", [([10, 70000], [], 1), ([10, 11, 11], [], 1), ([10, 11], [10, 10], 2), ([10, 11], [2], 1)])
def test_preferred_allocation_invalid_large_request(kx, req):
    """The faults the GPU finds, inside a request past the one-warp size."""
    import kxpu_b200 as K
    dev_numa = np.ones(1 << 16, np.uint64)
    big = (list(range(1000, 2000)) + req[0], req[1], req[2] + 1000)
    with pytest.raises(K.KxpuError) as e:
        kx.preferred_allocation(dev_numa, [([0], [], 1), big])
    assert e.value.status == K.binding.E_INVALID
    assert kx.preferred_allocation(dev_numa, [([0], [], 1)]) == [[0]]  # the context stays usable
