"""GPU tests of kxpu_pcie_tree_mdev (include/kxpu.h, addition to ABI v14): group_node, key, parent, depth and the node
count bitwise equal to the C checker (tests/pcie_mdev_oracle.c) and the Python restatement on every hand case, under a
seeded fuzz and on a 2^20-record walk, equal to kxpu_pcie_tree on that walk's PCI twin, and the invalid cases."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings

import pcie_mdev_cases as MC
import pcie_mdev_oracle as MO
import pyref_pcie_mdev as P
from kxpu_b200.binding import E_INVALID, E_UNSUPPORTED, KxpuError

pytestmark = pytest.mark.gpu


def _tree(kx, recs, paths, off, mem):
    t = kx.pcie_tree_mdev(recs, paths, off, mem)
    return {k: v.tolist() for k, v in t.items()}


@pytest.mark.parametrize("name", sorted(MC.HAND))
def test_hand_cases(kx, name):
    recs, paths, off, mem = MC.HAND[name]
    got = _tree(kx, recs, paths, off, mem)
    assert got == MO.tree(recs, paths, off, mem) == P.tree(recs, paths, off, mem)
    if name in MC.CHAIN_LEN and len(off) - 1 == len(recs):  # one group per record: group 0 is record 0's chain
        g = got["group_node"][0]
        assert (0 if g == MC.NO_NODE else got["depth"][g] + 1) == MC.CHAIN_LEN[name]


@settings(max_examples=200, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(MC.mdev_walks())
def test_fuzz(kx, w):
    assert _tree(kx, *w) == MO.tree(*w) == P.tree(*w)


def test_big_walk(kx, workloads):
    recs, paths, off, mem, twin, twin_paths = workloads.pcie_mdev_walk(1 << 20)
    got = kx.pcie_tree_mdev(recs, paths, off, mem)
    want = MO.tree(recs, paths, off, mem)
    for k in ("group_node", "key", "parent", "depth"):
        assert got[k].tolist() == want[k], k
    assert len(got["key"]) == len(want["key"]) > (1 << 15)  # every GPU of the walk is a node
    plain = kx.pcie_tree(twin, twin_paths, off, mem)
    for k in got:
        assert np.array_equal(got[k], plain[k]), k


def test_invalid(kx):
    recs, paths, off, mem = MC.HAND["two_vgpus_one_gpu"]
    with pytest.raises(KxpuError) as e:
        kx.pcie_tree_mdev(recs, paths, np.array([0, 2, 1], np.uint32), mem)
    assert e.value.status == E_INVALID
    with pytest.raises(KxpuError) as e:
        kx.pcie_tree_mdev(recs, paths, off, np.array([0, 2], np.uint32))
    assert e.value.status == E_INVALID
    gn, key, par, dep = np.zeros(2, np.uint32), np.zeros(16, np.uint64), np.zeros(16, np.uint32), np.zeros(16, np.uint8)
    import ctypes as C
    nn = C.c_uint32(7)
    rc = kx.L.kxpu_pcie_tree_mdev(kx.ctx, recs.ctypes.data, paths.ctypes.data, 1 << 28, off.ctypes.data, mem.ctypes.data,
                                  2, gn.ctypes.data, key.ctypes.data, par.ctypes.data, dep.ctypes.data, C.byref(nn))
    assert rc == E_UNSUPPORTED
    empty = kx.pcie_tree_mdev(recs[:0], paths[:0], np.zeros(1, np.uint32), mem[:0])
    assert all(len(v) == 0 for v in empty.values())
