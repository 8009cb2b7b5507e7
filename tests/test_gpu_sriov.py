"""GPU tests of the SR-IOV calls: kxpu_sriov bitwise equal to the C checker and the Python restatement on the hand cases,
under a seeded fuzz and on a 2^20-record walk; kxpu_pcie_tree_sriov equal to both, at the depth limit too, and bitwise
kxpu_pcie_tree's without PFs; the invalid and domain cases."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings

import pyref_sriov as P
import sriov_cases as SC
import sriov_oracle as SO
from kxpu_b200.binding import E_INVALID, E_UNSUPPORTED, KxpuError, rules_array

pytestmark = pytest.mark.gpu


def _check(kx, recs, srs, rules=SC.NV):
    c = kx.classify_rules(rules, recs)
    got = kx.sriov(rules, recs, srs, c["group_ids"], c["group_off"], c["group_members"])
    want = SO.sriov(rules, recs, srs, c["group_off"], c["group_members"])
    for k in ("pf_of", "numvfs", "group_sriov"):
        assert got[k].tolist() == want[k], k
    if len(recs) <= 4096:  # the Python restatement is too slow for the 2^20 walk
        assert want == P.sriov(rules, recs, srs, c["group_off"], c["group_members"])
    return c, got


@pytest.mark.parametrize("name", sorted(SC.HAND))
def test_hand_cases(kx, name):
    (recs, srs), pf_of, numvfs, groups = SC.HAND[name]
    c, got = _check(kx, recs, srs)
    assert got["pf_of"].tolist() == pf_of and got["numvfs"].tolist() == numvfs
    assert dict(zip(c["group_ids"].tolist(), got["group_sriov"].tolist())) == groups


def test_numvfs_shapes(kx):
    recs = np.array([SC.VC.gpu(i, 10 + i) for i in range(len(SC.NUMVFS))])
    srs = np.array([SC.sr(numvfs=t) for t, _ in SC.NUMVFS])
    _, got = _check(kx, recs, srs)
    assert got["numvfs"].tolist() == [v for _, v in SC.NUMVFS]


@settings(max_examples=200, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(SC.sriov_walks())
def test_fuzz(kx, w):
    _check(kx, *w)
    _check(kx, *w, rules=SC.VC.TWO)


def test_big_walk(kx, workloads):
    recs, srs = workloads.sriov_walk(1 << 20)
    c, got = _check(kx, recs, srs)
    assert c["n_groups"] == (1 << 20) - (1 << 16)  # the PFs on a host driver are no candidates
    assert (got["group_sriov"] != SC.VIABLE).sum() > (1 << 20) // 4  # the vfio-pci PFs and their VFs


def _tree(kx, recs, paths, off, mem, pf_of=None):
    t = kx.pcie_tree(recs, paths, off, mem, pf_of)
    return {k: v.tolist() for k, v in t.items()}


@settings(max_examples=200, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(SC.forests())
def test_tree_fuzz(kx, f):
    recs, paths, off, mem, pf_of = f
    got = _tree(kx, recs, paths, off, mem, pf_of)
    assert got == P.tree(recs, paths, off, mem, pf_of) == SO.tree(recs, paths, off, mem, pf_of)
    none = np.full(len(recs), SC.NO_PF, np.uint32)
    assert _tree(kx, recs, paths, off, mem, none) == _tree(kx, recs, paths, off, mem)


@pytest.mark.parametrize("levels", [1, 7, 8])
def test_tree_depth_limit(kx, levels):
    """A PF chain of 7 keys puts the VF at depth 7 below the PF; one of 8 leaves the VF on its own chain."""
    recs, paths, off, mem, pf_of = SC.deep(levels)
    got = _tree(kx, recs, paths, off, mem, pf_of)
    assert got == SO.tree(recs, paths, off, mem, pf_of) == P.tree(recs, paths, off, mem, pf_of)
    vf, pf = got["group_node"][1], got["group_node"][0]
    if levels < 8:
        assert got["depth"][vf] == levels and got["parent"][vf] == pf
    else:
        assert vf == pf and got == _tree(kx, recs, paths, off, mem)


def test_tree_big_without_pfs_is_pcie_tree(kx):
    n = 1 << 18
    recs = np.zeros(n, SC.XO.DEVREC_DTYPE)
    paths = np.zeros(n, SC.PCIPATH_DTYPE)
    for i in range(n):
        bdf = "%04x:%02x:%02x.%d" % (i >> 11, (i >> 3) & 0xff, 0, i & 7)
        text = "pci%04x:00/%04x:00:%02x.0/%s" % (i >> 11, i >> 11, (i >> 3) & 3, bdf)  # four root ports per domain
        recs[i]["bdf"], paths[i]["path"], paths[i]["len"] = bdf.encode(), text.encode(), len(text)
    off, mem = np.arange(n + 1, dtype=np.uint32), np.arange(n, dtype=np.uint32)
    a = kx.pcie_tree(recs, paths, off, mem)
    b = kx.pcie_tree(recs, paths, off, mem, np.full(n, SC.NO_PF, np.uint32))
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    # functions 1..7 of every device name function 0 as PF: each PF becomes one more node
    pf_of = (np.arange(n) & ~7).astype(np.uint32)
    pf_of[::8] = SC.NO_PF
    t = kx.pcie_tree(recs, paths, off, mem, pf_of)
    assert len(t["key"]) == len(a["key"]) + n // 8


def test_invalid_and_domain(kx):
    (recs, srs), *_ = SC.HAND["pf_on_vfio_with_vfs"]
    c = kx.classify_rules(SC.NV, recs)
    gids, off, mem = c["group_ids"], c["group_off"], c["group_members"]
    with pytest.raises(KxpuError) as e:
        kx.sriov(SC.NV, recs, srs, gids, np.array([0, 2, 1, 3], np.uint32), mem)
    assert e.value.status == E_INVALID
    with pytest.raises(KxpuError) as e:
        kx.sriov(SC.NV, recs, srs, gids, off, np.array([0, 1, 3], np.uint32))
    assert e.value.status == E_INVALID
    with pytest.raises(KxpuError) as e:
        kx.sriov([(b"10de", b"vfio/pci")], recs, srs, gids, off, mem)
    assert e.value.status == E_INVALID
    with pytest.raises(KxpuError) as e:
        kx.sriov([], recs, srs, gids, off, mem)
    assert e.value.status == E_INVALID
    empty = kx.sriov(SC.NV, recs[:0], srs[:0], gids[:0], np.zeros(1, np.uint32), mem[:0])
    assert all(len(v) == 0 for v in empty.values())
    # n at the limit: refused before any array is read (the buffers here hold three records)
    pf, nv, gs = np.zeros(3, np.uint32), np.zeros(3, np.uint32), np.zeros(3, np.uint32)
    ra = rules_array(SC.NV)
    rc = kx.L.kxpu_sriov(kx.ctx, ra.ctypes.data, 1, recs.ctypes.data, srs.ctypes.data, 1 << 30, None, off.ctypes.data,
                         mem.ctypes.data, len(off) - 1, pf.ctypes.data, nv.ctypes.data, gs.ctypes.data)
    assert rc == E_UNSUPPORTED
    paths = np.zeros(len(recs), SC.PCIPATH_DTYPE)
    with pytest.raises(KxpuError) as e:
        kx.pcie_tree(recs, paths, off, mem, np.array([SC.NO_PF, 3, 0], np.uint32))
    assert e.value.status == E_INVALID
