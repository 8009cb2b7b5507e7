"""GPU tests of kxpu_pcie_ports_mdev, kxpu_dra_slices_mdev_pcie and kxpu_dra_slices_vf_vgpu_pcie against the Python
restatement (tests/pyref_vgpu_pcie.py): the rule on its hand cases, on walks from n = 0 to 2^20 at the parse and group
tile edges and against kxpu_pcie_ports on the parents' own records; the slices from 0 to 2^20 devices at the slice seams,
with taint tables of 0, 1 and 3 entries, at every reachable position of the two names and with 16-byte VMD addresses;
pools with every key absent against kxpu_dra_slices_mdev_pf, kxpu_dra_slices_mdev_taints and kxpu_dra_slices_vf_vgpu;
every refusal with the outputs untouched."""
import ctypes as C

import numpy as np
import pytest

import pyref_vgpu_pcie as R
import vgpu_pcie_cases as CC
from kxpu_b200.binding import KxpuError

pytestmark = pytest.mark.gpu

TAINTS = [("vgpu.example.com/unhealthy", "vfio-device-missing", "NoSchedule"),
          ("vgpu.example.com/pcie-aer", "fatal", "NoSchedule"), ("vgpu.example.com/pcie-aer", "nonfatal", "NoSchedule")]


def _since(n, nt, seed):
    if nt == 0:
        return None
    rng = np.random.default_rng(seed)
    s = np.where(rng.random((n, nt)) < 0.3, rng.integers(0, 253402300799, (n, nt)), -1).astype(np.int64)
    if nt == 3:
        s[:, 2] = np.where(s[:, 1] >= 0, -1, s[:, 2])  # one key and effect carried once
    return s


def _call(kx, layout, dom, devs, nt, since):
    f = kx.dra_slices_mdev_pcie if layout == "mdev" else kx.dra_slices_vf_vgpu_pcie
    return f("vgpu.example.com", "node-a", "node-a", 5, dom, devs, TAINTS[:nt], since)


def _devs(layout, n, seed, **kw):
    return CC.random_mdev_devs(n, seed, **kw) if layout == "mdev" else CC.random_vf_devs(n, seed, **kw)


def _same(got, want):
    assert got[0] == want[0] and list(got[1]) == list(want[1])


# ------------------------------------------------------------------ kxpu_pcie_ports_mdev

@pytest.mark.parametrize("case", CC.HAND, ids=[c[0] for c in CC.HAND])
def test_ports_hand_cases(kx, case):
    _, rows, groups, want = case
    rp, sw = kx.pcie_ports_mdev(*CC.hand_walk(rows, groups))
    assert (list(rp), list(sw)) == tuple(CC.expected(want))


@pytest.mark.parametrize("per_group", [1, 3])
@pytest.mark.parametrize("n", [0, 1, 15, 16, 17, 255, 256, 257, 5000, 1 << 20])
def test_ports_parity_and_invariant(kx, n, per_group):
    mwalk, pwalk = CC.random_walk(n, seed=n, per_group=per_group)
    rp, sw = kx.pcie_ports_mdev(*mwalk)
    if n <= 5000:
        want = R.pcie_ports_mdev(*mwalk)
        assert list(rp) == want[0] and list(sw) == want[1]
    # the invariant: with every path known, the parents' own records give the same keys
    cw, cp = CC.random_walk(n, seed=n, unknown=0, per_group=per_group)
    a, b = kx.pcie_ports_mdev(*cw)
    c, d = kx.pcie_ports(*cp)
    assert np.array_equal(a, c) and np.array_equal(b, d)


def test_ports_refusals_leave_outputs(kx):
    recs, paths, off, mem = CC.hand_walk(CC.HAND[0][1], None)
    rp, sw = np.full(1, 7, np.uint64), np.full(1, 7, np.uint64)
    with pytest.raises(KxpuError):
        kx.pcie_ports_mdev_raw(recs, paths, off, np.array([5], np.uint32), rp, sw)
    with pytest.raises(KxpuError):
        kx.pcie_ports_mdev_raw(recs, paths, np.array([1, 0], np.uint32), mem, rp, sw)
    assert list(rp) == [7] and list(sw) == [7]


# ------------------------------------------------------------------ the two slice layouts

@pytest.mark.parametrize("layout", ["mdev", "vf_vgpu"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 127, 128, 129, 4099, 1 << 20])
@pytest.mark.parametrize("nt", [0, 1, 3])
def test_slices_parity(kx, layout, n, nt):
    if n == 1 << 20 and nt == 1:
        pytest.skip("2^20 runs untainted and with three taints")
    devs = _devs(layout, n, n + nt)
    since = _since(n, nt, n)
    got = _call(kx, layout, CC.DOMAIN, devs, nt, since)
    if n > 5000:
        # slice_off against the slices' own lengths, then the first and the last slices against the restatement on
        # their devices (its slice count rewritten to the whole pool's)
        per = 128 if nt == 0 else 64
        count = -(-n // per)
        offs = [int(x) for x in got[1]]
        assert len(offs) == count + 1 and offs[0] == 0 and offs[-1] == len(got[0])
        lines = got[0].split(b"\n")[:-1]
        assert [len(x) + 1 for x in lines] == [b - a for a, b in zip(offs, offs[1:])]
        for first in (0, count - 3):
            lo, hi = first * per, min(n, (first + 3) * per)
            want = R.slices(layout, "vgpu.example.com", "node-a", "node-a", 5, CC.DOMAIN, devs[lo:hi], TAINTS[:nt],
                            None if since is None else since[lo:hi])
            w = want[0].replace(b'"resourceSliceCount":%d' % (len(want[1]) - 1), b'"resourceSliceCount":%d' % count)
            assert b"\n".join(lines[first:first + 3]) + b"\n" == w
        return
    _same(got, R.slices(layout, "vgpu.example.com", "node-a", "node-a", 5, CC.DOMAIN, devs, TAINTS[:nt], since))


@pytest.mark.parametrize("layout,positions", [("mdev", CC.MDEV_POSITIONS), ("vf_vgpu", CC.VF_POSITIONS)])
@pytest.mark.parametrize("nt", [0, 1, 3])
def test_every_position(kx, layout, positions, nt):
    devs = _devs(layout, 130, 9, all_attrs=True)
    devs2 = _devs(layout, 130, 10)
    since = _since(130, nt, 3)
    for dom in positions:
        if dom is None:
            continue
        for d in (devs, devs2):
            _same(_call(kx, layout, dom, d, nt, since),
                  R.slices(layout, "vgpu.example.com", "node-a", "node-a", 5, dom, d, TAINTS[:nt], since))


@pytest.mark.parametrize("layout", ["mdev", "vf_vgpu"])
def test_vmd_addresses(kx, layout):
    devs = _devs(layout, 300, 4, long_addr=True, all_attrs=True)
    for nt in (0, 3):
        since = _since(300, nt, 5)
        _same(_call(kx, layout, "x.io", devs, nt, since),
              R.slices(layout, "vgpu.example.com", "node-a", "node-a", 5, "x.io", devs, TAINTS[:nt], since))


@pytest.mark.parametrize("n", [0, 1, 129, 4099])
@pytest.mark.parametrize("nt", [0, 1, 3])
def test_no_keys_equal_the_parent_layouts(kx, n, nt):
    since = _since(n, nt, 7)
    m = CC.random_mdev_devs(n, n, no_keys=True)
    for dom in ("example.com", "x.io", CC.DOMAIN):
        got = _call(kx, "mdev", dom, m, nt, since)
        _same(got, kx.dra_slices_mdev_pf("vgpu.example.com", "node-a", "node-a", 5, m["pf"], TAINTS[:nt], since))
    m2 = CC.random_mdev_devs(n, n, no_keys=True, no_physfn=True)
    _same(_call(kx, "mdev", CC.DOMAIN, m2, nt, since),
          kx.dra_slices_mdev_taints("vgpu.example.com", "node-a", "node-a", 5, m2["pf"]["dev"], TAINTS[:nt], since)
          if nt else kx.dra_slices_mdev_pf("vgpu.example.com", "node-a", "node-a", 5, m2["pf"], [], None))
    v = CC.random_vf_devs(n, n, no_keys=True)
    for dom in ("example.com", "x.io"):
        _same(_call(kx, "vf_vgpu", dom, v, nt, since),
              kx.dra_slices_vf_vgpu("vgpu.example.com", "node-a", "node-a", 5, v["dev"], TAINTS[:nt], since))


@pytest.mark.parametrize("layout", ["mdev", "vf_vgpu"])
def test_refusals_leave_outputs(kx, layout):
    raw = kx.dra_slices_mdev_pcie_raw if layout == "mdev" else kx.dra_slices_vf_vgpu_pcie_raw
    good = _devs(layout, 70, 1)
    cases = [(dom, good, [], None, -1) for dom in (None, "", "Pcie.example.com", "kubernetes.io", "x.k8s.io", "a" * 64)]
    for rp, sw in [(1 << 63 | 0x8000, CC.NO), (CC.fkey("0000:00:01.0"), 1 << 48 | 0x100), (CC.NO, CC.fkey("0000:01:00.0"))]:
        bad = good.copy()
        bad["root_port"][69], bad["pcie_switch"][69] = rp, sw
        cases.append((CC.DOMAIN, bad, [], None, -7))
        cases.append((CC.DOMAIN, bad, TAINTS[:1], np.full((70, 1), -1, np.int64), -7))
    for dom, devs, tab, since, want in cases:
        out, offs = np.full(64, 0xAB, np.uint8), np.full(4, 0xCD, np.uint64)
        length = C.c_size_t(12345)
        rc = raw("vgpu.example.com", "node-a", "node-a", 5, dom, devs, tab, since, out, length, offs)
        assert rc == want, (dom, rc)
        assert length.value == 12345 and (out == 0xAB).all() and (offs == 0xCD).all()
