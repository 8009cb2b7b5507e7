"""GPU tests of kxpu_pcie_ports and kxpu_dra_slices_pcie against the C checker (tests/dra_pcie_oracle.c): the rule on
its hand cases and on walks from n = 0 to 2^20 at the parse and group tile edges; the slices from 0 to 2^20 devices at
the slice seams (63 / 64 / 65, 127 / 128 / 129), with taint tables of 0, 1 and 3 entries, at every position of the two
names and with 16-byte VMD addresses; pools with every key absent against kxpu_dra_slices_pf and
kxpu_dra_slices_taints; every refusal with the outputs untouched."""
import ctypes as C

import numpy as np
import pytest

import dra_pcie_cases as CC
import dra_pcie_oracle as CO
import dra_pf_cases as PC
from kxpu_b200.binding import KxpuError, DraTaint
from test_gpu_dra_pf import since_for

pytestmark = pytest.mark.gpu


def _same(got, want):
    assert got[0] == want[0] and list(got[1]) == list(want[1])


# ------------------------------------------------------------------ kxpu_pcie_ports

@pytest.mark.parametrize("case", CC.HAND, ids=[c[0] for c in CC.HAND])
def test_ports_hand_cases(kx, case):
    _, groups, want = case
    rp, sw = kx.pcie_ports(*CC.walk(groups))
    assert (list(rp), list(sw)) == tuple(CC.expected(want))


@pytest.mark.parametrize("groups", [0, 1, 15, 16, 17, 255, 256, 257, 5000, 1 << 16])
def test_ports_parity(kx, groups):
    walk = CC.random_walk(groups, seed=groups)
    rp, sw = kx.pcie_ports(*walk)
    want = CO.pcie_ports(*walk)
    assert np.array_equal(rp, want[0]) and np.array_equal(sw, want[1])


def test_ports_million_records(kx):
    """2^20 records (a seeded walk's records repeated), one per group, then four to a group"""
    recs, paths, _, _ = CC.random_walk(4096, seed=3, max_members=2)
    n = 1 << 20
    recs, paths = np.resize(recs, n), np.resize(paths, n)
    for off, mem in ((np.arange(n + 1, dtype=np.uint32), np.arange(n, dtype=np.uint32)),
                     (np.append(np.arange(0, n, 4), n).astype(np.uint32), np.arange(n, dtype=np.uint32))):
        rp, sw = kx.pcie_ports(recs, paths, off, mem)
        want = CO.pcie_ports(recs, paths, off, mem)
        assert np.array_equal(rp, want[0]) and np.array_equal(sw, want[1])


def test_ports_refusals_touch_nothing(kx):
    recs, paths, off, mem = CC.walk([[m] for m in CC.EX.gpu_paths()])
    rp, sw = np.full(8, 7, np.uint64), np.full(8, 7, np.uint64)
    bad = [(off, np.array([0, 1, 2, 3, 4, 5, 6, 8], np.uint32), -1),  # a member >= n
           (np.array([0, 2, 1, 3, 4, 5, 6, 7, 8], np.uint32), mem, -1)]  # offsets decrease
    for o, m, rc in bad:
        with pytest.raises(KxpuError) as e:
            kx.pcie_ports_raw(recs, paths, o, m, rp, sw)
        assert e.value.status == rc
        assert (rp == 7).all() and (sw == 7).all()
    L = kx.L
    assert L.kxpu_pcie_ports(kx.ctx, None, None, 8, off.ctypes.data, mem.ctypes.data, 8, rp.ctypes.data, sw.ctypes.data) == -1
    assert L.kxpu_pcie_ports(kx.ctx, recs.ctypes.data, paths.ctypes.data, 8, None, mem.ctypes.data, 8, rp.ctypes.data,
                             sw.ctypes.data) == -1
    assert L.kxpu_pcie_ports(kx.ctx, recs.ctypes.data, paths.ctypes.data, 8, off.ctypes.data, None, 8, rp.ctypes.data,
                             sw.ctypes.data) == -1
    assert L.kxpu_pcie_ports(kx.ctx, recs.ctypes.data, paths.ctypes.data, 8, off.ctypes.data, mem.ctypes.data, 8, None,
                             sw.ctypes.data) == -1
    assert L.kxpu_pcie_ports(kx.ctx, recs.ctypes.data, paths.ctypes.data, 1 << 28, off.ctypes.data, mem.ctypes.data, 8,
                             rp.ctypes.data, sw.ctypes.data) == -7
    assert (rp == 7).all() and (sw == 7).all()


# ------------------------------------------------------------------ kxpu_dra_slices_pcie

def gpu(kx, devs, taints=(), since=None, dom=CC.DOMAIN, driver="d", pool="p", node="n", gen=1):
    return kx.dra_slices_pcie(driver, pool, node, gen, dom, devs, list(taints), since)


def cpu(devs, taints=(), since=None, dom=CC.DOMAIN, driver="d", pool="p", node="n", gen=1):
    return CO.dra_slices_pcie(driver, pool, node, gen, dom, devs, taints, since)


def test_golden_cfg1(kx):
    import os
    want = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_pcie_cfg1.jsonl"), "rb").read()
    blob, offs = gpu(kx, CC.cfg1(), driver="vfio.example.com", pool="node-a", node="node-a")
    assert blob == want and list(offs) == [0, len(want)]


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 4096, 1 << 20])
def test_untainted_parity(kx, n):
    devs = CC.random_devs(n, seed=n)
    _same(gpu(kx, devs), cpu(devs))


@pytest.mark.parametrize("table", [PC.TAINTS1, PC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 127, 128, 129, 1 << 20])
def test_tainted_parity(kx, table, n):
    devs = CC.random_devs(n, seed=7 + n)
    since = since_for(table, n, "some", seed=n)
    _same(gpu(kx, devs, table, since), cpu(devs, table, since))


@pytest.mark.parametrize("pos", [p for p in range(10) if CC.POSITIONS[p]])
@pytest.mark.parametrize("nt", [0, 1, 3])
def test_every_position(kx, pos, nt):
    n = 300
    devs = CC.random_devs(n, seed=pos, all_attrs=pos % 2 == 1)
    table = {0: (), 1: PC.TAINTS1, 3: PC.TAINTS3}[nt]
    since = None if nt == 0 else since_for(table, n, "some", seed=pos)
    _same(gpu(kx, devs, table, since, dom=CC.POSITIONS[pos]), cpu(devs, table, since, dom=CC.POSITIONS[pos]))


@pytest.mark.parametrize("dom", CC.GOOD_DOMAINS)
def test_domains_at_the_limits(kx, dom):
    devs = CC.random_devs(257, seed=9, all_attrs=True)
    _same(gpu(kx, devs, dom=dom), cpu(devs, dom=dom))
    since = since_for(PC.TAINTS3, 257, "all")
    _same(gpu(kx, devs, PC.TAINTS3, since, dom=dom), cpu(devs, PC.TAINTS3, since, dom=dom))


@pytest.mark.parametrize("nt", [0, 1, 3])
def test_long_vmd_addresses(kx, nt):
    n = 129
    devs = CC.random_devs(n, seed=1, all_attrs=True, long_addr=True)
    table = {0: (), 1: PC.TAINTS1, 3: PC.TAINTS3}[nt]
    since = None if nt == 0 else since_for(table, n, "all")
    _same(gpu(kx, devs, table, since, dom="a" * 63), cpu(devs, table, since, dom="a" * 63))


@pytest.mark.parametrize("n", [0, 1, 65, 129, 1 << 16])
@pytest.mark.parametrize("nt", [0, 1, 3])
def test_no_keys_is_the_pf_call(kx, n, nt):
    table = {0: (), 1: PC.TAINTS1, 3: PC.TAINTS3}[nt]
    since = None if nt == 0 else since_for(table, n, "some", seed=n)
    devs = CC.random_devs(n, seed=n, no_keys=True)
    for dom in (CC.DOMAIN, "a.io", "w.io"):
        _same(gpu(kx, devs, table, since, dom=dom), kx.dra_slices_pf("d", "p", "n", 1, devs["pf"], list(table), since))
    devs = CC.random_devs(n, seed=n, no_keys=True, no_physfn=True)
    _same(gpu(kx, devs, table, since),
          kx.dra_slices_taints("d", "p", "n", 1, devs["pf"]["dev"], list(table or PC.TAINTS3), since))


def _raw(kx, devs, dom, out, offs, driver=b"d", taints=(), since=None):
    tab = (DraTaint * max(len(taints), 1))(*[DraTaint(k.encode(), v.encode(), e.encode()) for k, v, e in taints])
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    rc = kx.L.kxpu_dra_slices_pcie(kx.ctx, driver, b"p", b"n", 1, None if dom is None else dom.encode(),
                                   devs.ctypes.data if len(devs) else None, len(devs), C.cast(tab, C.c_void_p),
                                   len(taints), None if since is None else since.ctypes.data, out.ctypes.data,
                                   len(out), C.byref(ln), offs.ctypes.data, C.byref(ns))
    return rc, ln.value, ns.value


def test_refusals_touch_nothing(kx):
    out, offs = np.full(1 << 16, 0x5A, np.uint8), np.full(64, 7, np.uint64)
    good = CC.cfg1()
    cases = [(good, d, -1) for d in CC.BAD_DOMAINS]
    cases.append((good, CC.DOMAIN, -1))  # with a bad driver below
    for why, rp, sw in CC.BAD_KEYS:
        devs = CC.cfg1()
        devs[2]["root_port"], devs[2]["pcie_switch"] = rp, sw
        cases.append((devs, CC.DOMAIN, -7))
        assert cpu(devs) == (-7, why)
    for i, (devs, dom, rc) in enumerate(cases):
        got = _raw(kx, devs, dom, out, offs, driver=b"D" if i == len(CC.BAD_DOMAINS) else b"d")
        assert got == (rc, 0xDEAD, 0xDEAD)
        assert (out == 0x5A).all() and (offs == 7).all()
    # a bad key on a tainted call, and a bad taint table with a good domain
    devs = CC.cfg1()
    devs[0]["root_port"] = 1 << 63
    since = np.zeros((4, 1), np.int64)
    assert _raw(kx, devs, CC.DOMAIN, out, offs, taints=PC.TAINTS1, since=since)[0] == -7
    assert _raw(kx, CC.cfg1(), CC.DOMAIN, out, offs, taints=[("bad key!", "", "NoSchedule")], since=since)[0] == -1
    assert (out == 0x5A).all() and (offs == 7).all()
