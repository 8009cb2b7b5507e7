"""GPU tests of kxpu_aer_ports and kxpu_aer_ports_mdev against the C checker (tests/aer_ports_oracle.c): the rule on its
hand cases, seeded walks from n = 0 to 2^20 at the parse, thread-block and scan-tile edges (switch trees of every depth,
mixed chain ends, VMD domains, unknown and malformed paths, mdevs on PFs and VFs), and every refusal with the outputs
untouched."""
import ctypes as C

import numpy as np
import pytest

import aer_ports_cases as AC
import aer_ports_oracle as CO
import dra_pcie_cases as DC
import vgpu_pcie_cases as VC
from kxpu_b200 import workloads as W
from kxpu_b200.binding import E_INVALID, E_UNSUPPORTED, KxpuError

pytestmark = pytest.mark.gpu


def _same(got, want):
    assert len(got) == len(want) == 3
    for g, w in zip(got, want):
        assert np.array_equal(np.asarray(g, np.uint64), np.asarray(w, np.uint64))


@pytest.mark.parametrize("case", AC.PCI, ids=[c[0] for c in AC.PCI])
def test_pci_hand_cases(kx, case):
    _, rows, want = case
    _same(kx.aer_ports(*AC.pci_walk(rows)), AC.expected(want))


@pytest.mark.parametrize("case", AC.MDEV, ids=[c[0] for c in AC.MDEV])
def test_mdev_hand_cases(kx, case):
    _, rows, want = case
    _same(kx.aer_ports(*AC.mdev_walk(rows)), AC.expected(want))


@pytest.mark.parametrize("groups", [0, 1, 15, 16, 17, 255, 256, 257, 5000])
def test_pci_random_walks(kx, groups):
    recs, paths, _, _ = DC.random_walk(groups, seed=groups, unknown=0.2)
    _same(kx.aer_ports(recs, paths), CO.aer_ports(recs, paths))


@pytest.mark.parametrize("n", [1, 255, 256, 257, 4095, 4096, 4097, 20000])
def test_mdev_random_walks(kx, n):
    (recs, paths, _, _), _ = VC.random_walk(n, seed=n)
    _same(kx.aer_ports(recs, paths), CO.aer_ports(recs, paths))


@pytest.mark.parametrize("depth,fanout,mixed", [(0, 1, False), (1, 32, False), (2, 8, False), (3, 4, False),
                                                (3, 4, True), (2, 16, True)])
def test_switch_trees_million_records(kx, depth, fanout, mixed):
    recs, paths = W.aer_port_walk(1 << 20, depth=depth, fanout=fanout, seed=depth * 64 + fanout, mixed=mixed)
    got = kx.aer_ports(recs, paths)
    _same(got, CO.aer_ports(recs, paths))
    if not mixed:  # every leaf has 2 * depth + 1 ports; per root port: itself, then per level its switches' ports
        assert got[0][-1] == (2 * depth + 1) << 20
        per_root = 1 + sum(fanout ** k + fanout ** (k + 1) for k in range(depth))
        assert len(got[2]) == (1 << 20) // fanout ** depth * per_root


def test_hgx_walk_million_records(kx):
    recs, paths, _, _ = W.pcie_walk(1 << 20, seed=21)
    _same(kx.aer_ports(recs, paths), CO.aer_ports(recs, paths))


def test_mdev_walk_million_records(kx):
    recs, paths, _, _ = W.pcie_ports_mdev_walk(1 << 20)
    _same(kx.aer_ports(recs, paths), CO.aer_ports(recs, paths))


@pytest.mark.parametrize("mdev", [False, True])
def test_refusals_touch_nothing(kx, mdev):
    if mdev:
        recs, paths = AC.mdev_walk(AC.MDEV[0][1])
    else:
        recs, paths = AC.pci_walk(AC.PCI[1][1])
    n = len(recs)
    off, of, key = np.full(n + 1, 7, np.uint32), np.full(8 * n, 7, np.uint32), np.full(8 * n, 7, np.uint64)
    nk = C.c_uint32(7)
    cases = [(dict(recs=None), E_INVALID), (dict(paths=None), E_INVALID), (dict(port_off=None), E_INVALID),
             (dict(port_of=None), E_INVALID), (dict(port_key=None), E_INVALID), (dict(n_ports=None), E_INVALID),
             (dict(n=1 << 28), E_UNSUPPORTED), (dict(n=(1 << 28) + 5), E_UNSUPPORTED)]
    for change, rc in cases:
        a = dict(recs=recs, paths=paths, port_off=off, port_of=of, port_key=key, n_ports=C.byref(nk), n=n)
        a.update(change)
        with pytest.raises(KxpuError) as e:
            kx.aer_ports_raw(a["recs"], a["paths"], a["port_off"], a["port_of"], a["port_key"], a["n_ports"], n=a["n"],
                             mdev=mdev)
        assert e.value.status == rc
        assert (off == 7).all() and (of == 7).all() and (key == 7).all() and nk.value == 7
    f = kx.L.kxpu_aer_ports_mdev if mdev else kx.L.kxpu_aer_ports
    assert f(None, recs.ctypes.data, paths.ctypes.data, n, off.ctypes.data, of.ctypes.data, key.ctypes.data,
             C.byref(nk)) == E_INVALID
    assert (off == 7).all() and (of == 7).all() and (key == 7).all() and nk.value == 7


@pytest.mark.parametrize("mdev", [False, True])
def test_empty_walk(kx, mdev):
    off = np.full(1, 7, np.uint32)
    kx.aer_ports_raw(None, None, off, None, None, None, n=0, mdev=mdev)
    assert off[0] == 0
    nk = C.c_uint32(7)
    kx.aer_ports_raw(None, None, off, None, None, C.byref(nk), n=0, mdev=mdev)
    assert nk.value == 0
