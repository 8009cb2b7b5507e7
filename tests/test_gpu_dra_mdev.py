"""GPU tests of kxpu_dra_slices_mdev (include/kxpu.h, ABI v10): bytes and slice_off against the CPU oracle
(oracle/kxpu_dra_mdev_oracle.c) at slice edges and large pools, the longest fields, every optional attribute coming and going
inside a slice and across a slice edge, the argument and domain refusals with the output untouched, the two-call
sizing, unaligned output pointers, and calls interleaved with kxpu_dra_slices and both CDI emitters on one context,
also with the look-back epoch wrapping every few calls."""
import ctypes as C
import os

import numpy as np
import pytest

import dra_cases as DC
import dra_mdev_cases as MC
from oracle import dra_mdev_oracle as DMO
from oracle import dra_oracle as DO
from oracle import mdev_oracle as MO
from oracle import xpu_oracle as XO

pytestmark = pytest.mark.gpu

LONG_DRIVER = "d" * 63
LONG_NAME = ".".join(["a" * 63] * 3 + ["b" * 61])
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_mdev_cfg1.jsonl")


def raw(kx, driver, pool, node, gen, devs, out=None, cap=0, offs=None):
    """one kxpu_dra_slices_mdev call: (status, len, n_slices); len / n_slices keep the sentinel 0xDEAD when not written"""
    devs = np.ascontiguousarray(devs)
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    rc = kx.L.kxpu_dra_slices_mdev(kx.ctx, driver.encode(), pool.encode(), node.encode(), gen,
                                   devs.ctypes.data if len(devs) else None, len(devs),
                                   None if out is None else out.ctypes.data, cap, C.byref(ln),
                                   None if offs is None else offs.ctypes.data, C.byref(ns))
    return rc, ln.value, ns.value


def check(kx, devs, driver="vgpu.nvidia.com", pool="node-a", node="node-a", gen=1):
    """kx.dra_slices_mdev == the oracle, bytes and slice_off"""
    blob, offs = kx.dra_slices_mdev(driver, pool, node, gen, devs)
    want, woffs = DMO.dra_slices_mdev(driver, pool, node, gen, devs)
    assert blob == want
    assert np.array_equal(offs, woffs)
    return blob, offs


def test_golden_cfg1(kx):
    c = MC.CFG1
    blob, _ = check(kx, MC.cfg1(), c["driver"], c["pool"], c["node"], c["gen"])
    assert blob == open(GOLDEN, "rb").read()


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 4097, 65536, 1 << 20])
def test_sizes_mixed(kx, n):
    check(kx, MC.random_devs(n, seed=2000 + n))


@pytest.mark.parametrize("n", [129, 65536])
def test_all_attributes_longest_fields(kx, n):
    devs = MC.random_devs(n, seed=8, all_attrs=True)
    blob, _ = check(kx, devs, LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1)
    assert blob.count(b'"resource.kubernetes.io/pcieRoot"') == n and blob.count(b'"parentDeviceID"') == n


def test_hand_patterns(kx):
    """each optional attribute (numaNode, parentDeviceID, productName, pcieRoot) comes and goes at its own period,
    inside one slice and across the slice edges at 128 and 256, next to types, parents and ids of every length"""
    recs = []
    for i in range(300):
        recs.append(MC.rec(group=[0, 4294967294, 300, 9][i % 4], numa=[0, 1, 1 << 63, 3, 1 << 17][i % 5],
                           device=[b"", b"2330", b"f", b"123456"][(i // 2) % 4],
                           product=[b"", b"X", b"P" * 63, b"Q" * 64][(i // 3) % 4], root=[b"", b"pci0000:c0"][(i // 7) % 2],
                           mdev_type=[b"T", b"NVIDIA_H100XM-1-10C", b"t" * 40][i % 3], vendor=[b"1", b"10de", b"abcdef"][i % 3],
                           parent=[b"0000:c1:00.0", b"1", b"ffff:ff:1f.7abcd"][(i // 5) % 3]))
    devs = np.concatenate(recs)
    edges = [127, 128, 255, 256]  # every optional attribute absent on both sides of each slice edge
    devs["device"][edges], devs["product_len"][edges], devs["pcie_root"][edges], devs["numa_mask"][edges] = b"", 0, b"", 0
    check(kx, devs)


@pytest.mark.parametrize("args", [
    ("d" * 64, "p", "n", 1), ("Vfio", "p", "n", 1), ("d", LONG_NAME + "x", "n", 1), ("d", "p", LONG_NAME + "x", 1),
    ("d", "p", "n", 1 << 63), ("a..b", "p", "n", 1), ("d", "p", "-n", 1)])
def test_invalid_arguments_write_nothing(kx, args):
    out = np.full(4096, 0xAB, np.uint8)
    offs = np.full(4, 0xABAB, np.uint64)
    rc, ln, ns = raw(kx, *args, MC.cfg1(), out, out.size, offs)
    assert (rc, ln, ns) == (-1, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()


@pytest.mark.parametrize("why,field,value", MC.BAD)
def test_out_of_domain_writes_nothing(kx, why, field, value):
    devs = np.concatenate([MC.random_devs(200, seed=3), MC.bad_rec(field, value), MC.random_devs(5, seed=4)])
    assert DMO.dra_slices_mdev("d", "p", "n", 1, devs) == (-7, why)
    out = np.full(1 << 18, 0xAB, np.uint8)
    offs = np.full(4, 0xABAB, np.uint64)
    rc, ln, ns = raw(kx, "d", "p", "n", 1, devs, out, out.size, offs)
    assert (rc, ln, ns) == (-7, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()
    assert "dra_slices_mdev: " in kx.L.kxpu_last_error(kx.ctx).decode() and why in kx.L.kxpu_last_error(kx.ctx).decode()


def test_sizing_exact_and_short(kx):
    devs = MC.random_devs(300, seed=11)
    want, woffs = DMO.dra_slices_mdev("d", "p", "n", 5, devs)
    rc, ln, ns = raw(kx, "d", "p", "n", 5, devs)
    assert (rc, ln, ns) == (-4, len(want), 3)
    out = np.full(len(want) + 16, 0xAB, np.uint8)
    offs = np.full(ns + 2, 0xABAB, np.uint64)
    assert raw(kx, "d", "p", "n", 5, devs, out, len(want) - 1, offs) == (-4, len(want), 3)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()
    assert raw(kx, "d", "p", "n", 5, devs, out, len(want), offs) == (0, len(want), 3)
    assert out[:len(want)].tobytes() == want and (out[len(want):] == 0xAB).all()
    assert np.array_equal(offs[:ns + 1], woffs) and offs[ns + 1] == 0xABAB
    assert raw(kx, "d", "p", "n", 5, devs, out, len(want), None) == (0, len(want), 3)  # slice_off may be NULL


def test_output_pointer_every_phase(kx):
    devs = MC.random_devs(129, seed=12)
    want, _ = DMO.dra_slices_mdev("d", "p", "n", 1, devs)
    buf = np.full(len(want) + 64, 0xAB, np.uint8)
    base = (16 - buf.ctypes.data % 16) % 16
    for ph in range(16):
        buf[:] = 0xAB
        view = buf[base + ph:base + ph + len(want)]
        assert raw(kx, "d", "p", "n", 1, devs, view, len(want))[0] == 0
        assert view.tobytes() == want
        assert (buf[:base + ph] == 0xAB).all() and (buf[base + ph + len(want):] == 0xAB).all()


def _interleave(kx):
    kind = b"vfio.example.com/xpu"
    mkind = b"vgpu.example.com/vgpu"
    cdi = np.zeros(5000, XO.CDIDEV_DTYPE)
    cdi["bdf"], cdi["iommu_group"], cdi["index"] = b"0000:c1:00.0", np.arange(5000), np.arange(5000)
    mcdi = np.zeros(3000, MO.MDEVCDI_DTYPE)
    mcdi["uuid"], mcdi["parent"] = MC.UUID, b"0000:c1:00.0"
    mcdi["iommu_group"], mcdi["index"] = np.arange(3000), np.arange(3000)
    for r in range(12):
        n = [0, 129, 4097, 300, 65536, 1][r % 6]
        check(kx, MC.random_devs(n, seed=r), gen=r + 1)
        pci = DC.random_devs([1, 4097, 129][r % 3], seed=50 + r)
        blob, offs = kx.dra_slices("vfio.nvidia.com", "node-a", "node-a", r + 1, pci)
        want, woffs = DO.dra_slices("vfio.nvidia.com", "node-a", "node-a", r + 1, pci)
        assert blob == want and np.array_equal(offs, woffs)
        assert kx.cdi_emit(1, cdi[:4000 + 100 * r], kind) == XO.cdi_emit_kind(1, kind, cdi[:4000 + 100 * r])
        assert kx.cdi_emit_mdev(r & 1, mcdi[:2000 + 50 * r], mkind) == MO.cdi_emit_mdev(r & 1, mkind, mcdi[:2000 + 50 * r])


def test_interleaved_with_other_emitters(kx):
    _interleave(kx)


@pytest.mark.parametrize("limit", ["2", "3", "5"])
def test_interleaved_under_epoch_wrap(monkeypatch, limit):
    import kxpu_b200 as K
    monkeypatch.setenv("KXPU_SCAN_EPOCH_LIMIT", limit)
    k = K.Kxpu(0)
    try:
        _interleave(k)
    finally:
        k.close()
