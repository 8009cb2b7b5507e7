"""GPU tests of kxpu_dra_slices (include/kxpu.h, ABI v9): bytes and slice_off against the CPU oracle
(oracle/kxpu_dra_oracle.c) at slice edges and large pools, every optional attribute in mixed patterns, the argument
and domain refusals with the output untouched, the two-call sizing, unaligned output pointers, and calls interleaved
with the CDI emitter on one context, also with the look-back epoch wrapping every few calls."""
import ctypes as C
import os

import numpy as np
import pytest

import dra_cases as DC
from oracle import dra_oracle as DO
from oracle import xpu_oracle as XO

pytestmark = pytest.mark.gpu

LONG_DRIVER = "d" * 63
LONG_NAME = ".".join(["a" * 63] * 3 + ["b" * 61])
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_cfg1.jsonl")


def raw(kx, driver, pool, node, gen, devs, out=None, cap=0, offs=None):
    """one kxpu_dra_slices call: (status, len, n_slices); len / n_slices keep the sentinel 0xDEAD when not written"""
    devs = np.ascontiguousarray(devs)
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    rc = kx.L.kxpu_dra_slices(kx.ctx, driver.encode(), pool.encode(), node.encode(), gen,
                              devs.ctypes.data if len(devs) else None, len(devs),
                              None if out is None else out.ctypes.data, cap, C.byref(ln),
                              None if offs is None else offs.ctypes.data, C.byref(ns))
    return rc, ln.value, ns.value


def check(kx, devs, driver="vfio.nvidia.com", pool="node-a", node="node-a", gen=1):
    """kx.dra_slices == the oracle, bytes and slice_off"""
    blob, offs = kx.dra_slices(driver, pool, node, gen, devs)
    want, woffs = DO.dra_slices(driver, pool, node, gen, devs)
    assert blob == want
    assert np.array_equal(offs, woffs)
    return blob, offs


def test_golden_cfg1(kx):
    blob, offs = check(kx, DC.cfg1(), **DC.CFG1)
    assert blob == open(GOLDEN, "rb").read()


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257, 4097, 65536, 1 << 20])
def test_sizes_mixed(kx, n):
    check(kx, DC.random_devs(n, seed=1000 + n))


@pytest.mark.parametrize("n", [129, 65536])
def test_all_attributes_longest_fields(kx, n):
    check(kx, DC.random_devs(n, seed=7, all_attrs=True), LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1)


def test_hand_patterns(kx):
    """masks 0 / bit 0 / bit 63 / two bits, product_len 0 / 1 / 63 / 64, groups 0 and 4294967294, root present or not,
    alternating inside one slice and across a slice edge"""
    recs = []
    for i in range(300):
        recs.append(DC.rec(group=[0, 4294967294, 214, 9][i % 4], numa=[0, 1, 1 << 63, 3, 1 << 17][i % 5],
                           product=[b"", b"X", b"P" * 63, b"Q" * 64][(i // 3) % 4], root=[b"", b"pci0000:c0"][(i // 2) % 2],
                           vendor=[b"1", b"10de", b"abcdef"][i % 3], device=[b"2330", b"f", b"123456"][(i // 7) % 3],
                           bdf=[b"0000:c1:00.0", b"1", b"ffff:ff:1f.7abcd"][(i // 5) % 3]))
    check(kx, np.concatenate(recs))


@pytest.mark.parametrize("args", [
    ("d" * 64, "p", "n", 1), ("Vfio", "p", "n", 1), ("d", LONG_NAME + "x", "n", 1), ("d", "p", LONG_NAME + "x", 1),
    ("d", "p", "n", 1 << 63), ("a..b", "p", "n", 1), ("d", "p", "-n", 1)])
def test_invalid_arguments_write_nothing(kx, args):
    out = np.full(4096, 0xAB, np.uint8)
    offs = np.full(4, 0xABAB, np.uint64)
    rc, ln, ns = raw(kx, *args, DC.cfg1(), out, out.size, offs)
    assert (rc, ln, ns) == (-1, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()


@pytest.mark.parametrize("why,field,value", DC.BAD)
def test_out_of_domain_writes_nothing(kx, why, field, value):
    devs = np.concatenate([DC.random_devs(200, seed=3), DC.bad_rec(field, value), DC.random_devs(5, seed=4)])
    assert DO.dra_slices("d", "p", "n", 1, devs)[0] == -7
    out = np.full(1 << 17, 0xAB, np.uint8)
    offs = np.full(4, 0xABAB, np.uint64)
    rc, ln, ns = raw(kx, "d", "p", "n", 1, devs, out, out.size, offs)
    assert (rc, ln, ns) == (-7, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()


def test_sizing_exact_and_short(kx):
    devs = DC.random_devs(300, seed=11)
    want, woffs = DO.dra_slices("d", "p", "n", 5, devs)
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
    devs = DC.random_devs(129, seed=12)
    want, _ = DO.dra_slices("d", "p", "n", 1, devs)
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
    cdi = np.zeros(5000, XO.CDIDEV_DTYPE)
    cdi["bdf"], cdi["iommu_group"], cdi["index"] = b"0000:c1:00.0", np.arange(5000), np.arange(5000)
    cdi_want = XO.cdi_emit_kind(1, kind, cdi)
    for r in range(12):
        n = [0, 129, 4097, 300, 65536, 1][r % 6]
        check(kx, DC.random_devs(n, seed=r), gen=r + 1)
        assert kx.cdi_emit(1, cdi[:4000 + 100 * r], kind) == XO.cdi_emit_kind(1, kind, cdi[:4000 + 100 * r])
    assert kx.cdi_emit(1, cdi, kind) == cdi_want


def test_interleaved_with_cdi_emit(kx):
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
