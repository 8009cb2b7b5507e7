"""GPU tests of kxpu_dra_slices_vf_vgpu: bytes and slice_off against the CPU oracle (tests/dra_vf_vgpu_oracle.c) from 0 to
2^20 devices, untainted and with taint tables of one and three entries, the longest fields, every optional attribute
coming and going inside a slice and across the 64- and 128-device slice edges, the argument, taint and domain refusals
with the output untouched, the two-call sizing, every output alignment, and calls interleaved with the passthrough and
mdev slice emitters on one context, also with the look-back epoch wrapping every few calls."""
import ctypes as C
import os

import numpy as np
import pytest

import dra_cases as DC
import dra_mdev_cases as MC
import dra_taint_cases as TC
import dra_vf_vgpu_cases as VC
import dra_vf_vgpu_oracle as VO
from kxpu_b200.binding import DraTaint
from oracle import aer_oracle as AO

pytestmark = pytest.mark.gpu

LONG_DRIVER = "d" * 63
LONG_NAME = ".".join(["a" * 63] * 3 + ["b" * 61])
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_vf_vgpu_cfg1.jsonl")


def since_for(table, n, kind, seed=0):
    """an [n, len(table)] taint-time table; the two AER entries of TAINTS3 are never carried together"""
    since = np.stack([TC.since_pattern(n, kind, seed=seed + t) for t in range(len(table))], axis=1) if n else \
        np.zeros((0, len(table)), np.int64)
    if len(table) == 3:
        since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    return since


def raw(kx, driver, pool, node, gen, devs, out=None, cap=0, offs=None, taints=(), since=None):
    """one kxpu_dra_slices_vf_vgpu call: (status, len, n_slices); len / n_slices keep the sentinel 0xDEAD when not
    written"""
    devs = np.ascontiguousarray(devs)
    tab = (DraTaint * max(len(taints), 1))(*[DraTaint(k.encode(), v.encode(), e.encode()) for k, v, e in taints])
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    rc = kx.L.kxpu_dra_slices_vf_vgpu(kx.ctx, driver.encode(), pool.encode(), node.encode(), gen,
                                      devs.ctypes.data if len(devs) else None, len(devs), C.cast(tab, C.c_void_p),
                                      len(taints), None if since is None else since.ctypes.data,
                                      None if out is None else out.ctypes.data, cap, C.byref(ln),
                                      None if offs is None else offs.ctypes.data, C.byref(ns))
    return rc, ln.value, ns.value


def check(kx, devs, driver="vgpu-vf.nvidia.com", pool="node-a", node="node-a", gen=1, taints=(), since=None):
    """kx.dra_slices_vf_vgpu == the oracle, bytes and slice_off"""
    blob, offs = kx.dra_slices_vf_vgpu(driver, pool, node, gen, devs, list(taints), since)
    want, woffs = VO.dra_slices_vf_vgpu(driver, pool, node, gen, devs, taints, since)
    assert blob == want
    assert np.array_equal(offs, woffs)
    return blob, offs


def test_golden_cfg1(kx):
    c = VC.CFG1
    blob, _ = check(kx, VC.cfg1(), c["driver"], c["pool"], c["node"], c["gen"])
    assert blob == open(GOLDEN, "rb").read()


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 4097, 65536, 1 << 20])
def test_sizes_mixed(kx, n):
    check(kx, VC.random_devs(n, seed=2000 + n))


@pytest.mark.parametrize("table", [VC.TAINTS1, VC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129, 4097, 65536, 1 << 20])
def test_sizes_tainted(kx, table, n):
    check(kx, VC.random_devs(n, seed=3000 + n), taints=table, since=since_for(table, n, "some", seed=n))


@pytest.mark.parametrize("n", [129, 65536])
def test_all_attributes_longest_fields(kx, n):
    devs = VC.random_devs(n, seed=8, all_attrs=True)
    blob, _ = check(kx, devs, LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1)
    assert blob.count(b'"resource.kubernetes.io/pcieRoot"') == n and blob.count(b'"parentDeviceID"') == n
    long_taints = [(TC.LONG_KEY, TC.LONG_VALUE, "NoExecute"), (TC.KEY, "", "NoSchedule"), (TC.KEY, TC.VALUE, "NoExecute"),
                   ("x/" + "y" * 63, TC.LONG_VALUE, "NoSchedule")]
    since = np.full((n, 4), TC.SINCE_MAX, np.int64)
    check(kx, devs, LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1, long_taints, since)


def _patterns(n):
    recs = []
    for i in range(n):
        recs.append(VC.rec(group=[0, 4294967294, 300, 9][i % 4], numa=[0, 1, 1 << 63, 3, 1 << 17][i % 5],
                           device=[b"", b"2330", b"f", b"123456"][(i // 2) % 4],
                           product=[b"", b"X", b"P" * 63, b"Q" * 64][(i // 3) % 4], root=[b"", b"pci0000:c0"][(i // 7) % 2],
                           type_key=[b"T", b"NVIDIA_H100XM-1-10C", b"t" * 40][i % 3], vendor=[b"1", b"10de", b"abcdef"][i % 3],
                           type_id=[1, 557, 4294967295, 10][(i // 11) % 4],
                           bdf=[b"0000:c1:00.4", b"1", b"ffff:ff:1f.7abcd"][(i // 13) % 3],
                           parent=[b"0000:c1:00.0", b"1", b"ffff:ff:1f.7abcd"][(i // 5) % 3]))
    devs = np.concatenate(recs)
    edges = [63, 64, 127, 128, 191, 192, 255, 256]  # every optional attribute absent on both sides of each slice edge
    devs["device"][edges], devs["product_len"][edges], devs["pcie_root"][edges], devs["numa_mask"][edges] = b"", 0, b"", 0
    return devs


def test_hand_patterns(kx):
    """each optional attribute (numaNode, parentDeviceID, productName, pcieRoot) comes and goes at its own period,
    inside one slice and across the slice edges at 64, 128, 192 and 256, next to keys, addresses and ids of every
    length; untainted (128 per slice) and tainted (64 per slice), the taints coming and going at the edges too"""
    devs = _patterns(300)
    check(kx, devs)
    since = since_for(VC.TAINTS3, 300, "some", seed=5)
    since[[63, 64, 127, 128, 191, 192, 255, 256]] = -1
    since[[62, 65, 126, 129], 0] = 7
    check(kx, devs, taints=VC.TAINTS3, since=since)
    check(kx, devs, taints=VC.TAINTS1, since=since[:, :1])


@pytest.mark.parametrize("args", [
    ("d" * 64, "p", "n", 1), ("Vfio", "p", "n", 1), ("d", LONG_NAME + "x", "n", 1), ("d", "p", LONG_NAME + "x", 1),
    ("d", "p", "n", 1 << 63), ("a..b", "p", "n", 1), ("d", "p", "-n", 1)])
def test_invalid_arguments_write_nothing(kx, args):
    out = np.full(4096, 0xAB, np.uint8)
    offs = np.full(4, 0xABAB, np.uint64)
    for taints, since in (((), None), (VC.TAINTS1, np.zeros(1, np.int64))):
        rc, ln, ns = raw(kx, *args, VC.cfg1(), out, out.size, offs, taints, since)
        assert (rc, ln, ns) == (-1, 0xDEAD, 0xDEAD)
        assert (out == 0xAB).all() and (offs == 0xABAB).all()


@pytest.mark.parametrize("key,value,effect", [t for t in TC.INVALID if None not in t])
def test_invalid_taints_write_nothing(kx, key, value, effect):
    out = np.full(4096, 0xAB, np.uint8)
    offs = np.full(4, 0xABAB, np.uint64)
    rc, ln, ns = raw(kx, "d", "p", "n", 1, VC.cfg1(), out, out.size, offs, [(key, value, effect)], np.zeros(1, np.int64))
    assert (rc, ln, ns) == (-1, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()
    five = [("k%d" % t, "", "NoSchedule") for t in range(5)]
    assert raw(kx, "d", "p", "n", 1, VC.cfg1(), out, out.size, offs, five, np.zeros(5, np.int64)) == (-1, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all()


@pytest.mark.parametrize("why,field,value", VC.BAD)
def test_out_of_domain_writes_nothing(kx, why, field, value):
    devs = np.concatenate([VC.random_devs(200, seed=3), VC.bad_rec(field, value), VC.random_devs(5, seed=4)])
    assert VO.dra_slices_vf_vgpu("d", "p", "n", 1, devs) == (-7, why)
    out = np.full(1 << 18, 0xAB, np.uint8)
    offs = np.full(8, 0xABAB, np.uint64)
    for taints, since in (((), None), (VC.TAINTS1, np.full(len(devs), -1, np.int64))):
        rc, ln, ns = raw(kx, "d", "p", "n", 1, devs, out, out.size, offs, taints, since)
        assert (rc, ln, ns) == (-7, 0xDEAD, 0xDEAD)
        assert (out == 0xAB).all() and (offs == 0xABAB).all()
        msg = kx.L.kxpu_last_error(kx.ctx).decode()
        assert "dra_slices_vf_vgpu: " in msg and why in msg


@pytest.mark.parametrize("case", ["since", "duplicate"])
def test_taint_domain_writes_nothing(kx, case):
    devs = VC.random_devs(100, seed=6)
    since = np.full((100, 3), -1, np.int64)
    since[70] = [-1, -1, TC.SINCE_MAX + 1] if case == "since" else [-1, 5, 6]
    assert VO.dra_slices_vf_vgpu("d", "p", "n", 1, devs, VC.TAINTS3, since) == \
        (-7, "taint_since" if case == "since" else "taint_duplicate")
    out = np.full(1 << 16, 0xAB, np.uint8)
    offs = np.full(4, 0xABAB, np.uint64)
    assert raw(kx, "d", "p", "n", 1, devs, out, out.size, offs, VC.TAINTS3, since) == (-7, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()


@pytest.mark.parametrize("tainted", [False, True])
def test_sizing_exact_and_short(kx, tainted):
    devs = VC.random_devs(300, seed=11)
    taints, since = (VC.TAINTS3, since_for(VC.TAINTS3, 300, "all")) if tainted else ((), None)
    want, woffs = VO.dra_slices_vf_vgpu("d", "p", "n", 5, devs, taints, since)
    S = 5 if tainted else 3
    rc, ln, ns = raw(kx, "d", "p", "n", 5, devs, taints=taints, since=since)
    assert (rc, ln, ns) == (-4, len(want), S)
    out = np.full(len(want) + 16, 0xAB, np.uint8)
    offs = np.full(ns + 2, 0xABAB, np.uint64)
    assert raw(kx, "d", "p", "n", 5, devs, out, len(want) - 1, offs, taints, since) == (-4, len(want), S)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()
    assert raw(kx, "d", "p", "n", 5, devs, out, len(want), offs, taints, since) == (0, len(want), S)
    assert out[:len(want)].tobytes() == want and (out[len(want):] == 0xAB).all()
    assert np.array_equal(offs[:ns + 1], woffs) and offs[ns + 1] == 0xABAB
    assert raw(kx, "d", "p", "n", 5, devs, out, len(want), None, taints, since) == (0, len(want), S)


def test_output_pointer_every_phase(kx):
    devs = VC.random_devs(129, seed=12)
    for taints, since in (((), None), (VC.TAINTS1, since_for(VC.TAINTS1, 129, "some"))):
        want, _ = VO.dra_slices_vf_vgpu("d", "p", "n", 1, devs, taints, since)
        buf = np.full(len(want) + 64, 0xAB, np.uint8)
        base = (16 - buf.ctypes.data % 16) % 16
        for ph in range(16):
            buf[:] = 0xAB
            view = buf[base + ph:base + ph + len(want)]
            assert raw(kx, "d", "p", "n", 1, devs, view, len(want), None, taints, since)[0] == 0
            assert view.tobytes() == want
            assert (buf[:base + ph] == 0xAB).all() and (buf[base + ph + len(want):] == 0xAB).all()


def _interleave(kx):
    for r in range(12):
        n = [0, 129, 4097, 300, 65536, 1][r % 6]
        table = [(), VC.TAINTS1, VC.TAINTS3][r % 3]
        since = since_for(table, n, "some", seed=r) if table else None
        check(kx, VC.random_devs(n, seed=r), gen=r + 1, taints=table, since=since)
        pci = DC.random_devs([1, 4097, 129][r % 3], seed=50 + r)
        ptab = [("vfio.nvidia.com/unhealthy", "vfio-device-missing", "NoSchedule")]
        psince = TC.since_pattern(len(pci), "some", seed=r).reshape(-1, 1)
        blob, offs = kx.dra_slices_taints("vfio.nvidia.com", "node-a", "node-a", r + 1, pci, ptab, psince)
        want, woffs = AO.dra_slices_taints("vfio.nvidia.com", "node-a", "node-a", r + 1, pci, ptab, psince)
        assert blob == want and np.array_equal(offs, woffs)
        mdev = MC.random_devs([300, 1, 4097][r % 3], seed=70 + r)
        blob, offs = kx.dra_slices_mdev_taints("vgpu.nvidia.com", "node-a", "node-a", r + 1, mdev, ptab, None)
        want, woffs = AO.dra_slices_mdev_taints("vgpu.nvidia.com", "node-a", "node-a", r + 1, mdev, ptab, None)
        assert blob == want and np.array_equal(offs, woffs)


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
