"""GPU tests of the calls for mdev vGPUs on SR-IOV VFs: kxpu_mdev_pf against the C oracle (tests/mdev_pf_oracle.c) on
the hand cases and on walks up to 2^20 mdevs among 2^20 PCI records, and kxpu_dra_slices_mdev_pf's bytes and slice_off
against the oracle from 0 to 2^20 devices, untainted and with taint tables of one and three entries; a pool whose every
physfn is empty against kxpu_dra_slices_mdev_taints byte for byte; every KXPU_E_INVALID and KXPU_E_UNSUPPORTED case of
both calls with the outputs untouched."""
import ctypes as C
import os

import numpy as np
import pytest

import dra_mdev_cases as MC
import dra_taint_cases as TC
import mdev_pf_cases as PC
import mdev_pf_oracle as MO
from kxpu_b200 import workloads as W
from kxpu_b200.binding import DraTaint

pytestmark = pytest.mark.gpu

NO_PF = PC.NO_PF
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_mdev_pf_cfg1.jsonl")
WALK = [b"0000:41:00.0", b"0000:41:00.4", b"0000:41:00.5", b"0000:c1:00.0", b"0000:41:00.0", b"0000:81:00.0"]


def since_for(table, n, kind, seed=0):
    since = np.stack([TC.since_pattern(n, kind, seed=seed + t) for t in range(len(table))], axis=1) if n else \
        np.zeros((0, len(table)), np.int64)
    if len(table) == 3:
        since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    return since


def check_join(kx, recs, m, s):
    got = kx.mdev_pf(recs, m, s)
    assert got.tolist() == MO.mdev_pf(recs, m, s)
    return got


def test_join_hand_cases(kx):
    pairs = [(b"0000:41:00.4", b"0000:41:00.0", 0), (b"0000:c1:00.0", b"", 0),
             (b"0000:41:00.4", b"0000:41:00.0", PC.SR_PHYSFN_ERR), (b"0000:41:00.4", b"0000:41:0A.0", 0),
             (b"0000:41:00.4", b"0000:41:20.0", 0), (b"0000:41:00.4", b"0000:e1:00.0", 0),
             (b"0000:81:00.0", b"0000:81:00.0", 0), (b"0000:41:00.4", b"0000:81:00.0", 0),
             (b"0000:41:00.4", b"0000:41:00.0abcd", 0), (b"0000:41:00.5", b"0000:c1:00.0", 0)]
    got = check_join(kx, PC.walk(WALK), *PC.mdevs(pairs))
    assert got.tolist() == [0, NO_PF, NO_PF, NO_PF, NO_PF, NO_PF, NO_PF, 5, NO_PF, 3]
    assert check_join(kx, PC.walk([]), *PC.mdevs(pairs[:3])).tolist() == [NO_PF] * 3
    assert check_join(kx, PC.walk(WALK), *PC.mdevs([])).tolist() == []


@pytest.mark.parametrize("n_recs,n_pfs,n_mdevs", [(1 << 10, 1 << 5, 1 << 10), (1 << 16, 1 << 11, 1 << 16),
                                                  (1 << 20, 1 << 15, 1 << 20), (1 << 12, 1 << 7, 1 << 18),
                                                  (1 << 18, 1 << 13, 1 << 8)])
def test_join_walks(kx, n_recs, n_pfs, n_mdevs):
    recs, m, s, want = W.mdev_pf_walk(n_recs, n_pfs, n_mdevs, seed=n_mdevs)
    got = check_join(kx, recs, m, s)
    assert np.array_equal(got, want)


def test_join_duplicates_take_the_lowest(kx):
    n = 1 << 16
    recs = PC.walk([b"0000:41:00.0"] * n)  # every record the same address: one slot, the lowest index wins
    m, s = PC.mdevs([(b"0000:41:00.%d" % (1 + k % 7), b"0000:41:00.0", 0) for k in range(4096)])
    assert (check_join(kx, recs, m, s) == 0).all()


def _join_raw(kx, recs, n, mrecs, msrs, m, pf_of, ctx=True):
    return kx.L.kxpu_mdev_pf(kx.ctx if ctx else None, recs, n, mrecs, msrs, m, pf_of)


def test_join_refusals_leave_the_output(kx):
    recs = PC.walk(WALK)
    m, s = PC.mdevs([(b"0000:41:00.4", b"0000:41:00.0", 0)] * 4)
    out = np.full(4, 0xABCD, np.uint32)
    r, mp, sp, op = recs.ctypes.data, m.ctypes.data, s.ctypes.data, out.ctypes.data
    for args, rc in [((r, 6, mp, sp, 4, op, False), -1), ((None, 6, mp, sp, 4, op), -1), ((r, 6, None, sp, 4, op), -1),
                     ((r, 6, mp, None, 4, op), -1), ((r, 6, mp, sp, 4, None), -1),
                     ((r, 1 << 30, mp, sp, 4, op), -7), ((r, 6, mp, sp, 1 << 30, op), -7)]:
        assert _join_raw(kx, *args) == rc, args
        assert (out == 0xABCD).all()
    assert _join_raw(kx, None, 0, mp, sp, 4, op) == 0 and (out == NO_PF).all()  # no PCI records: nothing resolves
    assert _join_raw(kx, r, 6, None, None, 0, None) == 0


# ---------------------------------------------------------------- kxpu_dra_slices_mdev_pf

def raw(kx, devs, out=None, cap=0, offs=None, taints=(), since=None, driver="d", pool="p", node="n", gen=1):
    devs = np.ascontiguousarray(devs)
    enc = lambda x: None if x is None else x.encode()  # noqa: E731
    tab = (DraTaint * max(len(taints), 1))(*[DraTaint(enc(k), enc(v), enc(e)) for k, v, e in taints])
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    rc = kx.L.kxpu_dra_slices_mdev_pf(kx.ctx, driver.encode(), pool.encode(), node.encode(), gen,
                                      devs.ctypes.data if len(devs) else None, len(devs), C.cast(tab, C.c_void_p),
                                      len(taints), None if since is None else since.ctypes.data,
                                      None if out is None else out.ctypes.data, cap, C.byref(ln),
                                      None if offs is None else offs.ctypes.data, C.byref(ns))
    return rc, ln.value, ns.value


def check(kx, devs, taints=(), since=None, driver="vgpu.nvidia.com", pool="node-a", node="node-a", gen=1):
    blob, offs = kx.dra_slices_mdev_pf(driver, pool, node, gen, devs, list(taints), since)
    want, woffs = MO.dra_slices_mdev_pf(driver, pool, node, gen, devs, taints, since)
    assert blob == want
    assert np.array_equal(offs, woffs)
    return blob, offs


def test_golden_cfg1(kx):
    blob, offs = check(kx, PC.cfg1())
    assert blob == open(GOLDEN, "rb").read()


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 127, 128, 129, 1000, 1 << 16, 1 << 20])
def test_sizes_untainted(kx, n):
    devs = PC.random_devs(n, seed=n)
    check(kx, devs)


@pytest.mark.parametrize("table", [PC.TAINTS1, PC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("n", [0, 1, 64, 65, 129, 4097, 1 << 20])
def test_sizes_tainted(kx, table, n):
    devs = PC.random_devs(n, seed=100 + n)
    check(kx, devs, table, since_for(table, n, "some"))


@pytest.mark.parametrize("per", [64, 128])
def test_every_attribute_at_the_seams(kx, per):
    n = 3 * per + 2
    devs = PC.random_devs(n, seed=per, all_attrs=True)
    for i in range(n):
        k, d = i % 32, devs[i]["dev"]
        if k & 1: d["numa_mask"] = 0
        if k & 2: d["device"] = b""
        if k & 4: d["product_len"] = 0
        if k & 8: d["pcie_root"] = b""
        if k & 16: devs[i]["physfn"], devs[i]["physfn_device"] = b"", b""
        elif k & 1: devs[i]["physfn_device"] = b""
    if per == 64:
        check(kx, devs, PC.TAINTS1, np.where(np.arange(n)[:, None] % 3 == 0, 5, -1))
    else:
        check(kx, devs)


@pytest.mark.parametrize("table", [None, PC.TAINTS1, PC.TAINTS3], ids=["null", "1", "3"])
@pytest.mark.parametrize("n", [0, 1, 64, 129, 1 << 20])
def test_empty_physfn_is_mdev_taints(kx, table, n):
    """every physfn empty: kxpu_dra_slices_mdev_taints' bytes and slice_off, byte for byte"""
    devs = PC.random_devs(n, seed=7 + n, no_physfn=True)
    taints = table or PC.TAINTS3
    since = None if table is None else since_for(table, n, "some", seed=n)
    blob, offs = kx.dra_slices_mdev_pf("vgpu.nvidia.com", "node-a", "node-a", 4, devs, list(taints), since)
    want, woffs = kx.dra_slices_mdev_taints("vgpu.nvidia.com", "node-a", "node-a", 4, devs["dev"], list(taints), since)
    assert blob == want and np.array_equal(offs, woffs)


def _untouched(kx, devs, rc_want, **kw):
    out = np.full(1 << 16, 0x5A, np.uint8)
    offs = np.full(8, 0x77, np.uint64)
    rc, ln, ns = raw(kx, devs, out, out.size, offs, **kw)
    assert rc == rc_want, kw
    assert (out == 0x5A).all() and (offs == 0x77).all() and ln == 0xDEAD and ns == 0xDEAD


@pytest.mark.parametrize("why,field,value", PC.BAD + MC.BAD)
def test_domain_refusals(kx, why, field, value):
    if field in ("physfn", "physfn_device"):
        bad = PC.bad_rec(field, value)
    else:
        bad = PC.rec(physfn=b"0000:41:00.0")
        bad["dev"] = MC.bad_rec(field, value)
    devs = np.concatenate([PC.cfg1(), bad])
    assert MO.dra_slices_mdev_pf("d", "p", "n", 1, devs) == (-7, why)
    _untouched(kx, devs, -7)
    _untouched(kx, devs, -7, taints=PC.TAINTS1, since=np.full((3, 1), -1, np.int64))


def test_other_refusals(kx):
    devs = PC.cfg1()
    _untouched(kx, PC.bad_rec("physfn_device", b"2330", physfn=b""), -7)
    _untouched(kx, devs, -7, taints=PC.TAINTS3, since=np.array([[-1, -1, -1], [TC.SINCE_MAX + 1, -1, -1]]))
    _untouched(kx, devs, -7, taints=PC.TAINTS3, since=np.array([[-1, 5, 6], [-1, -1, -1]]))
    for kw in [dict(driver="D"), dict(driver="d" * 64), dict(pool="p."), dict(node=""), dict(gen=1 << 63)]:
        _untouched(kx, devs, -1, **kw)
    for key, value, effect in TC.INVALID:
        _untouched(kx, devs, -1, taints=[(key, value, effect)], since=np.zeros((2, 1), np.int64))
    five = [("k%d" % t, "", "NoSchedule") for t in range(5)]
    _untouched(kx, devs, -1, taints=five, since=np.zeros((2, 5), np.int64))
    rc = kx.L.kxpu_dra_slices_mdev_pf(kx.ctx, b"d", b"p", b"n", 1, devs.ctypes.data, 1 << 24, None, 0, None, None, 0,
                                      C.byref(C.c_size_t()), None, C.byref(C.c_size_t()))
    assert rc == -7
    rc = kx.L.kxpu_dra_slices_mdev_pf(kx.ctx, b"d", b"p", b"n", 1, None, 2, None, 0, None, None, 0,
                                      C.byref(C.c_size_t()), None, C.byref(C.c_size_t()))
    assert rc == -1


def test_sizing(kx):
    devs = PC.random_devs(300, seed=3)
    rc, ln, ns = raw(kx, devs)
    assert rc == -4 and ns == 3
    out, offs = np.zeros(ln, np.uint8), np.zeros(ns + 1, np.uint64)
    rc, ln2, ns2 = raw(kx, devs, out, ln - 1, offs)
    assert rc == -4 and ln2 == ln
    rc, _, _ = raw(kx, devs, out, ln, offs)
    assert rc == 0 and out.tobytes() == MO.dra_slices_mdev_pf("d", "p", "n", 1, devs)[0]
