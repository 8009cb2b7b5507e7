"""GPU tests of kxpu_dra_slices_pf: bytes and slice_off against the C oracle (tests/dra_pf_oracle.c) from 0 to 2^20
devices, at the slice seams (127 / 128 / 129 untainted, 63 / 64 / 65 tainted), with taint tables of one and three
entries, mixed VF and non-VF records and 16-byte physfn values; a pool whose every physfn is empty against
kxpu_dra_slices_taints byte for byte; every KXPU_E_INVALID and KXPU_E_UNSUPPORTED case with the outputs untouched."""
import ctypes as C
import os

import numpy as np
import pytest

import dra_cases as DC
import dra_pf_cases as PC
import dra_pf_oracle as PO
import dra_taint_cases as TC
from kxpu_b200.binding import DraTaint

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_pf_cfg1.jsonl")


def since_for(table, n, kind, seed=0):
    since = np.stack([TC.since_pattern(n, kind, seed=seed + t) for t in range(len(table))], axis=1) if n else \
        np.zeros((0, len(table)), np.int64)
    if len(table) == 3:
        since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    return since


def raw(kx, devs, out=None, cap=0, offs=None, taints=(), since=None, driver="d", pool="p", node="n", gen=1):
    devs = np.ascontiguousarray(devs)
    enc = lambda x: None if x is None else x.encode()  # noqa: E731
    tab = (DraTaint * max(len(taints), 1))(*[DraTaint(enc(k), enc(v), enc(e)) for k, v, e in taints])
    if since is not None:
        since = np.ascontiguousarray(since, dtype=np.int64)
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    rc = kx.L.kxpu_dra_slices_pf(kx.ctx, driver.encode(), pool.encode(), node.encode(), gen,
                                 devs.ctypes.data if len(devs) else None, len(devs), C.cast(tab, C.c_void_p),
                                 len(taints), None if since is None else since.ctypes.data,
                                 None if out is None else out.ctypes.data, cap, C.byref(ln),
                                 None if offs is None else offs.ctypes.data, C.byref(ns))
    return rc, ln.value, ns.value


def check(kx, devs, taints=(), since=None, driver="vfio.example.com", pool="node-a", node="node-a", gen=1):
    blob, offs = kx.dra_slices_pf(driver, pool, node, gen, devs, list(taints), since)
    want, woffs = PO.dra_slices_pf(driver, pool, node, gen, devs, taints, since)
    assert blob == want
    assert np.array_equal(offs, woffs)
    return blob, offs


def test_golden_cfg1(kx):
    c = PC.CFG1
    blob, offs = check(kx, PC.cfg1(), driver=c["driver"], pool=c["pool"], node=c["node"], gen=c["gen"])
    assert blob == open(GOLDEN, "rb").read()


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 127, 128, 129, 1000, 1 << 16, 1 << 20])
def test_sizes_untainted(kx, n):
    check(kx, PC.random_devs(n, seed=n))


@pytest.mark.parametrize("table", [PC.TAINTS1, PC.TAINTS3], ids=["1", "3"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129, 4097, 1 << 20])
def test_sizes_tainted(kx, table, n):
    check(kx, PC.random_devs(n, seed=100 + n), table, since_for(table, n, "some"))


@pytest.mark.parametrize("n", [127, 128, 129, 1 << 20])
def test_one_vf_in_eight(kx, n):
    """the measured pool: canonical VFs among whole GPUs, untainted and with three taints"""
    devs = PC.random_devs(n, seed=n, vf_every=8)
    check(kx, devs)
    check(kx, devs, PC.TAINTS3, since_for(PC.TAINTS3, n, "some", seed=1))


@pytest.mark.parametrize("per", [64, 128])
def test_every_attribute_at_the_seams(kx, per):
    n = 3 * per + 2
    devs = PC.random_devs(n, seed=per, all_attrs=True)
    for i in range(n):
        k, d = i % 16, devs[i]["dev"]
        if k & 1: d["numa_mask"] = 0
        if k & 2: d["product_len"] = 0
        if k & 4: d["pcie_root"] = b""
        if k & 8: devs[i]["physfn"], devs[i]["physfn_device"] = b"", b""
        elif k & 1: devs[i]["physfn_device"] = b""
    blob = check(kx, devs, PC.TAINTS1, np.where(np.arange(n)[:, None] % 3 == 0, 5, -1)) if per == 64 else check(kx, devs)
    assert blob[0].count(b'"physfnAddress":{"string":"') == sum(1 for i in range(n) if not i % 16 & 8)


def test_sixteen_byte_physfn(kx):
    """a physfn that fills its field (no NUL) and a 6-byte id, on every device of a tainted and an untainted pool"""
    devs = PC.random_devs(300, seed=11, all_attrs=True)
    assert all(len(bytes(x)) == 16 for x in devs["physfn"])
    check(kx, devs)
    check(kx, devs, PC.TAINTS3, since_for(PC.TAINTS3, 300, "all", seed=2))


@pytest.mark.parametrize("table", [None, PC.TAINTS1, PC.TAINTS3], ids=["null", "1", "3"])
@pytest.mark.parametrize("n", [0, 1, 3, 64, 129, 1 << 20])
def test_empty_physfn_is_taints(kx, table, n):
    """every physfn empty: kxpu_dra_slices_taints' bytes and slice_off, byte for byte"""
    devs = PC.random_devs(n, seed=7 + n, no_physfn=True)
    taints = table or PC.TAINTS3
    since = None if table is None else since_for(table, n, "some", seed=n)
    blob, offs = kx.dra_slices_pf("vfio.example.com", "node-a", "node-a", 4, devs, list(taints), since)
    want, woffs = kx.dra_slices_taints("vfio.example.com", "node-a", "node-a", 4, devs["dev"], list(taints), since)
    assert blob == want and np.array_equal(offs, woffs)


def _untouched(kx, devs, rc_want, **kw):
    out = np.full(1 << 16, 0x5A, np.uint8)
    offs = np.full(8, 0x77, np.uint64)
    rc, ln, ns = raw(kx, devs, out, out.size, offs, **kw)
    assert rc == rc_want, kw
    assert (out == 0x5A).all() and (offs == 0x77).all() and ln == 0xDEAD and ns == 0xDEAD


@pytest.mark.parametrize("why,field,value", PC.BAD + DC.BAD)
def test_domain_refusals(kx, why, field, value):
    if field in ("physfn", "physfn_device"):
        bad = PC.bad_rec(field, value)
    else:
        bad = PC.rec(physfn=b"0000:4d:00.0")
        bad["dev"] = DC.bad_rec(field, value)
    devs = np.concatenate([PC.cfg1(), bad])
    assert PO.dra_slices_pf("d", "p", "n", 1, devs) == (-7, why)
    _untouched(kx, devs, -7)
    _untouched(kx, devs, -7, taints=PC.TAINTS1, since=np.full((3, 1), -1, np.int64))
    _untouched(kx, devs, -7, taints=PC.TAINTS3, since=np.full((3, 3), -1, np.int64))


def test_other_refusals(kx):
    devs = PC.cfg1()
    _untouched(kx, PC.bad_rec("physfn_device", b"56c0", physfn=b""), -7)
    _untouched(kx, devs, -7, taints=PC.TAINTS3, since=np.array([[-1, -1, -1], [TC.SINCE_MAX + 1, -1, -1]]))
    _untouched(kx, devs, -7, taints=PC.TAINTS3, since=np.array([[-1, 5, 6], [-1, -1, -1]]))
    for kw in [dict(driver="D"), dict(driver="d" * 64), dict(pool="p."), dict(node=""), dict(gen=1 << 63)]:
        _untouched(kx, devs, -1, **kw)
    for key, value, effect in TC.INVALID:
        _untouched(kx, devs, -1, taints=[(key, value, effect)], since=np.zeros((2, 1), np.int64))
    five = [("k%d" % t, "", "NoSchedule") for t in range(5)]
    _untouched(kx, devs, -1, taints=five, since=np.zeros((2, 5), np.int64))
    rc = kx.L.kxpu_dra_slices_pf(kx.ctx, b"d", b"p", b"n", 1, devs.ctypes.data, 1 << 24, None, 0, None, None, 0,
                                 C.byref(C.c_size_t()), None, C.byref(C.c_size_t()))
    assert rc == -7
    rc = kx.L.kxpu_dra_slices_pf(kx.ctx, b"d", b"p", b"n", 1, None, 2, None, 0, None, None, 0,
                                 C.byref(C.c_size_t()), None, C.byref(C.c_size_t()))
    assert rc == -1
    rc = kx.L.kxpu_dra_slices_pf(None, b"d", b"p", b"n", 1, devs.ctypes.data, 2, None, 0, None, None, 0,
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
    assert rc == 0 and out.tobytes() == PO.dra_slices_pf("d", "p", "n", 1, devs)[0]
