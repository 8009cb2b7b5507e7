"""GPU tests of kxpu_dra_slices_taint / kxpu_dra_slices_mdev_taint (include/kxpu.h, ABI v11): bytes and slice_off
against the CPU oracle (oracle/kxpu_dra_taint_oracle.c) for both layouts around the 64-device slice edges and in large
pools, mixed and all-tainted pools with the longest names, key and value, the timestamp edges, refusals that leave the
output untouched, the two-call sizing, every output alignment, taint_since == NULL against the v9 / v10 kernels, and
calls interleaved with kxpu_dra_slices and the CDI emitter on one context, also with the look-back epoch wrapping."""
import ctypes as C

import numpy as np
import pytest

import dra_cases as DC
import dra_mdev_cases as MC
import dra_taint_cases as TC
from oracle import dra_oracle as DO
from oracle import dra_taint_oracle as TO
from oracle import xpu_oracle as XO

pytestmark = pytest.mark.gpu

LONG_DRIVER = "d" * 63
LONG_NAME = ".".join(["a" * 63] * 3 + ["b" * 61])
LAYOUTS = {"pci": (DC, "dra_slices_taint", TO.dra_slices_taint, "dra_slices", "kxpu_dra_slices_taint"),
           "mdev": (MC, "dra_slices_mdev_taint", TO.dra_slices_mdev_taint, "dra_slices_mdev", "kxpu_dra_slices_mdev_taint")}


def raw(kx, layout, driver, pool, node, gen, devs, key, value, effect, since, out=None, cap=0, offs=None):
    """one bare call: (status, len, n_slices); len / n_slices keep the sentinel 0xDEAD when not written"""
    devs = np.ascontiguousarray(devs)
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    b = lambda s: s.encode() if isinstance(s, str) else s
    fn = getattr(kx.L, LAYOUTS[layout][4])
    rc = fn(kx.ctx, driver.encode(), pool.encode(), node.encode(), gen, devs.ctypes.data if len(devs) else None, len(devs),
            b(key), b(value), b(effect), None if since is None else since.ctypes.data,
            None if out is None else out.ctypes.data, cap, C.byref(ln), None if offs is None else offs.ctypes.data,
            C.byref(ns))
    return rc, ln.value, ns.value


def devices(layout, n, seed, all_attrs=False):
    return LAYOUTS[layout][0].random_devs(n, seed=seed, all_attrs=all_attrs)


def check(kx, layout, devs, since, driver="vfio.nvidia.com", pool="node-a", node="node-a", gen=1, key=TC.KEY,
          value=TC.VALUE, effect="NoSchedule"):
    """the kernel == the oracle, bytes and slice_off"""
    blob, offs = getattr(kx, LAYOUTS[layout][1])(driver, pool, node, gen, devs, key, value, effect, since)
    want, woffs = LAYOUTS[layout][2](driver, pool, node, gen, devs, key, value, effect, since)
    assert blob == want
    assert np.array_equal(offs, woffs)
    return blob, offs


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 127, 128, 129, 4097, 65536, 1 << 20])
def test_sizes_mixed(kx, layout, n):
    check(kx, layout, devices(layout, n, seed=2000 + n), TC.since_pattern(n, "some", seed=n))


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("kind", ["none", "all"])
@pytest.mark.parametrize("n", [64, 129, 65536])
def test_none_and_all_tainted_longest(kx, layout, kind, n):
    check(kx, layout, devices(layout, n, seed=7, all_attrs=True), TC.since_pattern(n, kind, seed=n), LONG_DRIVER, LONG_NAME,
          LONG_NAME, (1 << 63) - 1, TC.LONG_KEY, TC.LONG_VALUE)


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("value,effect", [("", "NoExecute"), (TC.LONG_VALUE, "NoSchedule")])
def test_timestamp_edges(kx, layout, value, effect):
    since = TC.since_pattern(200, "edges")
    blob, _ = check(kx, layout, devices(layout, 200, seed=9), since, key=TC.LONG_KEY, value=value, effect=effect)
    for t, s in TC.EDGES.items():
        assert ('"timeAdded":"%s"' % s).encode() in blob


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("n", [0, 1, 129, 65536])
def test_null_since_equals_untainted_kernel(kx, layout, n):
    devs = devices(layout, n, seed=3000 + n)
    want = getattr(kx, LAYOUTS[layout][3])("d", "p", "n", 6, devs)
    for key, value, effect in [(TC.KEY, TC.VALUE, "NoSchedule"), (None, None, None)]:
        got = getattr(kx, LAYOUTS[layout][1])("d", "p", "n", 6, devs, key, value, effect, None)
        assert got[0] == want[0] and np.array_equal(got[1], want[1])


def _untouched(kx, layout, devs, since, expect, driver="d", key=TC.KEY, value=TC.VALUE, effect="NoSchedule"):
    out = np.full(1 << 17, 0xAB, np.uint8)
    offs = np.full(8, 0xABAB, np.uint64)
    assert raw(kx, layout, driver, "p", "n", 1, devs, key, value, effect, since, out, out.size, offs) == \
        (expect, 0xDEAD, 0xDEAD)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_invalid_arguments_write_nothing(kx, layout):
    devs, since = devices(layout, 100, seed=4), TC.since_pattern(100, "all", seed=4)
    for key, value, effect in TC.INVALID:
        assert TO.dra_slices_taint("d", "p", "n", 1, DC.random_devs(1, seed=1), key, value, effect, since[:1]) == -1
        _untouched(kx, layout, devs, since, -1, key=key, value=value, effect=effect)
    _untouched(kx, layout, devs, since, -1, driver="Vfio")


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("t", [TC.SINCE_MAX + 1, (1 << 63) - 1])
def test_out_of_domain_writes_nothing(kx, layout, t):
    devs, since = devices(layout, 200, seed=5), TC.since_pattern(200, "some", seed=5)
    since[170] = t
    _untouched(kx, layout, devs, since, -7)
    cases = LAYOUTS[layout][0]
    why, field, value = cases.BAD[0]
    bad = np.concatenate([devs[:60], cases.bad_rec(field, value), devs[60:]])
    _untouched(kx, layout, bad, TC.since_pattern(201, "all", seed=6), -7)


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_sizing_exact_and_short(kx, layout):
    devs, since = devices(layout, 300, seed=11), TC.since_pattern(300, "some", seed=11)
    args = ("d", "p", "n", 5, devs, TC.KEY, TC.VALUE, "NoExecute", since)
    want, woffs = LAYOUTS[layout][2](*args)
    assert raw(kx, layout, *args) == (-4, len(want), 5)
    out = np.full(len(want) + 16, 0xAB, np.uint8)
    offs = np.full(5 + 2, 0xABAB, np.uint64)
    assert raw(kx, layout, *args, out, len(want) - 1, offs) == (-4, len(want), 5)
    assert (out == 0xAB).all() and (offs == 0xABAB).all()
    assert raw(kx, layout, *args, out, len(want), offs) == (0, len(want), 5)
    assert out[:len(want)].tobytes() == want and (out[len(want):] == 0xAB).all()
    assert np.array_equal(offs[:6], woffs) and offs[6] == 0xABAB
    assert raw(kx, layout, *args, out, len(want), None) == (0, len(want), 5)  # slice_off may be NULL


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_output_pointer_every_phase(kx, layout):
    devs, since = devices(layout, 129, seed=12), TC.since_pattern(129, "some", seed=12)
    args = ("d", "p", "n", 1, devs, TC.LONG_KEY, TC.LONG_VALUE, "NoSchedule", since)
    want, _ = LAYOUTS[layout][2](*args)
    buf = np.full(len(want) + 64, 0xAB, np.uint8)
    base = (16 - buf.ctypes.data % 16) % 16
    for ph in range(16):
        buf[:] = 0xAB
        view = buf[base + ph:base + ph + len(want)]
        assert raw(kx, layout, *args, view, len(want))[0] == 0
        assert view.tobytes() == want
        assert (buf[:base + ph] == 0xAB).all() and (buf[base + ph + len(want):] == 0xAB).all()


def _interleave(kx):
    kind = b"vfio.example.com/xpu"
    cdi = np.zeros(5000, XO.CDIDEV_DTYPE)
    cdi["bdf"], cdi["iommu_group"], cdi["index"] = b"0000:c1:00.0", np.arange(5000), np.arange(5000)
    for r in range(12):
        n = [0, 129, 4097, 300, 65536, 1][r % 6]
        layout = ["pci", "mdev"][r % 2]
        check(kx, layout, devices(layout, n, seed=r), TC.since_pattern(n, ["some", "all", "none"][r % 3], seed=r), gen=r + 1)
        pci = DC.random_devs(n, seed=100 + r)
        blob, offs = kx.dra_slices("d", "p", "n", r + 1, pci)
        want, woffs = DO.dra_slices("d", "p", "n", r + 1, pci)
        assert blob == want and np.array_equal(offs, woffs)
        assert kx.cdi_emit(1, cdi[:4000 + 100 * r], kind) == XO.cdi_emit_kind(1, kind, cdi[:4000 + 100 * r])


def test_interleaved_with_untainted_and_cdi_emit(kx):
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
