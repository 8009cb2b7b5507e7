"""GPU tests of kxpu_reset_check: bitwise equal to the C checker and the Python restatement on the hand-worked forests,
every reset_method text under every allow-list, a seeded fuzz and a 2^20-record walk; chains of KXPU_PCIE_MAX_DEPTH keys,
thousands of functions under one bridge and one bridge shared by many groups; every refusal, with the outputs left
untouched."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import pyref_reset as P
import reset_cases as RC
import reset_oracle as RO
from kxpu_b200.binding import E_INVALID, E_UNSUPPORTED, KxpuError, rules_array

pytestmark = pytest.mark.gpu


def _check(kx, recs, paths, rrs, allow=RC.ALL, rules=RC.NV, pyref=None):
    c = kx.classify_rules(rules, recs)
    got = kx.reset_check(rules, recs, paths, rrs, allow, c["group_off"], c["group_members"])
    got = {k: v.tolist() for k, v in got.items()}
    want = RO.reset_check(rules, recs, paths, rrs, allow, c["group_off"], c["group_members"])
    assert got == want
    if pyref if pyref is not None else len(recs) <= 4096:  # the Python restatement is too slow for the big walks
        assert want == P.reset_check(rules, recs, paths, rrs, allow, c["group_off"], c["group_members"])
    return c, got


@pytest.mark.parametrize("name", sorted(RC.HAND))
def test_hand_forests(kx, name):
    (recs, paths, rrs), allow, methods, verdict, groups = RC.HAND[name]
    c, got = _check(kx, recs, paths, rrs, allow)
    assert got["methods"] == methods and got["set_verdict"] == verdict
    assert dict(zip(c["group_ids"].tolist(), got["group_reset"])) == groups


@pytest.mark.parametrize("allow", RC.ALLOWS)
def test_reset_method_texts(kx, allow):
    rows = [RC.fn(b"0000:00:%02x.%d" % (k // 8, k % 8), k, ["pci0000:00"], method=t, rflags=f)
            for k, (t, f, _) in enumerate(RC.TEXTS)]
    _, got = _check(kx, *RC.walk(*rows), allow=allow)
    assert got["methods"] == [m for _, _, m in RC.TEXTS]


@settings(max_examples=200, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(RC.reset_walks(), st.sampled_from(RC.ALLOWS))
def test_fuzz(kx, w, allow):
    _check(kx, *w, allow=allow)
    _check(kx, *w, allow=allow, rules=[(b"10de", b"vfio-pci"), (b"1002", b"nvme")])


def test_big_walk(kx, workloads):
    recs, paths, rrs = workloads.reset_walk(1 << 20)
    c, got = _check(kx, recs, paths, rrs)
    assert c["n_groups"] == 1 << 20
    blocked = sum(g != RC.VIABLE for g in got["group_reset"])
    assert (1 << 20) // 20 < blocked < (1 << 20) // 5  # the functions with no method: a down port holds 8 groups
    _, narrow = _check(kx, recs, paths, rrs, allow=RC.FLR | RC.BUS)
    assert sum(g != RC.VIABLE for g in narrow["group_reset"]) > blocked


def _chain(depth):
    """a host bridge and depth - 1 bridges: a chain of depth keys"""
    return ["pci0000:00"] + ["0000:%02x:00.0" % k for k in range(depth - 1)]


def test_chains_at_the_depth_limit(kx):
    deep, over = _chain(8), _chain(9)
    recs, paths, rrs = RC.walk(RC.fn(b"0000:20:00.0", 1, deep), RC.fn(b"0000:20:00.1", 1, deep),
                               RC.fn(b"0000:20:00.2", 2, over),               # 9 keys: unknown
                               RC.fn(deep[-1].encode(), 3, deep[:-1], driver=b"pcieport", vendor=b"0x8086\n"))
    _, got = _check(kx, recs, paths, rrs)
    # the deep pair's own bridge is in the walk: it is not in the set of its secondary bus, but blocks the set above it
    assert got["set_verdict"] == [RC.SET_OK, RC.SET_OK, RC.NO_PATH, 3]
    assert got["group_reset"] == [RC.VIABLE, 2]


@pytest.mark.parametrize("n", [4096, 40000])
def test_thousands_under_one_bridge(kx, n):
    port = ["pci0000:00", "0000:00:01.0"]
    rows = [RC.fn(b"0000:%02x:%02x.%d" % (2 + k // 256, (k >> 3) & 31, k & 7), 9,
                  port + ["0000:01:%02x.%d" % ((k // 256) >> 3, (k // 256) & 7)]) for k in range(n)]
    recs, paths, rrs = RC.walk(*rows)
    _, got = _check(kx, recs, paths, rrs, pyref=False)
    assert set(got["set_verdict"]) == {RC.SET_OK} and got["group_reset"] == [RC.VIABLE]
    # one function far below the shared bridge on a host driver names itself for every function above it
    recs["driver"][n - 5] = b"nvme"
    _, got = _check(kx, recs, paths, rrs, pyref=False)
    shared = [i for i in range(n) if (2 + i // 256) == (2 + (n - 5) // 256)]
    assert all(got["set_verdict"][i] == n - 5 for i in shared) and got["group_reset"] == [min(shared)]


def test_bridge_shared_by_many_groups(kx):
    port = ["pci0000:00", "0000:00:01.0"]
    n = 3000
    rows = [RC.fn(b"0000:%02x:%02x.%d" % (1 + k // 256, (k >> 3) & 31, k & 7), 100 + (k * 7919) % 1000, port)
            for k in range(n)]
    recs, paths, rrs = RC.walk(*rows)
    _, got = _check(kx, recs, paths, rrs, pyref=False)
    groups = recs["iommu_group"].astype(np.int64)
    lo_first, hi_first = int(np.argmax(groups == groups.min())), int(np.argmax(groups == groups.max()))
    want = [hi_first if groups[i] == groups.min() else lo_first for i in range(n)]
    assert got["set_verdict"] == want and RC.VIABLE not in got["group_reset"]


def test_refusals(kx):
    (recs, paths, rrs), *_ = RC.HAND["three_groups_under_one_port"]
    c = kx.classify_rules(RC.NV, recs)
    off, mem = c["group_off"], c["group_members"]
    for args in ((RC.NV, RC.ALL, np.array([0, 2, 1, 4], np.uint32), mem),
                 (RC.NV, RC.ALL, off, np.array([0, 1, 2, 4], np.uint32)),
                 (RC.NV, RC.ALL | RC.UNNAMED, off, mem),
                 (RC.NV, 0x100, off, mem),
                 ([(b"10de", b"vfio/pci")], RC.ALL, off, mem),
                 ([(b"10de", b"vfio-pci"), (b"10de", b"vfio-pci")], RC.ALL, off, mem),
                 ([], RC.ALL, off, mem)):
        rules, allow, o, m = args
        with pytest.raises(KxpuError) as e:
            kx.reset_check(rules, recs, paths, rrs, allow, o, m)
        assert e.value.status == E_INVALID, args
    empty = kx.reset_check(RC.NV, recs[:0], paths[:0], rrs[:0], RC.ALL, np.zeros(1, np.uint32), mem[:0])
    assert all(len(v) == 0 for v in empty.values())
    # raw calls: nothing written on a refusal, NULLs refused, and n at the limit refused before any array is read
    ra = rules_array(RC.NV)
    n, G = len(recs), len(off) - 1
    meth, sv, gr = np.full(n, 0xAB, np.uint8), np.full(n, 7, np.uint32), np.full(G, 7, np.uint32)

    def raw(n_=n, recs_=recs.ctypes.data, paths_=paths.ctypes.data, rrs_=rrs.ctypes.data, off_=off, allow=RC.ALL,
            gr_=gr.ctypes.data):
        return kx.L.kxpu_reset_check(kx.ctx, ra.ctypes.data, 1, recs_, paths_, rrs_, n_, allow, off_.ctypes.data,
                                     mem.ctypes.data, G, meth.ctypes.data, sv.ctypes.data, gr_)
    assert raw(off_=np.array([0, 2, 1, 4], np.uint32)) == E_INVALID
    assert raw(allow=0xFF) == E_INVALID
    assert raw(paths_=None) == E_INVALID and raw(rrs_=None) == E_INVALID and raw(recs_=None) == E_INVALID
    assert raw(gr_=None) == E_INVALID
    assert raw(n_=1 << 28) == E_UNSUPPORTED
    bad_mem = np.array([0, 1, 2, 9], np.uint32)
    assert kx.L.kxpu_reset_check(kx.ctx, ra.ctypes.data, 1, recs.ctypes.data, paths.ctypes.data, rrs.ctypes.data, n,
                                 RC.ALL, off.ctypes.data, bad_mem.ctypes.data, G, meth.ctypes.data, sv.ctypes.data,
                                 gr.ctypes.data) == E_INVALID
    assert (meth == 0xAB).all() and (sv == 7).all() and (gr == 7).all()
    assert raw() == 0 and gr.tolist() == [0, 1, 2]
