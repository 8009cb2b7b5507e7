"""GPU tests of kxpu_aer_health and kxpu_dra_slices_taints / kxpu_dra_slices_mdev_taints (include/kxpu.h, ABI v12)
against the CPU oracle (oracle/kxpu_aer_oracle.c): every file case at unaligned and shared offsets, TOTAL lines at every
window phase, large seeded walks with vGPUs sharing their parent's files, limits, refusals that leave the outputs
untouched; taint lists of one to four entries at the longest key and value around the 64-device slice edges and in large
pools, and the two identities: taint_since == NULL gives kxpu_dra_slices[_mdev]'s bytes, one entry the _taint call's."""
import ctypes as C

import numpy as np
import pytest

import aer_cases as AC
import dra_cases as DC
import dra_mdev_cases as MC
import dra_taint_cases as TC
from kxpu_b200 import workloads as W
from kxpu_b200.binding import DraTaint
from oracle import aer_oracle as AO

pytestmark = pytest.mark.gpu

MAX = (1 << 64) - 1


def check_aer(kx, text, off, ln, fl, nl, goff, mem):
    got = kx.aer_health(text, off, ln, fl, nl, goff, mem)
    want = AO.aer_health(text, off, ln, fl, nl, goff, mem)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    return got


@pytest.mark.parametrize("gap", [0, 1, 3, 17])
def test_file_cases(kx, gap):
    fc, nc = AC.cases(AC.F), AC.cases(AC.N)
    files = [(a[1], b[1]) for a, b in zip(fc, nc)] + [(a[1], nc[0][1]) for a in fc] + [(fc[0][1], b[1]) for b in nc]
    n = len(files)
    # each record alone, then every record once more through shared files (as vGPUs read their parent's)
    share = list(range(n)) + list(range(n - 1, -1, -1))
    text, off, ln = AC.pack(files, gaps=[gap + (k % 7) for k in range(2 * n)], share=share)
    goff = np.arange(2 * n + 1, dtype=np.uint32)
    totals, _ = check_aer(kx, text, off, ln, 0, 0, goff, np.arange(2 * n, dtype=np.uint32))
    for i, (a, b) in enumerate(zip(fc, nc)):
        assert int(totals[2 * i]) == a[2] and int(totals[2 * i + 1]) == b[2], (a[0], b[0])


@pytest.mark.parametrize("fl,nl", [(0, 0), (1, 5), (MAX - 1, 0), (MAX, MAX)])
@pytest.mark.parametrize("n,share", [(1, 0), (4097, 0), (65536, 0), (65536, 16), (1 << 20, 16)])
def test_walks(kx, n, share, fl, nl):
    r = W.aer_records(n, seed=n + share, vgpus_per_parent=share)
    totals, aer = check_aer(kx, r["text"], r["file_off"], r["file_len"], fl, nl, r["group_off"], r["group_members"])
    if (fl, nl) == (0, 0) and n > 1000 and share == 0:  # about one function in 64 has errors
        assert 0 < int(((aer & 3) != 0).sum()) < len(aer) // 8


def test_groups_large_and_empty(kx):
    r = W.aer_records(3000, seed=5)
    n = 3000
    # one group of every record, empty groups around it, and groups that repeat members
    goff = np.array([0, 0, n, n, n + 40, n + 40], np.uint32)
    mem = np.concatenate([np.arange(n), np.full(40, 7)]).astype(np.uint32)
    check_aer(kx, r["text"], r["file_off"], r["file_len"], 0, 0, goff, mem)
    check_aer(kx, b"", np.zeros(0, np.uint64), np.zeros(0, np.uint32), 0, 0, np.zeros(3, np.uint32), np.zeros(0, np.uint32))


def raw_aer(kx, text, off, ln, goff, mem, totals, aer):
    t = np.frombuffer(text, np.uint8)
    return kx.L.kxpu_aer_health(kx.ctx, t.ctypes.data if len(t) else None, len(t), off.ctypes.data, ln.ctypes.data,
                                len(off) // 2, 0, 0, goff.ctypes.data, mem.ctypes.data if len(mem) else None,
                                len(goff) - 1, totals.ctypes.data, aer.ctypes.data)


def test_refusals_leave_outputs(kx):
    text, off, ln = AC.pack([(AC.aer_file(AC.F, [1] * 18), AC.aer_file(AC.N, [0] * 18))] * 3)
    g, m = np.array([0, 2, 3], np.uint32), np.array([0, 1, 2], np.uint32)
    cases = []
    bad = off.copy(); bad[3] = len(text) - ln[3] + 1
    cases.append((bad, ln, g, m))
    bad = off.copy(); bad[0] = MAX
    cases.append((bad, ln, g, m))
    cases.append((off, ln, np.array([0, 2, 1], np.uint32), m))
    cases.append((off, ln, g, np.array([0, 3, 2], np.uint32)))
    for o, l, gg, mm in cases:
        totals, aer = np.full(6, 0xAB, np.uint64), np.full(2, 0xCD, np.uint8)
        assert raw_aer(kx, text, o, l, gg, mm, totals, aer) == -1
        assert (totals == 0xAB).all() and (aer == 0xCD).all()
    totals, aer = np.full(6, 0xAB, np.uint64), np.full(2, 0xCD, np.uint8)
    assert raw_aer(kx, text, off, ln, g, m, totals, aer) == 0
    assert totals.tolist() == [18, 0] * 3 and aer.tolist() == [1, 1]
    n = 1 << 28
    assert kx.L.kxpu_aer_health(kx.ctx, None, 0, off.ctypes.data, ln.ctypes.data, n, 0, 0, g.ctypes.data, m.ctypes.data,
                                2, None, aer.ctypes.data) == -7
    assert kx.L.kxpu_aer_health(kx.ctx, None, 0, None, None, 0, 0, 0, g.ctypes.data, m.ctypes.data, n, None,
                                aer.ctypes.data) == -7


# ---------------------------------------------------------------- the taint lists
LAYOUTS = {"pci": (DC, "dra_slices_taints", AO.dra_slices_taints, "dra_slices", "dra_slices_taint", "kxpu_dra_slices_taints"),
           "mdev": (MC, "dra_slices_mdev_taints", AO.dra_slices_mdev_taints, "dra_slices_mdev", "dra_slices_mdev_taint",
                    "kxpu_dra_slices_mdev_taints")}


def devices(layout, n, seed, all_attrs=False):
    return LAYOUTS[layout][0].random_devs(n, seed=seed, all_attrs=all_attrs)


def check(kx, layout, devs, taints, since, driver="vfio.nvidia.com", pool="node-a", node="node-a", gen=1):
    blob, offs = getattr(kx, LAYOUTS[layout][1])(driver, pool, node, gen, devs, taints, since)
    want, woffs = LAYOUTS[layout][2](driver, pool, node, gen, devs, taints, since)
    assert blob == want
    assert np.array_equal(offs, woffs)
    return blob, offs


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129, 65536])
def test_lists_longest(kx, layout, k, n):
    table = AC.long_table(k)
    check(kx, layout, devices(layout, n, seed=n + k, all_attrs=True), table, AC.since_table(n, k, seed=n, frac=2),
          "d" * 63, ".".join(["a" * 63] * 3 + ["b" * 61]), ".".join(["a" * 63] * 3 + ["b" * 61]), (1 << 63) - 1)


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("frac", [1, 3, 1000])
def test_table3_large(kx, layout, frac):
    n = 1 << 20 if frac == 3 else 65536
    check(kx, layout, devices(layout, n, seed=frac), AC.TABLE3, AC.since_table(n, 3, seed=frac, frac=frac, table=AC.TABLE3))


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("n", [0, 1, 64, 65, 65536])
def test_identities(kx, layout, n):
    devs = devices(layout, n, seed=300 + n)
    mod, name = LAYOUTS[layout][0], LAYOUTS[layout]
    untainted = getattr(kx, name[3])("vfio.nvidia.com", "node-a", "node-a", 4, devs)
    got = getattr(kx, name[1])("vfio.nvidia.com", "node-a", "node-a", 4, devs, AC.TABLE3, None)
    assert got[0] == untainted[0] and np.array_equal(got[1], untainted[1])
    for key, value, effect in [(TC.KEY, TC.VALUE, "NoSchedule"), (TC.LONG_KEY, "", "NoExecute")]:
        for kind in ("some", "none", "all"):
            since = TC.since_pattern(n, kind, seed=n)
            one = getattr(kx, name[4])("vfio.nvidia.com", "node-a", "node-a", 4, devs, key, value, effect, since)
            got = getattr(kx, name[1])("vfio.nvidia.com", "node-a", "node-a", 4, devs, [(key, value, effect)],
                                       since.reshape(n, 1))
            assert got[0] == one[0] and np.array_equal(got[1], one[1])


def raw(kx, layout, devs, table, nt, since, out):
    ln, ns = C.c_size_t(0xDEAD), C.c_size_t(0xDEAD)
    offs = np.full(4, 0xEE, np.uint64)
    fn = getattr(kx.L, LAYOUTS[layout][5])
    rc = fn(kx.ctx, b"vfio.nvidia.com", b"node-a", b"node-a", 1, devs.ctypes.data, len(devs),
            None if table is None else C.cast(table, C.c_void_p), nt, since.ctypes.data, out.ctypes.data, len(out),
            C.byref(ln), offs.ctypes.data, C.byref(ns))
    return rc, ln.value, ns.value, offs


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_refusals_leave_outputs(kx, layout):
    devs = np.ascontiguousarray(devices(layout, 5, seed=1))
    tab = lambda entries: (DraTaint * len(entries))(*[DraTaint(*[None if x is None else x.encode() for x in e])
                                                      for e in entries])
    t3 = tab(AC.TABLE3)
    ok = np.full((5, 3), -1, np.int64); ok[:, 0] = 7; ok[2, 1] = 8; ok[3, 2] = 9
    cases = [(t3, 0, ok, -1), (None, 3, ok, -1), (None, 1, ok[:, :1], -1),
             (tab(AC.long_table(4) + [AC.TABLE3[0]]), 5, np.zeros((5, 5), np.int64), -1)]
    for key, value, effect in TC.INVALID:
        cases.append((tab([AC.TABLE3[0], (key, value, effect)]), 2, np.zeros((5, 2), np.int64), -1))
    dup = ok.copy(); dup[4, 1:] = [0, 0]
    cases.append((t3, 3, dup, -7))
    late = ok.copy(); late[1, 2] = TC.SINCE_MAX + 1
    cases.append((t3, 3, late, -7))
    for table, nt, since, want in cases:
        out = np.full(64, 0x5A, np.uint8)
        rc, ln, ns, offs = raw(kx, layout, devs, table, nt, np.ascontiguousarray(since), out)
        assert rc == want
        assert (out == 0x5A).all() and (offs == 0xEE).all()
        if want == -1:
            assert ln == 0xDEAD and ns == 0xDEAD
    out = np.zeros(1 << 16, np.uint8)
    rc, ln, ns, offs = raw(kx, layout, devs, t3, 3, ok, out)
    want, woffs = LAYOUTS[layout][2]("vfio.nvidia.com", "node-a", "node-a", 1, devs, AC.TABLE3, ok)
    assert rc == 0 and out[:ln].tobytes() == want and ns == 1 and list(offs[:2]) == list(woffs)


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_every_alignment_and_interleaving(kx, layout):
    devs = devices(layout, 200, seed=11)
    since = AC.since_table(200, 3, seed=2, table=AC.TABLE3)
    want, woffs = LAYOUTS[layout][2]("vfio.nvidia.com", "node-a", "node-a", 1, devs, AC.TABLE3, since)
    tab = (DraTaint * 3)(*[DraTaint(*[x.encode() for x in e]) for e in AC.TABLE3])
    for shift in range(16):
        buf = np.zeros(len(want) + 32, np.uint8)
        ln, ns = C.c_size_t(0), C.c_size_t(0)
        fn = getattr(kx.L, LAYOUTS[layout][5])
        d = np.ascontiguousarray(devs)
        assert fn(kx.ctx, b"vfio.nvidia.com", b"node-a", b"node-a", 1, d.ctypes.data, len(d), C.cast(tab, C.c_void_p), 3,
                  since.ctypes.data, buf.ctypes.data + shift, len(want), C.byref(ln), None, C.byref(ns)) == 0
        assert buf[shift:shift + ln.value].tobytes() == want
        # another emitter between two calls on the same context
        getattr(kx, LAYOUTS[layout][3])("d", "p", "n", 1, devs[:70])


def test_golden_cfg1(kx):
    import os
    want = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_taints_cfg1.jsonl"), "rb").read()
    blob, offs = kx.dra_slices_taints("vfio.nvidia.com", "node-a", "node-a", 1, DC.cfg1(), AC.TABLE3,
                                      np.array([[1767225600, 1767225660, -1]], np.int64))
    assert blob == want and list(offs) == [0, len(want)]
