"""CPU tests of the PCIe AER health and the taint lists (include/kxpu.h ABI v12): the C oracle
(oracle/kxpu_aer_oracle.c) against the Python restatement (tests/pyref_aer.py).  kxpu_aer_health on every file case of
tests/aer_cases.py (names with spaces, TOTAL lines that are not last or repeated, TOTAL_ERR_FATALX, '\\r', leading zeros,
2^64 - 2 / 2^64 - 1 / 2^64, empty files and files of 4096 and 4097 bytes), shared and unaligned files, empty groups,
limits of 0 and the maximum, the refusals, and a hypothesis fuzz; kxpu_dra_slices_taints / _mdev_taints with one to four
entries at the longest key and value, n = 0, 63, 64, 65 on both layouts, the duplicate key and effect refusal, the other
refusals, and the two identities: taint_since == NULL gives the untainted bytes, one entry the _taint call's."""
import json

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import aer_cases as AC
import dra_cases as DC
import dra_mdev_cases as MC
import dra_taint_cases as TC
import pyref_aer as PR
from oracle import aer_oracle as AO
from oracle import dra_mdev_oracle, dra_oracle
from oracle import dra_taint_oracle as TO

MAX = (1 << 64) - 1


def both_aer(*args):
    got, want = AO.aer_health(*args), PR.aer_health(*args)
    if isinstance(want, int):
        assert got == want
        return got
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    return got


@pytest.mark.parametrize("which", [AC.F, AC.N])
def test_file_cases(which):
    cs = AC.cases(which)
    other = AC.cases(AC.N if which == AC.F else AC.F)[0][1]
    files = [(c[1], other) if which == AC.F else (other, c[1]) for c in cs]
    text, off, ln = AC.pack(files)
    n = len(files)
    totals, aer = both_aer(text, off, ln, 0, 0, np.arange(n + 1, dtype=np.uint32), np.arange(n, dtype=np.uint32))
    k = 0 if which == AC.F else 1
    for i, (name, _, want) in enumerate(cs):
        assert int(totals[2 * i + k]) == want, name
        assert bool(aer[i] & 4) == (want == MAX), name


def test_folding_limits_and_sharing():
    f = lambda c: AC.aer_file(AC.F, [c] + [0] * 17)
    nf = lambda c: AC.aer_file(AC.N, [0] * 11 + [c] + [0] * 6)
    files = [(f(0), nf(0)), (f(2), nf(0)), (f(0), nf(5)), (b"", nf(1)), (f(MAX - 1), nf(MAX - 1))]
    text, off, ln = AC.pack(files, share=[0, 1, 2, 3, 4, 1, 1, 2])  # records 5..7 share files, as vGPUs do
    goff = np.array([0, 1, 1, 3, 5, 8, 8], np.uint32)  # two empty groups
    mem = np.array([0, 1, 2, 3, 4, 5, 6, 7], np.uint32)
    # records (fatal, non-fatal): (0, 0) (2, 0) (0, 5) (unknown, 1) (2^64 - 2, 2^64 - 2) (2, 0) (2, 0) (0, 5)
    for fl, nl, want in [(0, 0, [0, 0, 3, 7, 3, 0]), (2, 5, [0, 0, 0, 7, 0, 0]), (1, 4, [0, 0, 3, 7, 3, 0]),
                         (MAX, MAX, [0, 0, 0, 4, 0, 0]), (MAX - 2, MAX - 2, [0, 0, 0, 7, 0, 0])]:
        totals, aer = both_aer(text, off, ln, fl, nl, goff, mem)
        assert list(aer) == want, (fl, nl)
    assert list(totals[:10]) == [0, 0, 2, 0, 0, 5, MAX, 1, MAX - 1, MAX - 1]


def test_refusals():
    text, off, ln = AC.pack([(AC.aer_file(AC.F, [0] * 18), AC.aer_file(AC.N, [0] * 18))] * 3)
    g, m = np.array([0, 2, 3], np.uint32), np.array([0, 1, 2], np.uint32)
    assert both_aer(text, off, ln, 0, 0, g, m)[1].tolist() == [0, 0]
    bad = off.copy(); bad[3] = len(text) - ln[3] + 1
    assert both_aer(text, bad, ln, 0, 0, g, m) == -1                             # a range past text_len
    bad = off.copy(); bad[5] = len(text) + 1; ln2 = ln.copy(); ln2[5] = 0
    assert both_aer(text, bad, ln2, 0, 0, g, m) == -1                            # an empty file past text_len
    bad = off.copy(); bad[0] = (1 << 64) - 1
    assert both_aer(text, bad, ln, 0, 0, g, m) == -1                             # a range that wraps
    assert both_aer(text, off, ln, 0, 0, np.array([0, 2, 1], np.uint32), m) == -1  # group_off decreases
    assert both_aer(text, off, ln, 0, 0, g, np.array([0, 3, 2], np.uint32)) == -1  # a member >= n
    edge = off.copy(); edge[5] = len(text); ln3 = ln.copy(); ln3[5] = 0
    assert both_aer(text, edge, ln3, 0, 0, g, m)[1].tolist() == [0, 4]           # an empty file at text_len is unknown


_line = st.one_of(
    st.sampled_from(["TLP 0", "Data Link Protocol 3", "TOTAL_ERR_FATALX 3", "TOTAL_ERR_NONFATAL", "", "x TOTAL_ERR_FATAL 1"]),
    st.builds(lambda p, num: p + num, st.sampled_from(["TOTAL_ERR_FATAL ", "TOTAL_ERR_NONFATAL "]),
              st.one_of(st.integers(0, (1 << 64) + 5).map(str), st.sampled_from(["007", "00", "", "1\r", " 4", "5 ", "-1"]),
                        st.text("0123456789\r ", max_size=22))),
    st.text(st.characters(min_codepoint=32, max_codepoint=126), max_size=40))
_file = st.builds(lambda ls, nl: ("\n".join(ls) + ("\n" if nl else "")).encode(), st.lists(_line, max_size=8), st.booleans())


@settings(max_examples=300, deadline=None)
@given(st.lists(st.tuples(_file, _file), min_size=1, max_size=12), st.data())
def test_fuzz_aer(files, data):
    n = len(files)
    share = data.draw(st.lists(st.integers(0, n - 1), min_size=1, max_size=16))
    text, off, ln = AC.pack(files, gaps=data.draw(st.lists(st.integers(0, 40), min_size=2 * n, max_size=2 * n)),
                            share=share)
    sizes = data.draw(st.lists(st.integers(0, 3), max_size=8))
    goff = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    mem = np.array(data.draw(st.lists(st.integers(0, len(share) - 1), min_size=int(goff[-1]), max_size=int(goff[-1]))),
                   np.uint32)
    lim = st.sampled_from([0, 1, 3, 10 ** 19, MAX - 1, MAX])
    both_aer(text, off, ln, data.draw(lim), data.draw(lim), goff, mem)


# ---------------------------------------------------------------- the taint lists
LAYOUTS = {
    "pci": (AO.dra_slices_taints, PR.slices, DC, dra_oracle.dra_slices, TO.dra_slices_taint),
    "mdev": (AO.dra_slices_mdev_taints, PR.slices_mdev, MC, dra_mdev_oracle.dra_slices_mdev, TO.dra_slices_mdev_taint),
}


def both(layout, devs, taints, since, driver="vfio.nvidia.com", pool="node-a", node="node-a", gen=3):
    oracle, ref = LAYOUTS[layout][:2]
    got, want = oracle(driver, pool, node, gen, devs, taints, since), ref(driver, pool, node, gen, devs, taints, since)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == list(want[1])
    else:
        assert got == want
    return got


def devices(layout, n, seed, all_attrs=False):
    d = LAYOUTS[layout][2].random_devs(n, seed=seed, all_attrs=all_attrs)
    if n:
        d["iommu_group"] = np.arange(n)
    return d


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
@pytest.mark.parametrize("n", [0, 63, 64, 65])
def test_lists_longest(layout, k, n):
    table = AC.long_table(k)
    since = AC.since_table(n, k, seed=n + k, frac=2)
    blob, offs = both(layout, devices(layout, n, seed=n, all_attrs=True), table, since, "d" * 63, "p" * 63, "n" * 63,
                      (1 << 63) - 1)
    objs = [json.loads(blob[offs[s]:offs[s + 1] - 1]) for s in range(len(offs) - 1)]
    assert len(objs) == max(1, -(-n // 64))
    devs = [d for o in objs for d in o["spec"]["devices"]]
    for d, row in zip(devs, since):
        keys = [t["key"] for t in d.get("taints", [])]
        assert keys == [table[t][0] for t in range(k) if row[t] >= 0]


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 129])
def test_identities(layout, n):
    devs = devices(layout, n, seed=50 + n)
    untainted = LAYOUTS[layout][3]("vfio.nvidia.com", "node-a", "node-a", 3, devs)
    got = both(layout, devs, AC.TABLE3, None)
    assert got[0] == untainted[0] and list(got[1]) == list(untainted[1])
    for key, value, effect in [(TC.KEY, TC.VALUE, "NoSchedule"), (TC.LONG_KEY, "", "NoExecute")]:
        since = TC.since_pattern(n, "some", seed=n)
        one = LAYOUTS[layout][4]("vfio.nvidia.com", "node-a", "node-a", 3, devs, key, value, effect, since)
        got = both(layout, devs, [(key, value, effect)], since.reshape(n, 1))
        assert got[0] == one[0] and list(got[1]) == list(one[1])


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_table3_order_and_duplicates(layout):
    devs = devices(layout, 4, seed=1)
    since = np.array([[5, 7, -1], [-1, -1, 9], [1, -1, 2], [-1, -1, -1]], np.int64)
    blob, offs = both(layout, devs, AC.TABLE3, since)
    d = json.loads(blob[:offs[1] - 1])["spec"]["devices"]
    assert [[(t["key"], t["value"]) for t in x.get("taints", [])] for x in d] == [
        [(AC.DRV + "/unhealthy", "vfio-device-missing"), (AC.DRV + "/pcie-aer", "fatal")],
        [(AC.DRV + "/pcie-aer", "nonfatal")],
        [(AC.DRV + "/unhealthy", "vfio-device-missing"), (AC.DRV + "/pcie-aer", "nonfatal")], []]
    # fatal and nonfatal share key and effect: carrying both is refused, also when one time is 0
    bad = since.copy(); bad[3] = [-1, 0, 4]
    assert both(layout, devs, AC.TABLE3, bad) == (-7, "taint_duplicate")
    # a time above the maximum is reported first
    bad[2, 0] = TC.SINCE_MAX + 1
    assert both(layout, devs, AC.TABLE3, bad) == (-7, "taint_since")
    # the same key with another effect is allowed
    tab = [AC.TABLE3[1], (AC.DRV + "/pcie-aer", "fatal", "NoExecute")]
    both(layout, devs, tab, np.array([[1, 2]] * 4, np.int64))


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_invalid_tables(layout):
    devs = devices(layout, 3, seed=2)
    s = lambda k: np.zeros((3, k), np.int64)
    assert both(layout, devs, [], s(0)) == -1
    assert both(layout, devs, AC.long_table(4) + [AC.TABLE3[0]], s(5)) == -1
    for key, value, effect in TC.INVALID:
        if key is None or value is None or effect is None:
            continue  # NULL members: the GPU tests pass them through ctypes
        assert both(layout, devs, [AC.TABLE3[0], (key, value, effect)], s(2)) == -1, (key, value, effect)


@settings(max_examples=150, deadline=None)
@given(st.sampled_from(["pci", "mdev"]), st.integers(0, 140), st.integers(1, 4), st.integers(0, 1 << 30), st.booleans())
def test_fuzz_lists(layout, n, k, seed, long):
    table = AC.long_table(k) if long else (AC.TABLE3 + [("example.com/x", "", "NoExecute")])[:k]
    both(layout, devices(layout, n, seed=seed % 1000), table, AC.since_table(n, k, seed=seed, table=table))


def test_golden_cfg1():
    """the cfg1 H100 with the host's table: the device node missing since 2026-01-01T00:00:00Z and a fatal AER count
    since a minute later"""
    import os
    want = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dra_taints_cfg1.jsonl"), "rb").read()
    since = np.array([[1767225600, 1767225660, -1]], np.int64)
    blob, offs = both("pci", DC.cfg1(), AC.TABLE3, since, **{k: v for k, v in DC.CFG1.items()})
    assert blob == want and list(offs) == [0, len(want)]
