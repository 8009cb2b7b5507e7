"""CPU tests of the DRA taints (kxpu_dra_slices_taint / kxpu_dra_slices_mdev_taint, include/kxpu.h ABI v11): the C
oracle (oracle/kxpu_dra_taint_oracle.c) against the Python restatement (tests/pyref_dra_taint.py) for both record
layouts with no, some and all devices tainted around the 64-device slice edges, the timestamp edges, the longest key and
value, both effects, every refusal, and taint_since == NULL giving exactly the v9 / v10 oracles' bytes."""
import json

import numpy as np
import pytest

import dra_cases as DC
import dra_mdev_cases as MC
import dra_taint_cases as TC
import pyref_dra_taint as PR
from oracle import dra_mdev_oracle, dra_oracle
from oracle import dra_taint_oracle as TO
from test_dra import LONG_DRIVER, LONG_NAME

LAYOUTS = {
    "pci": (TO.dra_slices_taint, PR.slices, DC, dra_oracle.dra_slices),
    "mdev": (TO.dra_slices_mdev_taint, PR.slices_mdev, MC, dra_mdev_oracle.dra_slices_mdev),
}


def both(layout, driver, pool, node, gen, devs, key, value, effect, since):
    oracle, ref = LAYOUTS[layout][:2]
    got, want = oracle(driver, pool, node, gen, devs, key, value, effect, since), ref(driver, pool, node, gen, devs, key,
                                                                                     value, effect, since)
    if isinstance(got, tuple) and isinstance(got[0], bytes):
        assert isinstance(want, tuple) and got[0] == want[0] and list(got[1]) == list(want[1])
    else:
        assert got == want
    return got


def devices(layout, n, seed, all_attrs=False):
    d = LAYOUTS[layout][2].random_devs(n, seed=seed, all_attrs=all_attrs)
    if n:
        d["iommu_group"] = np.arange(n)  # unique names across the pool
    return d


def parse(blob, offs):
    return [json.loads(blob[offs[s]:offs[s + 1] - 1]) for s in range(len(offs) - 1)]


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("kind", ["none", "some", "all"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 128, 129])
def test_sizes(layout, kind, n):
    since = TC.since_pattern(n, kind, seed=n)
    blob, offs = both(layout, "vfio.nvidia.com", "node-a", "node-a", 3, devices(layout, n, seed=n), TC.KEY, TC.VALUE,
                      "NoSchedule", since)
    objs = parse(blob, offs)
    assert len(objs) == max(1, -(-n // 64))
    assert all(o["spec"]["pool"]["resourceSliceCount"] == len(objs) for o in objs)
    devs = [d for o in objs for d in o["spec"]["devices"]]
    assert len(devs) == n and all(len(o["spec"]["devices"]) <= 64 for o in objs)
    for d, t in zip(devs, since):
        assert ("taints" in d) == (t >= 0)
        assert list(d) == (["name", "attributes", "taints"] if t >= 0 else ["name", "attributes"])


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_timestamp_edges(layout):
    since = TC.since_pattern(len(TC.EDGES), "edges")
    blob, offs = both(layout, "d", "p", "n", 1, devices(layout, len(since), seed=1), TC.KEY, "", "NoExecute", since)
    got = [d["taints"] for o in parse(blob, offs) for d in o["spec"]["devices"]]
    assert got == [[{"key": TC.KEY, "effect": "NoExecute", "timeAdded": TC.EDGES[int(t)]}] for t in since]


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("value", ["", "v", TC.LONG_VALUE])
@pytest.mark.parametrize("effect", ["NoSchedule", "NoExecute"])
def test_longest_names_key_value(layout, value, effect):
    since = TC.since_pattern(300, "some", seed=2)
    blob, offs = both(layout, LONG_DRIVER, LONG_NAME, LONG_NAME, (1 << 63) - 1, devices(layout, 300, seed=2, all_attrs=True),
                      TC.LONG_KEY, value, effect, since)
    for o in parse(blob, offs):
        for d in o["spec"]["devices"]:
            for t in d.get("taints", []):
                assert list(t) == (["key", "value", "effect", "timeAdded"] if value else ["key", "effect", "timeAdded"])
                assert t["key"] == TC.LONG_KEY and t.get("value", "") == value and t["effect"] == effect


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("n", [0, 1, 128, 129, 300])
def test_null_since_is_the_untainted_call(layout, n):
    """taint_since == NULL: the v9 / v10 oracle's bytes and slice_off (128 devices per slice), whatever the taint
    arguments hold"""
    devs = devices(layout, n, seed=n)
    want = LAYOUTS[layout][3]("d", "p", "n", 4, devs)
    for key, value, effect in [(TC.KEY, TC.VALUE, "NoSchedule")] + TC.INVALID[:3]:
        got = both(layout, "d", "p", "n", 4, devs, key, value, effect, None)
        assert got[0] == want[0] and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("key,value,effect", TC.INVALID)
def test_invalid_taint_arguments(layout, key, value, effect):
    since = TC.since_pattern(5, "all")
    assert both(layout, "d", "p", "n", 1, devices(layout, 5, seed=3), key, value, effect, since) == -1


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_invalid_before_unsupported(layout):
    """a bad name or taint argument is reported before a record or a time outside the domain"""
    devs = devices(layout, 3, seed=4)
    since = np.array([0, TC.SINCE_MAX + 1, 5], np.int64)
    assert both(layout, "Bad", "p", "n", 1, devs, TC.KEY, TC.VALUE, "NoSchedule", since) == -1
    assert both(layout, "d", "p", "n", 1, devs, TC.KEY, TC.VALUE, "Evict", since) == -1
    assert both(layout, "d", "p", "n", 1, devs, TC.KEY, TC.VALUE, "NoSchedule", since) == (-7, "taint_since")


@pytest.mark.parametrize("layout", ["pci", "mdev"])
@pytest.mark.parametrize("t", [TC.SINCE_MAX + 1, 1 << 40, (1 << 63) - 1])
def test_since_above_year_9999(layout, t):
    since = TC.since_pattern(200, "some", seed=5)
    since[150] = t
    assert both(layout, "d", "p", "n", 1, devices(layout, 200, seed=5), TC.KEY, TC.VALUE, "NoSchedule", since) == \
        (-7, "taint_since")


@pytest.mark.parametrize("layout", ["pci", "mdev"])
def test_record_domain_still_refused(layout):
    """each v9 / v10 record rule refuses the taint call too, and is named before a bad time on a later record"""
    cases = LAYOUTS[layout][2]
    for why, field, value in cases.BAD:
        devs = np.concatenate([devices(layout, 70, seed=6), cases.bad_rec(field, value), devices(layout, 2, seed=7)])
        since = TC.since_pattern(len(devs), "all", seed=6)
        since[-1] = TC.SINCE_MAX + 1
        assert both(layout, "d", "p", "n", 1, devs, TC.KEY, TC.VALUE, "NoSchedule", since) == (-7, why)


def test_key_forms():
    """a key without a prefix, one with a one-label prefix and the longest one are accepted"""
    devs = devices("pci", 2, seed=8)
    since = np.array([0, -1], np.int64)
    for key in ("unhealthy", "a/b", "x.y.z/u_1-2.3", TC.LONG_KEY):
        blob, offs = both("pci", "d", "p", "n", 1, devs, key, TC.VALUE, "NoSchedule", since)
        assert parse(blob, offs)[0]["spec"]["devices"][0]["taints"][0]["key"] == key
