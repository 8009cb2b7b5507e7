"""GPU tests of kxpu_classify_named: bit-exact against the C oracle (tests/names_oracle.py, itself checked against the
Python restatement on the CPU) on the hand walks, beside a vGPU class, under hypothesis, and on multi-vendor walks from
n = 0 to 2^20 at the scan tile (2048) and launch (256) edges with one-entry and 64-entry tables; the empty table bitwise
kxpu_classify_vf_vgpu's; every refused table with the outputs untouched."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings

import names_cases as NC
import names_oracle as NO
from kxpu_b200.binding import E_INVALID, KxpuError, NAME_DTYPE

pytestmark = pytest.mark.gpu
KEYS = ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups", "dev_rule")


def _check(kx, rules, bits, recs, keys, table, topo=False, viable=False):
    got = kx.classify_named(rules, bits, recs, keys, NO.table(table), topo=topo, viable=viable)
    want = NO.classify_named(rules, bits, recs, keys, table, topo=topo, viable=viable)
    extra = (("dev_slot",) if len(table) else ()) + (("group_numa",) if topo else ()) + (("group_blocker",) if viable else ())
    for k in KEYS + extra:
        assert np.array_equal(np.asarray(got[k], np.uint64), np.asarray(want[k], np.uint64)), k
    for k in ("n_accepted", "n_groups", "n_devids"):
        assert got[k] == want[k], k
    return got


@pytest.mark.parametrize("case", NC.HAND, ids=[c[0] for c in NC.HAND])
def test_hand_cases(kx, case):
    _, recs, keys, bits, table = case
    _check(kx, NC.RULES, bits, recs, keys, table)


def test_beside_a_vgpu_class(kx):
    recs, keys, bits, table = NC.vgpu_case()
    for topo, viable in ((False, False), (True, True)):
        got = _check(kx, NC.RULES, bits, recs, keys, table, topo=topo, viable=viable)
        assert got["n_devids"] == 3 and got["dev_slot"].tolist()[0] == 0


@settings(max_examples=60, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(NC.named_inputs())
def test_hypothesis(kx, inp):
    recs, keys, table = inp
    _check(kx, NC.RULES, NC.VGPU_BIT, recs, keys, table, viable=True)
    _check(kx, NC.RULES, 0, recs, None, table)


def _tables(recs, rules):
    """a one-entry table ("*" of rule 0) and a 64-entry one: 63 ids of rules 0 and 1 that occur, slots shared, and "*" """
    ids = []
    for r in recs[: 1 << 16]:
        v, d = bytes(r["vendor_txt"])[2:6], bytes(r["device_txt"])[2:6]
        rule = [k for k, (rv, _) in enumerate(rules) if rv == v]
        if rule and rule[0] < 2 and int(r["device_len"]) == 7 and (rule[0], d) not in ids:
            ids.append((rule[0], d))
        if len(ids) == 63:
            break
    big = [(r, d, k % 17) for k, (r, d) in enumerate(ids)] + [(0, b"*", 63)]
    return [(0, b"*", 0)], big


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 2047, 2048, 2049, 4097, 1 << 17, 1 << 20])
def test_walks(kx, workloads, oracle_rows, n):
    rules = workloads.XPU_RULES
    recs = workloads.xpu_records(oracle_rows["key"], max(n, 1))[:n]
    one, big = _tables(workloads.xpu_records(oracle_rows["key"], 1 << 16), rules)
    assert len(big) == 64
    for table in ((big,) if n == 1 << 20 else (one, big)):
        got = _check(kx, rules, 0, recs, None, table, viable=n < (1 << 20))
        if n >= 4097:
            assert (got["dev_slot"] != 0xFFFFFFFF).any() and got["n_devids"] > 1


def test_empty_table_is_vf_vgpu(kx, workloads, oracle_rows):
    recs, rules = workloads.xpu_records(oracle_rows["key"], 1 << 18), workloads.XPU_RULES
    for topo, viable in ((False, False), (True, False), (True, True)):
        want = kx.classify_vf_vgpu(rules, 0, recs, None, topo=topo, viable=viable)
        got = kx.classify_named(rules, 0, recs, None, [], topo=topo, viable=viable)
        assert "dev_slot" not in got
        for k in want:
            assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k


@pytest.mark.parametrize("k", range(len(NC.INVALID)))
def test_refused_tables(kx, k):
    table, n_rules, bits = NC.INVALID[k]
    recs, keys, _, _ = NC.vgpu_case()
    rules = NC.RULES[:n_rules]
    with pytest.raises(KxpuError) as e:
        kx.classify_named(rules, bits, recs, keys, np.array([(r, s, d) for r, d, s in table], NAME_DTYPE))
    assert e.value.status == E_INVALID
