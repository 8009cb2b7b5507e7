"""GPU tests of the vGPU-on-VF calls: kxpu_vf_vgpu_types equal to the C checker and the Python restatement on the hand
cases, every current_vgpu_type shape, a seeded fuzz and the 2^20-record walk; kxpu_classify_vf_vgpu equal to the checker
on a seeded fuzz and on that walk, and bitwise kxpu_classify_rules / _topo / _viable with an empty mask on the existing
classify workloads; the argument errors and limits."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import pyref_vf_vgpu as P
import vf_vgpu_cases as VV
import vf_vgpu_oracle as VO
from kxpu_b200.binding import E_INVALID, E_UNSUPPORTED, KxpuError, VGPUKEY_DTYPE

pytestmark = pytest.mark.gpu
CLASSIFY_KEYS = ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups", "dev_rule")


def _types(kx, recs, tables, pyref=True):
    got = kx.vf_vgpu_types(recs, tables)
    want = VO.vf_vgpu_types(recs, tables)
    assert [k.tobytes() for k in got["keys"]] == want["keys"]
    assert got["type_id"].tolist() == want["type_id"] and got["status"].tolist() == want["status"]
    if pyref:
        assert want == P.vf_vgpu_types(recs, tables)
    return got


@pytest.mark.parametrize("name", sorted(VV.HAND))
def test_hand_cases(kx, name):
    tables, curs, _ = VV.HAND[name]
    _types(kx, VV.vts(*[VV.vt(c) for c in curs]), tables)


def test_current_shapes(kx):
    recs = VV.vts(*[VV.vt(c, f) for (c, f), _ in VV.CURRENT])
    got = _types(kx, recs, [b"557 : A\n"])
    assert list(zip(got["status"].tolist(), got["type_id"].tolist())) == [w for _, w in VV.CURRENT]


@settings(max_examples=150, deadline=None, suppress_health_check=list(HealthCheck))
@given(VV.type_inputs())
def test_types_fuzz(kx, inp):
    tables, recs = inp
    _types(kx, recs, tables)


def test_types_many_ids_grow_the_table(kx):
    """More distinct IDs than the first run's table holds: the call runs again with room for every line."""
    tables = [b"".join(b"%d : type-%d\n" % (k, k % 997) for k in range(1, 20001))]
    recs = VV.vts(*[VV.vt(b"%d" % k) for k in (1, 2, 19999, 20000, 20001, 4096)])
    got = _types(kx, recs, tables, pyref=False)
    assert got["status"].tolist() == [VV.NAMED] * 4 + [VV.UNNAMED, VV.NAMED]


def _classify(kx, recs, keys, mask, topo, viable):
    got = kx.classify_vf_vgpu(VV.RULES, mask, recs, keys, topo=topo, viable=viable)
    want = VO.classify_vf_vgpu(VV.RULES, mask, recs, keys, topo=topo, viable=viable)
    for k in CLASSIFY_KEYS + (("group_numa",) if topo else ()) + (("group_blocker",) if viable else ()):
        assert [int(x) for x in got[k]] == [int(x) for x in want[k]], k
    return got


@settings(max_examples=150, deadline=None, suppress_health_check=list(HealthCheck))
@given(VV.classify_inputs(), st.sampled_from([0, VV.VGPU_BIT, 1 | VV.VGPU_BIT, 7]), st.booleans(), st.booleans())
def test_classify_fuzz(kx, inp, mask, topo, viable):
    recs, keys = inp
    _classify(kx, recs, keys, mask, topo, viable)


def test_big_walk(kx, workloads):
    recs, vts, tables = workloads.vf_vgpu_walk(1 << 20)
    got = _types(kx, vts, tables, pyref=False)
    st_ = got["status"]
    assert (st_ == VV.NAMED).sum() > 0 and (st_ == VV.UNNAMED).sum() > 0 and (st_ == VV.BAD).sum() > 0
    rules = [(b"10de", b"nvidia")]
    for topo, viable in ((False, False), (True, True)):
        c = kx.classify_vf_vgpu(rules, 1, recs, got["keys"], topo=topo, viable=viable)
        want = VO.classify_vf_vgpu(rules, 1, recs, got["keys"], topo=topo, viable=viable)
        for k in CLASSIFY_KEYS:
            assert np.array_equal(np.asarray(c[k], np.uint64), np.asarray(want[k], np.uint64)), k
        assert c["n_groups"] == int((st_ == VV.NAMED).sum()) and c["n_devids"] == len(workloads.H100_VGPU_TYPES)


@pytest.mark.parametrize("which", ["xpu", "topo", "viab"])
def test_empty_mask_is_the_existing_call(kx, workloads, oracle_rows, which):
    if which == "viab":
        recs, rules = workloads.viab_records(1 << 18), [(b"10de", b"vfio-pci"), (b"1002", b"vfio-pci")]
        want = kx.classify_viable(rules, recs, topo=True)
        got = kx.classify_vf_vgpu(rules, 0, recs, None, topo=True, viable=True)
        extra = ("group_numa", "group_blocker")
    elif which == "topo":
        recs, rules = workloads.topo_records(oracle_rows["key"], 1 << 18), [(b"10de", b"vfio-pci")]
        want = kx.classify_topo(rules, recs)
        got = kx.classify_vf_vgpu(rules, 0, recs, None, topo=True)
        extra = ("group_numa",)
    else:
        recs, rules = workloads.xpu_records(oracle_rows["key"], 1 << 18), workloads.XPU_RULES
        want = kx.classify_rules(rules, recs)
        got = kx.classify_vf_vgpu(rules, 0, recs, None)
        extra = ()
    for k in CLASSIFY_KEYS + extra:
        assert np.array_equal(got[k], want[k]), k
    for k in ("n_accepted", "n_groups", "n_devids"):
        assert got[k] == want[k]


def test_errors_and_limits(kx):
    recs = np.array([VV.dev(b"0000:03:00.4", 31)], VV.XO.DEVREC_DTYPE)
    keys = np.array([VV.key(b"A")], VGPUKEY_DTYPE)
    with pytest.raises(KxpuError) as e:
        kx.classify_vf_vgpu(VV.RULES, 1 << 3, recs, keys)  # a bit at n_rules
    assert e.value.status == E_INVALID
    with pytest.raises(KxpuError) as e:
        kx.classify_vf_vgpu(VV.RULES, VV.VGPU_BIT, recs, None)
    assert e.value.status == E_INVALID
    with pytest.raises(KxpuError) as e:
        kx.vf_vgpu_types(VV.vts(VV.vt(b"557")), (b"557 : A\n", [0, 8, 4]))
    assert e.value.status == E_INVALID
    with pytest.raises(KxpuError) as e:
        kx.vf_vgpu_types(VV.vts(VV.vt(b"557")), (b"", [0, 1 << 40]))
    assert e.value.status == E_UNSUPPORTED
    L = kx.L
    one = VV.vts(VV.vt(b"557"))
    out = np.zeros(1, VGPUKEY_DTYPE)
    toff = np.zeros(1, np.uint64)
    tid, st_ = np.zeros(1, np.uint32), np.zeros(1, np.uint8)
    assert L.kxpu_vf_vgpu_types(kx.ctx, one.ctypes.data, 1 << 30, None, toff.ctypes.data, 0, out.ctypes.data,
                                tid.ctypes.data, st_.ctypes.data) == E_UNSUPPORTED
    assert kx.vf_vgpu_types(VV.vts(), [b"557 : A"])["status"].tolist() == []
