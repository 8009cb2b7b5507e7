"""CPU tests of kxpu_classify_named's statements: the C oracle (tests/names_oracle.c over the C classify oracles)
against the Python restatement on hand walks and under hypothesis, the empty table against kxpu_classify_vf_vgpu's
oracle, every table the call refuses, and the host plugin's refusals of XpuClass::resourceNames."""
import ctypes as C

import pytest
from hypothesis import given, settings

import dra_host as DH
import fake_sysfs
import names_cases as NC
import names_oracle as NO
import pyref_names as P
import vf_vgpu_oracle as VO


def _both(recs, keys, bits, table, **kw):
    got = NO.classify_named(NC.RULES, bits, recs, keys, table, **kw)
    want = P.classify_named(NC.RULES, bits, recs, None if keys is None else [k.tobytes() for k in keys], table, **kw)
    return got, want


@pytest.mark.parametrize("case", NC.HAND, ids=[c[0] for c in NC.HAND])
def test_hand_cases(case):
    _, recs, keys, bits, table = case
    got, want = _both(recs, keys, bits, table)
    assert got == want


def test_hand_expectations():
    recs = NC.HAND[2][1]  # 2331, 2330, 2331, 2321 with 2330 and 2331 on slot 0
    out = P.classify_named(NC.RULES, 0, recs, None, NC.HAND[2][4])
    assert out["dev_groups"] == [1, 2, 3, 4] and out["dev_off"] == [0, 3, 4]
    assert out["dev_slot"] == [0, P.NO_SLOT] and out["dev_ids"][0] == 0
    star = P.classify_named(NC.RULES, 0, NC.HAND[1][1], None, NC.HAND[1][4])
    assert star["n_devids"] == 1 and star["dev_groups"] == [1, 2, 3]
    # slot 0's lowest candidate is a member of group 1, whose first member keeps its id key
    nf = P.classify_named(NC.RULES, 0, NC.HAND[6][1], None, NC.HAND[6][4])
    assert nf["dev_slot"] == [P.NO_SLOT, 0] and nf["dev_ids"] == [int.from_bytes(b"2330", "little"), 1]


def test_beside_a_vgpu_class():
    recs, keys, bits, table = NC.vgpu_case()
    for topo in (False, True):
        for viable in (False, True):
            got, want = _both(recs, keys, bits, table, topo=topo, viable=viable)
            assert got == want


def test_empty_table_is_vf_vgpu():
    recs, keys, bits, _ = NC.vgpu_case()
    assert NO.classify_named(NC.RULES, bits, recs, keys, []) == VO.classify_vf_vgpu(NC.RULES, bits, recs, keys)


@settings(max_examples=150, deadline=None)
@given(NC.named_inputs())
def test_hypothesis(inp):
    recs, keys, table = inp
    for bits in (0, NC.VGPU_BIT):
        got, want = _both(recs, keys, bits, table, viable=bool(bits))
        assert got == want


@pytest.mark.parametrize("k", range(len(NC.INVALID)))
def test_invalid_tables(k):
    table, n_rules, bits = NC.INVALID[k]
    assert not NO.check(table, n_rules, bits)
    assert not P.valid(table, n_rules, bits)
    assert NO.check([(0, b"2330", 0), (0, b"*", 1), (1, b"*", 1)], 3, NC.VGPU_BIT)


# -- host refusals
NV = "10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-xxxx"
MGR = "10de,nvidia,nvidia.com,nvidia.com/vgpu,cdi-vgpu-vf"
AMD = "1002,vfio-pci,amd.com,amd.com/gpu,cdi-amd"


def set_names(hp, cls, names, vgpu=False):
    hp.L.kxh_set_resource_names.restype = C.c_int
    hp.L.kxh_set_resource_names.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
    spec = ";".join("%s=%s" % kv for kv in names.items())
    assert hp.L.kxh_set_resource_names(hp.h, int(vgpu), cls, spec.encode()) == 0


@pytest.fixture
def plugin(tmp_path):
    base = fake_sysfs.make_tree(str(tmp_path), [])
    hps = []

    def make(classes):
        hp = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
        assert hp.L.kxh_set_classes(hp.h, classes.encode()) == 0
        hps.append(hp)
        return hp
    yield make
    for hp in hps:
        hp.close()


CLS = "class 10de/vfio-pci (nvidia.com/gpu)"
REFUSALS = [
    (NV, {"*": "-pgpu"}, CLS + ': resourceNames["*"] = "-pgpu" is not a qualified name (1-63 bytes, alphanumeric at both '
                         "ends, [-A-Za-z0-9_.] inside)"),
    (NV, {"*": "a" * 64}, CLS + ': resourceNames["*"] = "' + "a" * 64 + '" is not a qualified name (1-63 bytes, alphanumeric '
                          "at both ends, [-A-Za-z0-9_.] inside)"),
    (NV, {"*": "p/gpu"}, CLS + ': resourceNames["*"] = "p/gpu" is not a qualified name (1-63 bytes, alphanumeric at both '
                         "ends, [-A-Za-z0-9_.] inside)"),
    (NV, {"*": ""}, CLS + ': resourceNames["*"] = "" is not a qualified name (1-63 bytes, alphanumeric at both ends, '
                    "[-A-Za-z0-9_.] inside)"),
    (NV, {"23A0": "pgpu"}, CLS + ': resourceNames key "23A0" is neither 4 lowercase hex digits nor "*"'),
    (NV, {"0x2330": "pgpu"}, CLS + ': resourceNames key "0x2330" is neither 4 lowercase hex digits nor "*"'),
    (NV, {"%04x" % k: "g%d" % k for k in range(65)},
     CLS + ": resourceNames brings the entries of all classes to 65, over 64"),
]


@pytest.mark.parametrize("k", range(len(REFUSALS)))
def test_host_refusals(plugin, k):
    classes, names, msg = REFUSALS[k]
    hp = plugin(classes)
    set_names(hp, 0, names)
    assert DH.initiate(hp) == msg


def test_host_refuses_one_name_on_two_classes(plugin):
    hp = plugin(NV + ";" + AMD)
    set_names(hp, 0, {"*": "gpu-any"})
    set_names(hp, 1, {"74a1": "gpu-any"})
    assert DH.initiate(hp) == ('class 1002/vfio-pci (amd.com/gpu): resourceNames["74a1"] = "gpu-any" is also configured on '
                               "class 10de/vfio-pci (nvidia.com/gpu); socket names ignore the namespace")


def test_host_refuses_a_vf_vgpu_class(plugin):
    import vf_vgpu_host as VH
    hp = plugin(NV + ";" + MGR)
    VH.set_vf_vgpu(hp, 1)
    set_names(hp, 1, {"*": "vgpu"})
    assert DH.initiate(hp) == ("class 10de/nvidia (nvidia.com/vgpu): resourceNames cannot rename a vfVgpu class, whose vGPUs "
                               "are named by their type keys")


def test_host_refuses_a_vgpu_class(plugin):
    hp = plugin(NV)
    hp.L.kxh_set_vgpu_classes.argtypes = [C.c_void_p, C.c_char_p]
    assert hp.L.kxh_set_vgpu_classes(hp.h, b"10de,nvidia-vgpu-vfio,nvidia.com,nvidia.com/mdev,cdi-mdev") == 0
    set_names(hp, 0, {"*": "vgpu"}, vgpu=True)
    assert DH.initiate(hp) == ("vGPU class 10de/nvidia-vgpu-vfio (nvidia.com/mdev): resourceNames cannot rename a vGPU "
                               "class, whose vGPUs are named by their type keys")
