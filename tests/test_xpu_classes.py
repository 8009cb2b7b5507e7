"""CPU tests of discovery for any configured vendor: the oracle's rule-list classify, kind-parametrised CDI
emit and Allocate names against the pinned NVIDIA-only restatement and the independent Python walk, and the
host gather under a class list."""
import json

import numpy as np
import pytest

import fake_sysfs
import pyref_xpu
import xpu_host
from oracle import xpu_oracle as xo

NV = [(b"10de", b"vfio-pci")]
KIND63 = "v" + "e" * 22 + ".example/" + "c" + "l" * 29 + "9"  # 63 bytes: the longest supported kind


def _edge_records(workloads, rows, n=5000, seed=3):
    """the records of test_classify_edge_cases: read-error flags, directories, 0x10DE, tiny group universe"""
    recs = workloads.cfg3_records(rows["key"], n=n, seed=seed)
    rng = np.random.default_rng(5)
    recs["iommu_group"] = rng.integers(0, 300, len(recs)).astype(np.uint32)
    for bit, p in ((8, 0.05), (4, 0.02), (1, 0.02), (16, 0.01)):
        recs["flags"] |= np.where(rng.random(len(recs)) < p, bit, 0).astype(np.uint8)
    odd = rng.random(len(recs)) < 0.02
    recs["vendor_txt"][odd] = np.frombuffer(b"0x10DE\n\0", np.uint8)
    short = rng.random(len(recs)) < 0.01
    recs["vendor_len"][short] = 1
    return recs


def _rec_dicts(recs):
    out = []
    for r in recs:
        fl = int(r["flags"])
        out.append(dict(bdf=r["bdf"], is_dir=bool(fl & 16),
                        vendor=None if fl & 1 else bytes(r["vendor_txt"][:r["vendor_len"]]),
                        device=None if fl & 8 else bytes(r["device_txt"][:r["device_len"]]),
                        driver=None if fl & 2 else r["driver"], group=None if fl & 4 else int(r["iommu_group"])))
    return out


def assert_same(a, b, with_rule=True):
    for k in ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups",
              "n_accepted", "n_groups", "n_devids") + (("dev_rule",) if with_rule else ()):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def check_against_pyref(res, rules, recs):
    iommu, devmap, accept = pyref_xpu.classify_rules(rules, _rec_dicts(recs))
    want_acc = np.array([0xFFFFFFFF if a is None else a for a in accept], dtype=np.uint32)
    assert np.array_equal(res["accept_index"], want_acc)
    assert list(res["group_ids"]) == list(iommu.keys())
    for gi, g in enumerate(iommu):
        mem = res["group_members"][res["group_off"][gi]:res["group_off"][gi + 1]]
        assert [(recs["bdf"][m], int(res["accept_index"][m])) for m in mem] == iommu[g]
    got = [(int(r), int(x).to_bytes(8, "little").rstrip(b"\0")) for r, x in zip(res["dev_rule"], res["dev_ids"])]
    assert got == list(devmap.keys())
    for di, d in enumerate(devmap):
        assert list(res["dev_groups"][res["dev_off"][di]:res["dev_off"][di + 1]]) == devmap[d]


def test_nvidia_rule_equals_classify_cfg3(oracle, workloads, oracle_rows):
    recs = workloads.cfg3_records(oracle_rows["key"])
    res = xo.classify_rules(NV, recs)
    assert_same(res, oracle.classify(recs), with_rule=False)
    assert res["n_devids"] > 0 and (res["dev_rule"] == 0).all()


def test_nvidia_rule_equals_classify_edge_cases(oracle, workloads, oracle_rows):
    recs = _edge_records(workloads, oracle_rows)
    res = xo.classify_rules(NV, recs)
    assert_same(res, oracle.classify(recs), with_rule=False)
    assert (res["dev_rule"] == 0).all()


def test_xpu_records_five_rules_match_pyref(oracle, workloads, oracle_rows):
    recs = workloads.xpu_records(oracle_rows["key"], n=20000)
    res = xo.classify_rules(workloads.XPU_RULES, recs)
    check_against_pyref(res, workloads.XPU_RULES, recs)
    assert set(res["dev_rule"].tolist()) == set(range(5))
    ids = [int(x) for x in res["dev_ids"]]
    assert len(ids) > len(set(ids))  # one device id under two vendors: two entries


def test_invalid_rule_lists(oracle):
    recs = np.zeros(4, dtype=oracle.DEVREC_DTYPE)
    bad = [[], [(b"10de", b"vfio-pci")] * 2, [(b"", b"vfio-pci")], [(b"1234567", b"vfio-pci")], [(b"10\nde", b"vfio-pci")],
           [(b"10de", b"")], [(b"10de", b"a" * 16)], [(b"10de", b"vfio/pci")], [(b"%04x" % i, b"vfio-pci") for i in range(17)]]
    for rules in bad:
        assert xo.classify_rules(rules, recs) is None, rules
        assert not pyref_xpu.rules_ok(rules), rules
    ra = xo.rules_array(NV)
    ra["vendor"] = b"10\0de"  # a byte after the terminating NUL
    assert xo.classify_rules(ra, recs) is None
    assert xo.classify_rules([(b"a" * 6, b"d" * 15)], recs) is not None


def test_classify_rules_hypothesis_fuzz(oracle):
    """kxo_classify_rules against pyref_xpu.classify_rules: mixed vendors (lengths 1-6), drivers, read-error flags and
    rule lists of 1-16 rules, the same vendor with two drivers included."""
    from hypothesis import HealthCheck, given, settings, strategies as st
    vendors = [b"10de", b"1002", b"8086", b"1", b"15b3ab", b"10DE", b"abc"]
    drivers = [b"vfio-pci", b"nvidia", b"amdgpu", b"vfio-pc", b"", b"i915"]
    # a record carries at most 8 bytes of the file: the 6-byte vendor comes without its newline
    vtxt = st.sampled_from([(b"0x" + v + b"\n")[:8] for v in vendors] + [b"0x10de", b"0x", b"0", b"", b"\n\n10de\n", b"0x1002\n\n"])
    dtxt = st.sampled_from([b"0x2330\n", b"0x73bf\n", b"0x2330", b"0x\n", b"0", b"0xabcdef", b"0x1\n"])
    rec = st.tuples(vtxt, dtxt, st.sampled_from(drivers), st.integers(0, 6), st.sampled_from([0, 0, 0, 0, 1, 2, 4, 8, 16, 12]))
    rule = st.tuples(st.sampled_from(vendors), st.sampled_from([d for d in drivers if d]))
    dt = oracle.DEVREC_DTYPE

    @settings(max_examples=300, deadline=None, suppress_health_check=list(HealthCheck))
    @given(st.lists(rule, min_size=1, max_size=16, unique=True), st.lists(rec, min_size=0, max_size=200))
    def run(rules, items):
        recs = np.zeros(len(items), dtype=dt)
        for i, (v, d, drv, grp, fl) in enumerate(items):
            recs["bdf"][i] = b"0000:%02x:%02x.%d" % (i >> 8, (i >> 3) & 31, i & 7)
            recs["vendor_txt"][i, :len(v[:8])] = np.frombuffer(v[:8], np.uint8)
            recs["device_txt"][i, :len(d[:8])] = np.frombuffer(d[:8], np.uint8)
            recs["vendor_len"][i], recs["device_len"][i] = len(v), len(d)
            recs["driver"][i] = drv
            recs["iommu_group"][i] = grp
            recs["flags"][i] = fl
        res = xo.classify_rules(rules, recs)
        check_against_pyref(res, rules, recs)
        if rules == NV:
            assert_same(res, oracle.classify(recs), with_rule=False)
    run()


@pytest.mark.parametrize("fmt", [0, 1])
def test_cdi_emit_kind_nvidia_is_byte_identical(oracle, workloads, fmt):
    devs = workloads.cfg5_devices()
    assert xo.cdi_emit_kind(fmt, b"nvidia.com/gpu", devs) == oracle.cdi_emit(fmt, devs)
    assert xo.cdi_emit_kind(fmt, b"nvidia.com/gpu", devs[:0]) == oracle.cdi_emit(fmt, devs[:0])
    idx = np.arange(0, 10**6, 977, dtype=np.uint64)
    assert xo.alloc_names_kind(b"nvidia.com/gpu", idx)[0] == oracle.alloc_names(idx)[0]


@pytest.mark.parametrize("kind", ["amd.com/gpu", "intel.com/gpu", KIND63])
def test_cdi_emit_kind_documents_parse(oracle, workloads, kind):
    import yaml
    assert len(KIND63) == 63
    devs = workloads.cfg5_devices(300)
    kb = kind.encode()
    for fmt, load in ((0, yaml.safe_load), (1, json.loads)):
        doc = load(xo.cdi_emit_kind(fmt, kb, devs).decode())
        assert doc["kind"] == kind and len(doc["devices"]) == 300
        for d, want in zip(doc["devices"], devs):
            g, i = int(want["iommu_group"]), int(want["index"])
            assert d["name"] == str(i) and d["annotations"]["cdi.k8s.io/vfio%d" % g] == "%s=%d" % (kind, i)
        empty = load(xo.cdi_emit_kind(fmt, kb, devs[:0]).decode())
        assert empty["kind"] == kind and not empty["devices"]
    triples = [(d["bdf"].decode(), int(d["iommu_group"]), int(d["index"])) for d in devs]
    assert xo.cdi_emit_kind(0, kb, devs) == pyref_xpu.cdi_yaml(triples, kind)
    assert xo.cdi_emit_kind(1, kb, devs) == pyref_xpu.cdi_json(triples, kind)
    blob, offs = xo.alloc_names_kind(kb, np.array([0, 7, 12345], np.uint64))
    assert [blob[offs[k]:offs[k + 1]] for k in range(3)] == [kb + b"=0", kb + b"=7", kb + b"=12345"]


def test_kind_domain(oracle):
    good = ["nvidia.com/gpu", "a/b", "amd.com/gpu", "x-y_z.w9/c_d-e3", KIND63]
    bad = ["", "nvidia.com", "/gpu", "nvidia.com/", "1nv.com/gpu", "nv.com/1gpu", "nv./gpu", "nv.com/gpu-", "nv.com/g.pu",
           "a/b/c", "nv com/gpu", "nv.com/gpu\n", "nvidia.com/gpu=", "\"a\"/b", "a" * 62 + "/b", "ü.com/gpu"]
    for k in good:
        assert xo.kind_ok(k.encode()) and pyref_xpu.kind_ok(k), k
    devs = np.zeros(1, dtype=oracle.CDIDEV_DTYPE)
    for k in bad:
        assert not xo.kind_ok(k.encode()) and not pyref_xpu.kind_ok(k), k
        assert xo.cdi_emit_kind(0, k.encode(), devs) is None
        assert xo.alloc_names_kind(k.encode(), np.zeros(1, np.uint64)) is None


HOST_DEVICES = [
    dict(bdf="0000:c1:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=214),
    dict(bdf="0000:c5:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=215),
    dict(bdf="0000:0a:00.0", vendor=b"0x1002\n", device=b"0x73bf\n", driver="vfio-pci", group=30),
    dict(bdf="0000:0b:00.0", vendor=b"0x1002\n", device=b"0x73bf\n", driver="amdgpu", group=31),
    dict(bdf="0000:00:1f.0", vendor=b"0x8086\n", device=b"0x1572\n", driver="vfio-pci", group=3),
]
CLASSES = [("10de", "vfio-pci", "nvidia.com", "nvidia.com/gpu", "cdi-vfio-xxxx"),
           ("1002", "vfio-pci", "amd.com", "amd.com/gpu", "cdi-vfio-amd")]


@pytest.mark.parametrize("fast", [False, True])
def test_gather_under_two_classes_reads_amd_records(tmp_path, fast):
    from kxpu_b200.binding import DEVREC_DTYPE
    base = fake_sysfs.make_tree(str(tmp_path), HOST_DEVICES)
    default = fake_sysfs.gather(base, DEVREC_DTYPE)
    assert xpu_host.gather_classes(base, DEVREC_DTYPE, [CLASSES[0]], fast=fast).tobytes() == default.tobytes()
    recs = {r["bdf"]: r for r in xpu_host.gather_classes(base, DEVREC_DTYPE, CLASSES, fast=fast, threads=2)}
    amd = recs[b"0000:0a:00.0"]
    assert amd["driver"] == b"vfio-pci" and amd["iommu_group"] == 30 and amd["flags"] == 0
    assert bytes(amd["device_txt"][:7]) == b"0x73bf\n"
    other = recs[b"0000:0b:00.0"]  # AMD on amdgpu: the driver is read, nothing behind it
    assert other["driver"] == b"amdgpu" and other["iommu_group"] == 0 and other["device_len"] == 0
    intel = recs[b"0000:00:1f.0"]  # no class: nothing behind the vendor is read
    assert intel["driver"] == b"" and intel["device_len"] == 0
    # the default list reads the AMD record only up to its vendor, as the reference does
    d = {r["bdf"]: r for r in default}[b"0000:0a:00.0"]
    assert d["driver"] == b"" and d["device_len"] == 0
