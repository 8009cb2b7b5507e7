"""GPU tests of discovery for any configured vendor: kxpu_classify_rules, kxpu_cdi_emit_kind and
kxpu_alloc_names_kind against the oracle (and, for the NVIDIA rule / kind, against the NVIDIA-only calls byte
for byte), and the host flow with two accelerator classes on a fake sysfs."""
import json
import os

import numpy as np
import pytest

import fake_sysfs
import xpu_host
from oracle import xpu_oracle as xo

pytestmark = pytest.mark.gpu

NV = [(b"10de", b"vfio-pci")]
KIND63 = "v" + "e" * 22 + ".example/" + "c" + "l" * 29 + "9"
KINDS = ["nvidia.com/gpu", "amd.com/gpu", KIND63]


def assert_same(a, b, with_rule=True):
    for k in ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups",
              "n_accepted", "n_groups", "n_devids") + (("dev_rule",) if with_rule else ()):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def test_nvidia_rule_is_classify_bitwise(kx, workloads, oracle_rows):
    recs = workloads.cfg3_records(oracle_rows["key"])
    res = kx.classify_rules(NV, recs)
    assert_same(res, kx.classify(recs), with_rule=False)
    assert (res["dev_rule"] == 0).all()
    base = workloads.cfg3_records(oracle_rows["key"], n=70000, seed=9)
    for n in [0, 1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4097, 70000]:
        assert_same(kx.classify_rules(NV, base[:n]), kx.classify(base[:n]), with_rule=False)


def test_classify_launch_count_unchanged(kx, workloads, oracle_rows):
    recs = workloads.cfg3_records(oracle_rows["key"], n=4096)
    c0 = kx.launch_count()
    kx.classify(recs)
    c1 = kx.launch_count()
    kx.classify_rules(NV, recs)
    assert kx.launch_count() - c1 == c1 - c0


def test_five_rules_on_xpu_records(kx, oracle, workloads, oracle_rows):
    recs = workloads.xpu_records(oracle_rows["key"])
    res = kx.classify_rules(workloads.XPU_RULES, recs)
    assert_same(res, xo.classify_rules(workloads.XPU_RULES, recs))
    ids = res["dev_ids"].tolist()
    assert len(ids) > len(set(ids))  # one device id under two vendors gives two entries
    assert set(res["dev_rule"].tolist()) == set(range(5))


def _recs(dt, items):
    recs = np.zeros(len(items), dtype=dt)
    for i, (v, d, drv, grp) in enumerate(items):
        recs["bdf"][i] = b"0000:%02x:%02x.%d" % (i >> 8, (i >> 3) & 31, i & 7)
        vt, dtt = b"0x" + v + b"\n", b"0x" + d + b"\n"
        recs["vendor_txt"][i, :len(vt)] = np.frombuffer(vt, np.uint8)
        recs["device_txt"][i, :len(dtt)] = np.frombuffer(dtt, np.uint8)
        recs["vendor_len"][i], recs["device_len"][i] = len(vt), len(dtt)
        recs["driver"][i] = drv
        recs["iommu_group"][i] = grp
    return recs


def test_mixed_groups_shared_ids_and_sixteen_rules(kx, oracle):
    from kxpu_b200.binding import DEVREC_DTYPE
    rules = [(b"10de", b"vfio-pci"), (b"1002", b"vfio-pci"), (b"1002", b"amdgpu")]
    items = [(b"10de", b"73bf", b"vfio-pci", 5),   # group 5 belongs to rule 0 (its first member)
             (b"1002", b"73bf", b"vfio-pci", 5),   # same group, another rule: a member of group 5
             (b"1002", b"73bf", b"vfio-pci", 6),   # same device id under 1002: a second device-map entry
             (b"1002", b"73bf", b"amdgpu", 7),     # same vendor, the other driver rule: a third entry
             (b"8086", b"1572", b"vfio-pci", 8)]   # no rule
    recs = _recs(DEVREC_DTYPE, items)
    res = kx.classify_rules(rules, recs)
    assert_same(res, xo.classify_rules(rules, recs))
    assert list(res["accept_index"]) == [0, 1, 2, 3, 0xFFFFFFFF]
    assert list(res["group_ids"]) == [5, 6, 7] and list(res["dev_rule"]) == [0, 1, 2]
    assert list(res["dev_groups"]) == [5, 6, 7]
    # 16 rules
    rng = np.random.default_rng(1)
    rules16 = [(b"%04x" % v, d) for v in (0x10de, 0x1002, 0x8086, 0x15b3, 0x1d0f, 0x1da3, 0x1e52, 0x8087) for d in (b"vfio-pci", b"amdgpu")]
    items = [(r[0], b"%04x" % int(rng.integers(0, 0x30)), r[1] if rng.random() < 0.8 else b"nvidia", int(rng.integers(0, 500)))
             for r in (rules16[int(rng.integers(0, 16))] for _ in range(5000))]
    recs = _recs(DEVREC_DTYPE, items)
    res = kx.classify_rules(rules16, recs)
    assert_same(res, xo.classify_rules(rules16, recs))
    assert len(set(res["dev_rule"].tolist())) == 16


def test_device_id_table_retry_over_two_rules(kx, oracle, workloads):
    """200 000 distinct (rule, device id) keys cannot fit the 2^17 slots of the first device-id table"""
    from kxpu_b200.binding import DEVREC_DTYPE
    n = 200000
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    recs["bdf"] = workloads.enumerate_bdfs(n).view("S16").reshape(n)
    recs["vendor_txt"][0::2] = np.frombuffer(b"0x10de\n\0", np.uint8)
    recs["vendor_txt"][1::2] = np.frombuffer(b"0x1002\n\0", np.uint8)
    recs["device_txt"] = np.frombuffer(b"".join(b"0x%05x\n" % (i // 2) for i in range(n)), np.uint8).reshape(n, 8)
    recs["vendor_len"], recs["device_len"] = 7, 8
    recs["driver"] = b"vfio-pci"
    recs["iommu_group"] = np.arange(n, dtype=np.uint32)
    rules = [(b"10de", b"vfio-pci"), (b"1002", b"vfio-pci")]
    res = kx.classify_rules(rules, recs)
    assert res["n_devids"] == n > (1 << 17)
    assert_same(res, xo.classify_rules(rules, recs))


def test_invalid_rule_lists(kx):
    import kxpu_b200 as K
    recs = np.zeros(4, dtype=K.binding.DEVREC_DTYPE)
    bad = [[(b"10de", b"vfio-pci")] * 2, [(b"", b"vfio-pci")], [(b"1234567", b"vfio-pci")], [(b"10\nde", b"vfio-pci")],
           [(b"10de", b"")], [(b"10de", b"a" * 16)], [(b"10de", b"vfio/pci")], [(b"%04x" % i, b"vfio-pci") for i in range(17)]]
    for rules in bad:
        with pytest.raises(K.KxpuError) as e:
            kx.classify_rules(rules, recs)
        assert e.value.status == K.binding.E_INVALID, rules
    with pytest.raises(K.KxpuError) as e:
        kx.classify_rules(np.zeros(0, K.binding.RULE_DTYPE), recs)
    assert e.value.status == K.binding.E_INVALID


@pytest.mark.parametrize("kind", KINDS)
def test_cdi_emit_kind_cfg5_tiles_and_sizing(kx, oracle, workloads, kind):
    kb = kind.encode()
    devs = workloads.cfg5_devices()
    for fmt in (0, 1):
        want = xo.cdi_emit_kind(fmt, kb, devs)
        assert kx.cdi_emit(fmt, devs, kind=kind) == want
        if kind == "nvidia.com/gpu":
            assert want == kx.cdi_emit(fmt, devs)
        assert kx.cdi_emit(fmt, devs[:0], kind=kind) == xo.cdi_emit_kind(fmt, kb, devs[:0])
        assert kx.cdi_emit_len(fmt, devs[:0], kind=kind) == len(xo.cdi_emit_kind(fmt, kb, devs[:0]))
    rng = np.random.default_rng(11)
    n = 1000
    devs = workloads.cfg5_devices(n)
    devs["index"] = rng.integers(0, 2**63, n, dtype=np.uint64) >> rng.integers(0, 63, n).astype(np.uint64)
    devs["iommu_group"] = (rng.integers(0, 2**32 - 1, n, dtype=np.uint64) >> rng.integers(0, 31, n).astype(np.uint64)).astype(np.uint32)
    for cnt in [1, 2, 3, 127, 128, 129, 255, 256, 257, 383, 384, 385, 1000]:
        for fmt in (0, 1):
            want = xo.cdi_emit_kind(fmt, kb, devs[:cnt])
            assert kx.cdi_emit(fmt, devs[:cnt], kind=kind) == want
            assert kx.cdi_emit_len(fmt, devs[:cnt], kind=kind) == len(want)


@pytest.mark.parametrize("kind", KINDS)
def test_alloc_names_kind(kx, oracle, kind):
    rng = np.random.default_rng(2)
    idx = rng.integers(0, 2**63, 5000, dtype=np.uint64) >> rng.integers(0, 63, 5000).astype(np.uint64)
    blob, offs = kx.alloc_names(idx, kind=kind)
    wblob, woffs = xo.alloc_names_kind(kind.encode(), idx)
    assert blob == wblob and np.array_equal(offs, woffs)
    if kind == "nvidia.com/gpu":
        assert blob == kx.alloc_names(idx)[0]


def test_kinds_outside_the_domain_are_rejected(kx, workloads):
    import kxpu_b200 as K
    devs = workloads.cfg5_devices(4)
    for kind in ["nvidia.com", "1a/b", "a/b.c", "a" * 62 + "/b", "a/b\n", "a/\"b\""]:
        with pytest.raises(K.KxpuError) as e:
            kx.cdi_emit(0, devs, kind=kind)
        assert e.value.status == K.binding.E_UNSUPPORTED, kind
        with pytest.raises(K.KxpuError) as e:
            kx.alloc_names(np.zeros(2, np.uint64), kind=kind)
        assert e.value.status == K.binding.E_UNSUPPORTED, kind


HOST_DEVICES = [
    dict(bdf="0000:c1:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=214),
    dict(bdf="0000:c5:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=215),
    dict(bdf="0000:0a:00.0", vendor=b"0x1002\n", device=b"0x73bf\n", driver="vfio-pci", group=30),
    dict(bdf="0000:00:1f.0", vendor=b"0x8086\n", device=b"0x1572\n", driver="vfio-pci", group=3),
]
CLASSES = [("10de", "vfio-pci", "nvidia.com", "nvidia.com/gpu", "cdi-vfio-xxxx"),
           ("1002", "vfio-pci", "amd.com", "amd.com/gpu", "cdi-vfio-amd")]


def test_host_flow_two_classes(tmp_path, kx, pci_text):
    import yaml
    base = fake_sysfs.make_tree(str(tmp_path), HOST_DEVICES)
    pciids = tmp_path / "pci.ids"
    pciids.write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    hp = xpu_host.HostPlugin(kx, base, str(pciids), str(cdi) + "/", CLASSES)
    st = hp.init("YAML")
    # one walk, one busIndex over both classes (walk order: 0000:00:1f.0, 0000:0a:00.0, 0000:c1:00.0, 0000:c5:00.0)
    assert st["iommuMap"] == [["30", [["0000:0a:00.0", 0]]], ["214", [["0000:c1:00.0", 1]]], ["215", [["0000:c5:00.0", 2]]]]
    assert st["iommuClass"] == [1, 0, 0]
    assert st["deviceMap"] == [["73bf", ["30"]], ["2330", ["214", "215"]]] and st["deviceClass"] == [1, 0]
    res = {p["resource"]: p for p in st["plugins"]}
    assert set(res) == {"nvidia.com/GH100_H100_SXM5_80GB", "amd.com/NAVI_21_RADEON_RX_6800_6800_XT___6900_XT"}
    amd = res["amd.com/NAVI_21_RADEON_RX_6800_6800_XT___6900_XT"]
    assert amd["class"] == 1 and amd["devs"] == [["30", "Healthy"]]
    assert amd["socket"] == "/var/lib/kubelet/device-plugins/kata-xpu-NAVI_21_RADEON_RX_6800_6800_XT___6900_XT.sock"
    files = st["cdiFiles"]
    assert [os.path.basename(f) for f in files] == ["cdi-vfio-xxxx.yaml", "cdi-vfio-amd.yaml"]
    nv, ad = (yaml.safe_load(open(f, "rb").read()) for f in files)
    assert nv["kind"] == "nvidia.com/gpu" and [d["name"] for d in nv["devices"]] == ["1", "2"]
    assert ad["kind"] == "amd.com/gpu" and [d["name"] for d in ad["devices"]] == ["0"]
    assert ad["devices"][0]["annotations"]["cdi.k8s.io/vfio30"] == "amd.com/gpu=0"
    # Allocate per class
    assert hp.allocate(["214", "215"]) == {"envs": {"KUBERNETES_CDI_VENDOR_CLASS": "nvidia.com/gpu"},
                                           "cdi_devices": ["nvidia.com/gpu=1", "nvidia.com/gpu=2"]}
    assert hp.allocate(["30"]) == {"envs": {"KUBERNETES_CDI_VENDOR_CLASS": "amd.com/gpu"}, "cdi_devices": ["amd.com/gpu=0"]}
    with pytest.raises(RuntimeError, match="invalid allocation request: devices of more than one class"):
        hp.allocate(["30", "214"])
    # JSON: the same two files as .json
    st = hp.init("JSON")
    assert [os.path.basename(f) for f in st["cdiFiles"]] == ["cdi-vfio-xxxx.json", "cdi-vfio-amd.json"]
    assert json.load(open(st["cdiFiles"][1]))["kind"] == "amd.com/gpu"
    # re-validation: the AMD device moved to another IOMMU group
    link = os.path.join(base, "0000:0a:00.0", "iommu_group")
    os.unlink(link)
    os.symlink(os.path.join(str(tmp_path), "iommu_groups", "3"), link)
    with pytest.raises(RuntimeError, match="invalid allocation request: unknown device: 0000:0a:00.0"):
        hp.allocate(["30"])
    hp.close()


def test_host_class_without_devices_gets_the_empty_document(tmp_path, kx, pci_text):
    base = fake_sysfs.make_tree(str(tmp_path), HOST_DEVICES[:2])
    pciids = tmp_path / "pci.ids"
    pciids.write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    hp = xpu_host.HostPlugin(kx, base, str(pciids), str(cdi) + "/", CLASSES)
    st = hp.init("JSON")
    doc = json.load(open(st["cdiFiles"][1]))
    assert doc == {"cdiVersion": "0.6.0", "kind": "amd.com/gpu", "devices": None, "containerEdits": {}}
    hp.close()
