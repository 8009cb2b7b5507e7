"""GPU tests of vGPU (mdev) discovery: kxpu_classify_mdev, kxpu_mdev_names and kxpu_cdi_emit_mdev against the C
oracle (oracle/kxpu_mdev_oracle.c)."""
import numpy as np
import pytest

from oracle import mdev_oracle as mo

pytestmark = pytest.mark.gpu

KIND63 = "v" + "e" * 22 + ".example/" + "c" + "l" * 29 + "9"
KINDS = ["nvidia.com/vgpu", "intel.com/gvt", KIND63]
SIZES = [0, 1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4097, 70000]
NAME_ERR = 32


def assert_same(a, b):
    for k in ("accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups",
              "n_accepted", "n_groups", "n_devids", "dev_rule"):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def _recs(items):
    """[(vendor, driver, group, name)] -> kxpu_mdevrec, one UUID per record"""
    from kxpu_b200 import workloads as W
    recs = np.zeros(len(items), mo.MDEVREC_DTYPE)
    recs["uuid"] = W.uuids(len(items)).view("S36").reshape(len(items))
    for i, (v, d, g, nm) in enumerate(items):
        vt = b"0x" + v + b"\n"
        recs["parent"][i] = b"0000:%02x:00.0" % (i & 255)
        recs["parent_vendor_txt"][i, :len(vt)] = np.frombuffer(vt, np.uint8)
        recs["vendor_len"][i] = len(vt)
        recs["driver"][i] = d
        recs["type_name"][i, :len(nm)] = np.frombuffer(nm, np.uint8)
        recs["name_len"][i] = len(nm)
        recs["iommu_group"][i] = g
    return recs


def test_classify_mdev_records(kx, workloads):
    recs = workloads.mdev_records()
    res = kx.classify_mdev(workloads.MDEV_RULES, recs)
    assert_same(res, mo.classify_mdev(workloads.MDEV_RULES, recs))
    assert res["n_devids"] > 1000 and set(res["dev_rule"].tolist()) == set(range(len(workloads.MDEV_RULES)))
    base = workloads.mdev_records(70000, seed=9)
    for n in SIZES:
        assert_same(kx.classify_mdev(workloads.MDEV_RULES, base[:n]), mo.classify_mdev(workloads.MDEV_RULES, base[:n]))


def test_intern_table_grows(kx):
    """200 000 distinct type keys cannot fit the 2^17 slots of the first intern table"""
    n = 200000
    from kxpu_b200 import workloads as W
    recs = np.zeros(n, mo.MDEVREC_DTYPE)
    recs["uuid"] = W.uuids(n).view("S36").reshape(n)
    recs["parent"] = b"0000:c1:00.0"
    recs["parent_vendor_txt"] = np.frombuffer(b"0x10de\n\0", np.uint8)
    recs["vendor_len"] = 7
    recs["driver"] = b"nvidia-vgpu"
    names = np.frombuffer(b"".join(b"GRID T%07d-%d" % (i // 2, i & 1) for i in range(n)), np.uint8).reshape(n, 15)
    recs["type_name"][:, :15] = names
    recs["name_len"] = 15
    recs["iommu_group"] = np.arange(n, dtype=np.uint32)
    rules = [(b"10de", b"nvidia-vgpu")]
    res = kx.classify_mdev(rules, recs)
    assert res["n_devids"] == n > (1 << 17)
    assert_same(res, mo.classify_mdev(rules, recs))


def test_keys_rules_and_mixed_groups(kx):
    rules = [(b"10de", b"nvidia-vgpu"), (b"10de", b"vfio_mdev"), (b"1002", b"vfio_mdev")]
    items = [(b"10de", b"nvidia-vgpu", 5, b"GRID T4-1Q\n"),  # group 5: rule 0, key GRID_T4-1Q
             (b"1002", b"vfio_mdev", 5, b"MxGPU"),           # a member of group 5 under rule 2
             (b"10de", b"vfio_mdev", 6, b"GRID T4-1Q"),      # one key under two rules: a second entry
             (b"10de", b"nvidia-vgpu", 7, b" GRID T4-1Q()"),  # equal after sanitising: joins entry 0
             (b"10de", b"nvidia-vgpu", 8, b"\n\t "),         # empty key: no group
             (b"10de", b"nvidia-vgpu", 8, b"GRID_T4-2Q"),
             (b"8086", b"vfio_mdev", 9, b"GVTg")]            # no rule
    recs = _recs(items)
    res = kx.classify_mdev(rules, recs)
    assert_same(res, mo.classify_mdev(rules, recs))
    assert res["accept_index"].tolist() == [0, 1, 2, 3, 0xFFFFFFFF, 4, 0xFFFFFFFF]
    assert res["dev_ids"].tolist() == [0, 0, 5] and res["dev_rule"].tolist() == [0, 1, 0]
    assert res["dev_groups"].tolist() == [5, 7, 6, 8]
    import kxpu_b200 as K
    with pytest.raises(K.KxpuError) as e:
        kx.classify_mdev([(b"10de", b"vfio_mdev")] * 2, recs)
    assert e.value.status == K.binding.E_INVALID


def test_mdev_names(kx, workloads):
    recs = workloads.mdev_records(100000, seed=3)
    idx = np.random.default_rng(1).integers(0, len(recs), 20000).astype(np.uint32)
    blob, offs = kx.mdev_names(recs, idx)
    wblob, woffs = mo.mdev_names(recs, idx)
    assert blob == wblob and np.array_equal(offs, woffs)
    res = kx.classify_mdev(workloads.MDEV_RULES, recs)
    blob, offs = kx.mdev_names(recs, res["dev_ids"])
    assert all(offs[d + 1] > offs[d] for d in range(res["n_devids"]))  # every entry has a non-empty key
    assert kx.mdev_names(recs, np.zeros(0, np.uint32))[0] == b""
    import kxpu_b200 as K
    with pytest.raises(K.KxpuError) as e:
        kx.mdev_names(recs, np.array([len(recs)], np.uint32))
    assert e.value.status == K.binding.E_INVALID


@pytest.mark.parametrize("kind", KINDS)
def test_cdi_emit_mdev(kx, workloads, kind):
    kb = kind.encode()
    devs = workloads.mdev_devices()
    for fmt in (0, 1):
        assert kx.cdi_emit_mdev(fmt, devs, kind) == mo.cdi_emit_mdev(fmt, kb, devs)
        assert kx.cdi_emit_mdev(fmt, devs[:0], kind) == mo.cdi_emit_mdev(fmt, kb, devs[:0])
    rng = np.random.default_rng(11)
    n = 1000
    devs = workloads.mdev_devices(n, seed=2)
    devs["index"] = rng.integers(0, 2**63, n, dtype=np.uint64) >> rng.integers(0, 63, n).astype(np.uint64)
    devs["iommu_group"] = (rng.integers(0, 2**32 - 1, n, dtype=np.uint64) >> rng.integers(0, 31, n).astype(np.uint64)).astype(np.uint32)
    devs["uuid"][::7] = b"12345678-1234-1234-1234-123456789012"
    for cnt in [1, 2, 3, 127, 128, 129, 255, 256, 257, 383, 384, 385, 1000]:
        for fmt in (0, 1):
            assert kx.cdi_emit_mdev(fmt, devs[:cnt], kind) == mo.cdi_emit_mdev(fmt, kb, devs[:cnt])


def test_cdi_emit_mdev_domain(kx, workloads):
    import kxpu_b200 as K
    devs = workloads.mdev_devices(300)
    for bad in (b"12345678-1234-1234-1234-12345678901", b"ABCDEF12-1234-1234-1234-123456789012", b"12345678_1234-1234-1234-123456789012"):
        d = devs.copy()
        d["uuid"][257] = bad
        with pytest.raises(K.KxpuError) as e:
            kx.cdi_emit_mdev(0, d, "nvidia.com/vgpu")
        assert e.value.status == K.binding.E_UNSUPPORTED
    for parent in (b"0000:C1:00.0", b""):  # a byte outside [0-9a-f:.], an empty parent
        d = devs.copy()
        d["parent"][3] = parent
        for fmt in (0, 1):
            with pytest.raises(K.KxpuError) as e:
                kx.cdi_emit_mdev(fmt, d, "nvidia.com/vgpu")
            assert e.value.status == K.binding.E_UNSUPPORTED
    with pytest.raises(K.KxpuError) as e:
        kx.cdi_emit_mdev(1, devs, "nvidia.com")
    assert e.value.status == K.binding.E_UNSUPPORTED
