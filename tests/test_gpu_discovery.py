"""GPU parity tests of classify (K5), CDI emit (K6), Allocate names (K7) and the
ListAndWatch wire bytes through the C ABI, against the oracle."""
import hashlib
import os

import numpy as np
import pytest

from conftest import GOLDEN
from test_oracle import check_classify

pytestmark = pytest.mark.gpu

CLS_KEYS = ["accept_index", "group_ids", "group_off", "group_members", "dev_ids", "dev_off", "dev_groups"]


def assert_classify_equal(a, b):
    for k in ("n_accepted", "n_groups", "n_devids"):
        assert a[k] == b[k], k
    for k in CLS_KEYS:
        assert np.array_equal(a[k], b[k]), k


def test_cfg1_one_mocked_gpu(kx, oracle, workloads, pci_text):
    """BASELINE.json configs[0]: one VFIO NVIDIA GPU end to end: classify -> name -> CDI -> Allocate."""
    recs = workloads.cfg1_record()
    res = kx.classify(recs)
    assert_classify_equal(res, oracle.classify(recs))
    assert list(res["accept_index"]) == [0] and list(res["group_ids"]) == [214]
    assert int(res["dev_ids"][0]).to_bytes(8, "little").rstrip(b"\0") == b"2330"
    tab = kx.pciids_load(pci_text)
    row = kx.lookup(tab, np.array([0x10de2330], np.uint32))
    assert kx.names(tab, row)[0][0] == b"GH100_H100_SXM5_80GB"
    tab.free()
    devs = np.zeros(1, dtype=oracle.CDIDEV_DTYPE)
    devs["bdf"], devs["iommu_group"], devs["index"] = b"0000:c1:00.0", 214, 0
    assert kx.cdi_emit(0, devs) == open(os.path.join(GOLDEN, "cfg1.yaml"), "rb").read()
    assert kx.cdi_emit(1, devs) == open(os.path.join(GOLDEN, "cfg1.json"), "rb").read()
    assert kx.alloc_names(np.array([0], np.uint64))[0] == b"nvidia.com/gpu=0"
    assert kx.lw_encode(np.array([214], np.uint32)) == b"\x0a\x0e\x0a\x03214\x12\x07Healthy"


def test_classify_edge_cases(kx, oracle, workloads, oracle_rows):
    recs = workloads.cfg3_records(oracle_rows["key"], n=5000, seed=3)
    rng = np.random.default_rng(5)
    recs["iommu_group"] = rng.integers(0, 300, len(recs)).astype(np.uint32)
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.05, 8, 0).astype(np.uint8)
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.02, 4, 0).astype(np.uint8)
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.02, 1, 0).astype(np.uint8)
    recs["flags"] |= np.where(rng.random(len(recs)) < 0.01, 16, 0).astype(np.uint8)
    odd = rng.random(len(recs)) < 0.02
    recs["vendor_txt"][odd] = np.frombuffer(b"0x10DE\n\0", np.uint8)
    res = kx.classify(recs)
    assert_classify_equal(res, oracle.classify(recs))
    check_classify(res, recs)  # and against the independent Python walk


def test_classify_sizes_and_degenerate(kx, oracle, workloads, oracle_rows):
    base = workloads.cfg3_records(oracle_rows["key"], n=70000, seed=9)
    for n in [0, 1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4097, 70000]:
        recs = base[:n].copy()
        assert_classify_equal(kx.classify(recs), oracle.classify(recs))
    # nothing accepted
    recs = base[:1000].copy()
    recs["driver"] = b"nvidia"
    r = kx.classify(recs)
    assert r["n_accepted"] == 0 and r["n_groups"] == 0 and (r["accept_index"] == 0xFFFFFFFF).all()
    # everything in ONE group (long member list), then every record its own group
    recs = base[:20000].copy()
    recs["iommu_group"] = 7
    assert_classify_equal(kx.classify(recs), oracle.classify(recs))
    recs["iommu_group"] = np.arange(20000, dtype=np.uint32)[::-1]
    assert_classify_equal(kx.classify(recs), oracle.classify(recs))
    # distinct 5-digit device ids, every record its own group: 200 000 ids cannot fit the 2^17 slots of the
    # first device-id table (the run is repeated with a full-size one); 100 000 may or may not need the retry
    for n in (200000, 100000):
        recs = np.zeros(n, dtype=base.dtype)
        recs["bdf"] = workloads.enumerate_bdfs(n).view("S16").reshape(n)
        recs["vendor_txt"] = np.frombuffer(b"0x10de\n\0", np.uint8)
        recs["device_txt"] = np.frombuffer(b"".join(b"0x%05x\n" % i for i in range(n)), np.uint8).reshape(n, 8)
        recs["vendor_len"], recs["device_len"] = 7, 8
        recs["driver"] = b"vfio-pci"
        recs["iommu_group"] = np.arange(n, dtype=np.uint32)
        res = kx.classify(recs)
        assert res["n_devids"] == res["n_groups"] == n
        assert_classify_equal(res, oracle.classify(recs))
    assert 200000 > (1 << 17)


def test_cfg3_one_million_devices(kx, oracle, workloads, oracle_rows):
    """BASELINE.json configs[2]: 2^20 synthetic VFIO devices, bit-exact device lists."""
    recs = workloads.cfg3_records(oracle_rows["key"])
    assert len(recs) == 1 << 20
    res = kx.classify(recs)
    want = oracle.classify(recs)
    assert_classify_equal(res, want)
    assert res["n_accepted"] > 400000
    # size-independent properties: busIndex is a dense 0..A-1 ramp in walk order; CSR covers it
    acc = res["accept_index"][res["accept_index"] != 0xFFFFFFFF]
    assert np.array_equal(acc, np.arange(res["n_accepted"], dtype=np.uint32))
    assert res["group_off"][-1] == res["n_accepted"] and res["dev_off"][-1] == res["n_groups"]
    assert np.array_equal(np.sort(res["dev_groups"]), np.sort(res["group_ids"]))
    # ListAndWatch payload for the largest device id list
    sizes = np.diff(res["dev_off"])
    d = int(np.argmax(sizes))
    groups = res["dev_groups"][res["dev_off"][d]:res["dev_off"][d + 1]]
    assert kx.lw_encode(groups) == oracle.lw_encode(groups)


def test_cfg5_cdi_burst(kx, oracle, workloads):
    """BASELINE.json configs[4]: 65 536 CDI device emits, byte-identical JSON and YAML."""
    devs = workloads.cfg5_devices()
    j = kx.cdi_emit(1, devs)
    y = kx.cdi_emit(0, devs)
    oj, oy = oracle.cdi_emit(1, devs), oracle.cdi_emit(0, devs)
    assert len(j) == 20585718 and len(y) == 13330372
    assert hashlib.sha256(j).hexdigest() == hashlib.sha256(oj).hexdigest() and j == oj
    assert hashlib.sha256(y).hexdigest() == hashlib.sha256(oy).hexdigest() and y == oy
    names, offs = kx.alloc_names(devs["index"])
    onames, ooffs = oracle.alloc_names(devs["index"])
    assert names == onames and np.array_equal(offs, ooffs)


def test_cdi_emit_small_and_wide(kx, oracle, workloads):
    devs = workloads.cfg5_devices(300)
    for n in [0, 1, 2, 7, 8, 9, 300]:
        for fmt in (0, 1):
            assert kx.cdi_emit(fmt, devs[:n]) == oracle.cdi_emit(fmt, devs[:n])
    wide = np.zeros(4, dtype=oracle.CDIDEV_DTYPE)
    wide["bdf"] = [b"10000:00:00.0", b"0000:59:19.7", b"ffff:ff:1f.7", b"0001:00:00.0"]
    wide["iommu_group"] = [0, 4294967295, 12345, 9]
    wide["index"] = [18446744073709551615, 0, 1000000, 99]
    for fmt in (0, 1):
        assert kx.cdi_emit(fmt, wide) == oracle.cdi_emit(fmt, wide)
    idx = np.array([0, 9, 10, 99, 100, 18446744073709551615], np.uint64)
    assert kx.alloc_names(idx)[0] == oracle.alloc_names(idx)[0]
    bad = np.zeros(1, dtype=oracle.CDIDEV_DTYPE)
    bad["bdf"] = b'00"0:00:00.0'
    import kxpu_b200 as K
    with pytest.raises(K.KxpuError) as e:
        kx.cdi_emit(1, bad)
    assert e.value.status == -7


def test_lw_encode_health(kx, oracle):
    rng = np.random.default_rng(1)
    g = rng.integers(0, 2**32 - 1, 5000, dtype=np.uint64).astype(np.uint32)
    h = (rng.random(5000) < 0.7).astype(np.uint8)
    assert kx.lw_encode(g, h) == oracle.lw_encode(g, h)
    assert kx.lw_encode(g[:0]) == b""


def test_ctx_is_thread_safe(kx, oracle, pci_text):
    """grpc-go runs Allocate handlers concurrently on one shared ctx (generic_device_plugin.go:320):
    hammer one kxpu_ctx from several OS threads with the three per-request calls."""
    import threading
    tab = kx.pciids_load(pci_text)
    want_names, _ = oracle.alloc_names(np.arange(64, dtype=np.uint64))
    errors = []

    def worker(seed):
        try:
            rng = np.random.default_rng(seed)
            for _ in range(40):
                idx = rng.integers(0, 1 << 40, 64, dtype=np.uint64)
                got, _ = kx.alloc_names(idx)
                assert got == oracle.alloc_names(idx)[0]
                rows = kx.lookup(tab, np.array([0x10de2330, 0x10de2901, 0x80861572], np.uint32))
                assert rows[0] >= 0 and rows[1] == -1 and rows[2] >= 0
                assert kx.names(tab, rows)[0] == [b"GH100_H100_SXM5_80GB", b"", b"ETHERNET_CONTROLLER_X710_FOR_10GBE_SFP"]
                g = rng.integers(0, 5000, 17).astype(np.uint32)
                assert kx.lw_encode(g) == oracle.lw_encode(g)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(s,)) for s in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[:3]
    assert kx.alloc_names(np.arange(64, dtype=np.uint64))[0] == want_names
    tab.free()


def test_cdi_emit_tile_boundaries_and_sizing(kx, oracle, workloads):
    """The emitter works in tiles of 128 devices whose bytes leave shared memory with one bulk store:
    every count around the tile edges, mixed field widths (so that fragments start at every 16-byte
    phase), and the two-call sizing protocol."""
    rng = np.random.default_rng(11)
    n = 1000
    devs = workloads.cfg5_devices(n)
    devs["index"] = rng.integers(0, 2**63, n, dtype=np.uint64) >> rng.integers(0, 63, n).astype(np.uint64)
    devs["iommu_group"] = (rng.integers(0, 2**32 - 1, n, dtype=np.uint64) >> rng.integers(0, 31, n).astype(np.uint64)).astype(np.uint32)
    for cnt in [1, 2, 3, 127, 128, 129, 255, 256, 257, 383, 384, 385, 1000]:
        for fmt in (0, 1):
            want = oracle.cdi_emit(fmt, devs[:cnt])
            assert kx.cdi_emit(fmt, devs[:cnt]) == want
            assert kx.cdi_emit_len(fmt, devs[:cnt]) == len(want)


def _rec_strategy():
    from hypothesis import strategies as st
    vendor = st.sampled_from([b"0x10de\n", b"0x10de", b"0x10DE\n", b"0x8086\n", b"0x10de\n\n", b"10de\n", b"0x10d\n", b"0x", b"0", b"",
                              b"\n\n10de\n", b"0x10de\n\0"])
    device = st.sampled_from([b"0x2330\n", b"0x2331\n", b"0x20b0\n", b"0x2330", b"0x\n", b"0x", b"0", b"0xabcdef", b"0x1\n", b"0x2330\n\n"])
    driver = st.sampled_from([b"vfio-pci", b"nvidia", b"vfio-pc", b"vfio-pci2", b"", b"Vfio-pci"])  # NUL-padded C strings: no embedded NUL
    return st.tuples(vendor, device, driver, st.integers(0, 6), st.sampled_from([0, 0, 0, 0, 1, 2, 4, 8, 16, 12]))


def test_classify_hypothesis_fuzz(kx, oracle):
    """Oracle-vs-GPU fuzz of kxpu_classify with hypothesis-generated records: odd id files (short,
    upper case, extra newlines), near-miss driver names, read-error flags, tiny group universes so
    that groups interleave and first members fail their device read."""
    from hypothesis import given, settings, strategies as st, HealthCheck
    import kxpu_b200 as K
    dt = K.binding.DEVREC_DTYPE

    @settings(max_examples=120, deadline=None, suppress_health_check=list(HealthCheck))
    @given(st.lists(_rec_strategy(), min_size=0, max_size=300))
    def run(items):
        recs = np.zeros(len(items), dtype=dt)
        for i, (v, d, drv, grp, fl) in enumerate(items):
            recs["bdf"][i] = b"0000:%02x:%02x.%d" % (i >> 8, (i >> 3) & 31, i & 7)
            recs["vendor_txt"][i, :len(v[:8])] = np.frombuffer(v[:8], np.uint8)
            recs["device_txt"][i, :len(d[:8])] = np.frombuffer(d[:8], np.uint8)
            recs["vendor_len"][i], recs["device_len"][i] = len(v), len(d)
            recs["driver"][i] = drv
            recs["iommu_group"][i] = grp
            recs["flags"][i] = fl
        assert_classify_equal(kx.classify(recs), oracle.classify(recs))
        check_classify(kx.classify(recs), recs)
    run()
