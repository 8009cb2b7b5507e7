"""CPU tests of the vGPU (mdev) checkers: the C oracle (oracle/kxpu_mdev_oracle.c) against the independent Python
restatement (tests/pyref_mdev.py) under a fuzz, against the pinned PCI walk (kxo_classify_rules) on cfg3, and the
emitted CDI documents parsed back with PyYAML / json."""
import json

import numpy as np
import pytest
import yaml
from hypothesis import given, settings
from hypothesis import strategies as st

import pyref_mdev as P
from oracle import mdev_oracle as MO
from oracle import xpu_oracle as XO

MDEVREC, MDEVCDI = MO.MDEVREC_DTYPE, MO.MDEVCDI_DTYPE
VENDOR_ERR, DRIVER_ERR, IOMMU_ERR, IS_DIR, NAME_ERR = 1, 2, 4, 16, 32
RULES = [(b"10de", b"nvidia-vgpu"), (b"10de", b"vfio_mdev"), (b"1002", b"vfio_mdev")]
KIND63 = b"v" + b"e" * 22 + b".example/" + b"c" + b"l" * 29 + b"9"


def to_recs(items):
    """pyref_mdev dicts -> kxpu_mdevrec array"""
    recs = np.zeros(len(items), MDEVREC)
    for i, r in enumerate(items):
        recs["uuid"][i] = r["uuid"] if len(r["uuid"]) == 36 else b""
        recs["parent"][i] = b"0000:%02x:00.0" % (i & 255)
        v = r["vendor"][:8]
        recs["parent_vendor_txt"][i, :len(v)] = np.frombuffer(v, np.uint8)
        recs["vendor_len"][i] = len(r["vendor"])
        recs["driver"][i] = r["driver"]
        nm = r["name"][:40]
        recs["type_name"][i, :len(nm)] = np.frombuffer(nm, np.uint8)
        recs["name_len"][i] = min(len(r["name"]), 255)
        recs["iommu_group"][i] = r["group"]
        recs["flags"][i] = (VENDOR_ERR * r["vendor_err"] | DRIVER_ERR * r["driver_err"] | IOMMU_ERR * r["iommu_err"] |
                            IS_DIR * r["is_dir"] | NAME_ERR * r["name_err"])
    return recs


def check_against_pyref(rules, items):
    recs = to_recs(items)
    got = MO.classify_mdev(rules, recs)
    acc, groups, devs = P.classify_mdev(rules, items)
    assert [None if a == 0xFFFFFFFF else int(a) for a in got["accept_index"]] == acc
    assert got["group_ids"].tolist() == [g for g, _ in groups]
    assert [got["group_members"][got["group_off"][k]:got["group_off"][k + 1]].tolist() for k in range(len(groups))] == \
        [m for _, m in groups]
    assert got["dev_ids"].tolist() == [f for f, _, _ in devs]
    assert got["dev_rule"].tolist() == [r for _, r, _ in devs]
    assert [got["dev_groups"][got["dev_off"][d]:got["dev_off"][d + 1]].tolist() for d in range(len(devs))] == \
        [g for _, _, g in devs]
    return got


UUIDS = [b"0f1e2d3c-4b5a-6978-8796-a5b4c3d2e1f0", b"12345678-1234-1234-1234-123456789012",
         b"aaaaaaaa-bbbb-cccc-dddd-eeeeeeeeeeee", b"AAAAAAAA-BBBB-CCCC-DDDD-EEEEEEEEEEEE", b"12345678-1234-1234-1234-12345678901",
         b"123456781234-1234-1234-1234567890123"]
NAMES = st.one_of(st.sampled_from([b"GRID T4-1Q\n", b"GRID  T4-1Q", b" GRID T4-1Q\n\n", b"\t\n", b"", b"A(1)/B+",
                                   b"A1B", b"x" * 40, b"y" * 41, b"GRID\x85T4"]),
                  st.binary(max_size=44))
RARE = st.sampled_from([False] * 7 + [True])  # a read error in about one record of eight
REC = st.fixed_dictionaries(dict(
    uuid=st.sampled_from(UUIDS), vendor=st.sampled_from([b"0x10de\n", b"0x1002\n", b"0x8086\n", b"0x10de", b"0", b"0x10de\n\n\n"]),
    driver=st.sampled_from([b"nvidia-vgpu", b"vfio_mdev", b"i915"]), group=st.integers(0, 6) | st.just(0xFFFFFFFF),
    name=NAMES, is_dir=RARE, vendor_err=RARE, driver_err=RARE, iommu_err=RARE, name_err=RARE))


@settings(max_examples=300, deadline=None)
@given(st.lists(REC, max_size=40))
def test_oracle_equals_pyref_fuzz(items):
    check_against_pyref(RULES, items)


@settings(max_examples=300, deadline=None)
@given(st.binary(max_size=40))
def test_type_key_fuzz(name):
    assert MO.type_key(name) == P.type_key(name)


def test_uuid_form():
    for u in UUIDS:
        assert MO.uuid_ok(u) == P.uuid_ok(u)
    assert [P.uuid_ok(u) for u in UUIDS] == [True, True, True, False, False, False]


def test_groups_keys_and_rules():
    def rec(uuid, vendor, driver, group, name, **kw):
        r = dict(uuid=uuid, vendor=vendor, driver=driver, group=group, name=name, is_dir=False, vendor_err=False,
                 driver_err=False, iommu_err=False, name_err=False)
        r.update(kw)
        return r
    u = UUIDS[0]
    items = [rec(u, b"0x10de\n", b"nvidia-vgpu", 5, b"GRID T4-1Q\n"),       # group 5, rule 0, key GRID_T4-1Q
             rec(u, b"0x1002\n", b"vfio_mdev", 5, b"other"),               # member of group 5 under rule 2
             rec(u, b"0x10de\n", b"vfio_mdev", 6, b" GRID T4-1Q"),          # same key under rule 1: a second entry
             rec(u, b"0x10de\n", b"nvidia-vgpu", 7, b"GRID  T4-1Q"),        # GRID__T4-1Q: another key
             rec(u, b"0x10de\n", b"nvidia-vgpu", 8, b"GRID T4-1Q(a)"),      # GRID_T4-1Qa
             rec(u, b"0x10de\n", b"nvidia-vgpu", 9, b"\n", ),               # empty key: no group 9 yet
             rec(u, b"0x10de\n", b"nvidia-vgpu", 9, b"GRID T4-1Q", name_err=True),
             rec(u, b"0x10de\n", b"nvidia-vgpu", 9, b"GRID_T4-1Q"),         # equal after sanitising: joins entry 0
             rec(u, b"0x10de\n", b"nvidia-vgpu", 9, b"x")]                  # later member, no key needed
    got = check_against_pyref(RULES, items)
    assert got["accept_index"].tolist() == [0, 1, 2, 3, 4, 0xFFFFFFFF, 0xFFFFFFFF, 5, 6]
    # entry 1 is (rule 1, GRID_T4-1Q): its first record is record 0, the first candidate with the key under any rule
    assert got["dev_ids"].tolist() == [0, 0, 3, 4] and got["dev_rule"].tolist() == [0, 1, 0, 0]
    assert got["dev_groups"].tolist() == [5, 9, 6, 7, 8]
    assert MO.classify_mdev([], to_recs(items)) is None
    assert MO.classify_mdev([(b"10de", b"vfio_mdev")] * 2, to_recs(items)) is None


def test_pci_tie_on_cfg3(workloads, oracle_rows):
    """cfg3's PCI records (all 2^20) as mdev records (type name = the device id) classify like kxo_classify_rules"""
    pci = workloads.cfg3_records(oracle_rows["key"])
    n = len(pci)
    recs = np.zeros(n, MDEVREC)
    recs["uuid"] = workloads.uuids(n).view("S36").reshape(n)
    recs["parent"] = pci["bdf"]
    recs["parent_vendor_txt"], recs["vendor_len"] = pci["vendor_txt"], pci["vendor_len"]
    recs["driver"], recs["iommu_group"] = pci["driver"], pci["iommu_group"]
    dl = pci["device_len"].astype(np.int64)
    recs["type_name"][:, :6] = pci["device_txt"][:, 2:8]
    assert (pci["device_txt"][:, :2] == np.frombuffer(b"0x", np.uint8)).all()
    recs["name_len"] = np.where(dl >= 2, dl - 2, 0)  # the name is the id after "0x": its key is read_id's id
    fl = pci["flags"]
    name_err = ((fl & 8) != 0) | (dl < 2) | (dl > 8)  # a failed device read is a failed name read
    recs["flags"] = (fl & (VENDOR_ERR | DRIVER_ERR | IOMMU_ERR | IS_DIR)) | np.where(name_err, NAME_ERR, 0)
    rules = workloads.XPU_RULES
    want = XO.classify_rules(rules, pci)
    got = MO.classify_mdev(rules, recs)
    for k in ("accept_index", "group_ids", "group_off", "group_members", "dev_off", "dev_groups", "n_accepted", "n_groups",
              "n_devids", "dev_rule"):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k
    first = got["dev_ids"].astype(np.int64)
    packed = np.zeros(len(first), np.uint64)
    for k in range(4):
        packed |= pci["device_txt"][first, 2 + k].astype(np.uint64) << np.uint64(8 * k)
    assert np.array_equal(packed, want["dev_ids"])
    assert want["n_devids"] > 100 and len(set(want["dev_rule"].tolist())) == len(rules)


def devices(items):
    devs = np.zeros(len(items), MDEVCDI)
    for i, (u, g, p, x) in enumerate(items):
        devs[i] = (u, g, p, x)
    return devs


DEVS = [(b"12345678-1234-1234-1234-123456789012", 7, b"0000:00:01.0", 0),      # all-decimal uuid, quoted parent
        (b"0f1e2d3c-4b5a-6978-8796-a5b4c3d2e1f0", 4294967295, b"0000:c1:00.0", 18446744073709551615),  # plain parent
        (b"aaaaaaaa-bbbb-cccc-dddd-eeeeeeeeeeee", 30, b"00:59", 2),             # base-60 parent: quoted in YAML
        (b"00000000-0000-0000-0000-000000000000", 0, b"1:2:3.4", 3)]


@pytest.mark.parametrize("kind", [b"nvidia.com/vgpu", b"intel.com/gvt", KIND63])
def test_documents_parse(kind):
    devs = devices(DEVS)
    yd, jd = MO.cdi_emit_mdev(0, kind, devs), MO.cdi_emit_mdev(1, kind, devs)
    ref = [dict(uuid=u, group=g, parent=p, index=x) for u, g, p, x in DEVS]
    assert yd == P.cdi_yaml(kind, ref) and jd == P.cdi_json(kind, ref)
    want = dict(cdiVersion="0.6.0", kind=kind.decode(), devices=[
        dict(name=str(x), annotations={"attach-pci": "true", "bdf": p.decode(), "cdi.k8s.io/vfio%d" % g: "%s=%d" % (kind.decode(), x),
                                       "mdev": u.decode()},
             containerEdits=dict(deviceNodes=[dict(path="/dev/vfio/%d" % g)])) for u, g, p, x in DEVS])
    assert yaml.safe_load(yd) == want
    assert json.loads(jd) == dict(want, containerEdits={})
    # an all-decimal address reads as base 60 and is quoted, one with a hex letter stays plain; every uuid is plain
    assert b'bdf: "0000:00:01.0"' in yd and b'bdf: "00:59"' in yd and b"bdf: 0000:c1:00.0\n" in yd
    assert b"mdev: 12345678-1234-1234-1234-123456789012\n" in yd and b"mdev: 00000000-0000-0000-0000-000000000000\n" in yd
    assert list(json.loads(jd)["devices"][0]["annotations"]) == ["attach-pci", "bdf", "cdi.k8s.io/vfio7", "mdev"]
    # zero devices
    assert yaml.safe_load(MO.cdi_emit_mdev(0, kind, devs[:0])) == dict(cdiVersion="0.6.0", kind=kind.decode(), devices=[])
    assert json.loads(MO.cdi_emit_mdev(1, kind, devs[:0])) == dict(cdiVersion="0.6.0", kind=kind.decode(), devices=None,
                                                                   containerEdits={})


def test_documents_outside_the_domain():
    ok = devices(DEVS[:1])
    assert MO.cdi_emit_mdev(0, b"nvidia.com", ok) is None
    for u, p in [(UUIDS[3], b"0000:00:01.0"), (b"12345678-1234-1234-1234-12345678901", b"0000:00:01.0"),
                 (UUIDS[0], b"0000:00:01.0 "), (UUIDS[0], b"")]:
        assert MO.cdi_emit_mdev(1, b"nvidia.com/vgpu", devices([(u, 1, p, 0)])) is None


def test_mdev_names_oracle(workloads):
    recs = workloads.mdev_records(4096)
    idx = np.arange(0, 4096, 3, dtype=np.uint32)
    blob, offs = MO.mdev_names(recs, idx)
    for j, i in enumerate(idx):
        r = recs[i]
        name = bytes(r["type_name"][:min(r["name_len"], 40)])
        want = b"" if (r["flags"] & NAME_ERR) or r["name_len"] > 40 else P.type_key(name)
        assert blob[offs[j]:offs[j + 1]] == want


def test_workload_shape(workloads):
    recs = workloads.mdev_records(1 << 16)
    u = recs["uuid"]
    assert (u[:-1] < u[1:]).all() and all(P.uuid_ok(x) for x in u[:64])
    got = MO.classify_mdev(workloads.MDEV_RULES, recs)
    assert set(got["dev_rule"].tolist()) == set(range(len(workloads.MDEV_RULES)))
    assert 0.05 < (recs["flags"] != 0).mean() < 0.15
