"""CPU tests of the host's mdev walk (Plugin::gatherMdevRecords) on a fake /sys/bus/mdev/devices tree: the records
byte for byte, and the entries the walk records so that classify skips them."""
import numpy as np

import fake_mdev
import fake_sysfs
from oracle import mdev_oracle as mo

VGPU = [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia"),
        ("8086", "vfio_mdev", "intel.com", "intel.com/gvt", "cdi-mdev-intel")]
PARENTS = [dict(bdf="0000:3b:00.0", vendor=b"0x10de\n", device=b"0x1eb8\n", driver="nvidia", group=40),
           dict(bdf="0000:00:02.0", vendor=b"0x8086\n", device=b"0x3e92\n", driver="i915", group=1)]
U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(16)]
MDEVS = [dict(uuid=U[1], parent="0000:3b:00.0", group=300),
         dict(uuid=U[2], parent="0000:3b:00.0", group=301, type_id="nvidia-222x", name=b" GRID T4-1Q"),  # same key
         dict(uuid=U[3], parent="0000:3b:00.0", group=302, type_id="nvidia-223", name=b"GRID T4-2Q\n"),
         dict(uuid=U[4], parent="0000:00:02.0", group=310, type_id="i915-GVTg_V5_4", name=b"GVTg_V5_4\n"),
         dict(uuid=U[5], parent="0000:3b:00.0", group=None),                                  # no iommu_group link
         dict(uuid=U[6], parent="0000:3b:00.0", group=305, driver=None),                      # unbound
         dict(uuid=U[7], parent="0000:3b:00.0", group=306, mdev_type=False),                  # no mdev_type link
         dict(uuid=U[8], parent="0000:3b:00.0", group=307, type_id="long", name=b"N" * 41),    # 41-byte name
         dict(uuid="not-a-uuid", parent="0000:3b:00.0", group=308),                           # not a UUID
         dict(uuid=U[9], kind="dir")]                                                         # a directory entry
VENDOR = {"0000:3b:00.0": b"0x10de\n", "0000:00:02.0": b"0x8086\n"}


def make(tmp_path):
    fake_sysfs.make_tree(str(tmp_path), PARENTS)
    return fake_mdev.make_tree(str(tmp_path), MDEVS)


def test_gather_records_byte_for_byte(tmp_path):
    base = make(tmp_path)
    recs = fake_mdev.gather(base, VGPU)
    order = sorted(range(len(MDEVS)), key=lambda k: MDEVS[k]["uuid"])
    want = np.array([fake_mdev.expected_record(MDEVS[k], VENDOR.get(MDEVS[k].get("parent"), b"")) for k in order],
                    dtype=mo.MDEVREC_DTYPE)
    assert len(recs) == len(want)
    for k in range(len(want)):
        assert recs[k].tobytes() == want[k].tobytes(), MDEVS[order[k]]["uuid"]
    flags = {MDEVS[order[k]]["uuid"]: int(recs[k]["flags"]) for k in range(len(recs))}
    assert flags[U[5]] == 4 and flags[U[6]] == 2 and flags[U[7]] == 32 and flags[U[8]] == 32 and flags[U[9]] == 16


def test_skipped_entries_are_not_accepted(tmp_path):
    base = make(tmp_path)
    recs = fake_mdev.gather(base, VGPU)
    res = mo.classify_mdev([(v.encode(), d.encode()) for v, d, _, _, _ in VGPU], recs)
    accepted = sorted(recs["uuid"][res["accept_index"] != 0xFFFFFFFF].astype(str).tolist())
    assert accepted == U[1:5]
    assert res["group_ids"].tolist() == [300, 301, 302, 310]
    keys = mo.mdev_names(recs, res["dev_ids"])
    assert [keys[0][keys[1][d]:keys[1][d + 1]] for d in range(res["n_devids"])] == [b"GRID_T4-1Q", b"GRID_T4-2Q", b"GVTg_V5_4"]
