"""CPU tests of the host gather under Plugin::groupViability (include/kxpu.h, ABI v8) on fake sysfs trees: which
records become blockers, that nothing more is read with the setting off, and that both gathers agree."""
import os

import numpy as np
import pytest

import fake_sysfs
import viab_host
from kxpu_b200.binding import DEVREC_DTYPE, REC_BLOCKS

AUDIO = dict(vendor=b"0x10de\n", device=b"0x22a3\n")
DEVS = [
    dict(bdf="0000:01:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=10),  # class candidate
    dict(bdf="0000:01:00.1", driver="snd_hda_intel", group=10, **AUDIO),                          # blocker
    dict(bdf="0000:02:00.0", vendor=b"0x8086\n", device=b"0x1533\n", driver=None, group=11),       # unbound
    dict(bdf="0000:03:00.0", vendor=b"0x10b5\n", device=b"0xc010\n", driver="pcieport", group=12),  # switch port
    dict(bdf="0000:04:00.0", vendor=b"0x8086\n", device=b"0x1533\n", driver="pci-stub", group=13),
    dict(bdf="0000:05:00.0", vendor=b"0x8086\n", device=b"0x1533\n", driver="vfio-pci", group=13),  # class driver, other vendor
    dict(bdf="0000:06:00.0", vendor=b"0x144d\n", device=b"0xa80a\n", driver="nvme", group=14),     # blocker
    dict(bdf="0000:07:00.0", vendor=b"0x144d\n", device=b"0xa80a\n", driver="nvme", group="012"),  # malformed group link
    dict(bdf="0000:08:00.0", vendor=None, device=None, driver="ixgbe", group=15),                 # vendor unreadable: blocker
    dict(bdf="0000:09:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver=None, group=16),      # class vendor, unbound
    dict(bdf="0000:0a:00.0", kind="dir"),
]


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return fake_sysfs.make_tree(str(tmp_path_factory.mktemp("viab")), DEVS)


def _blockers(recs):
    return {r["bdf"].decode(): (int(r["iommu_group"]), r["driver"].decode())
            for r in recs if int(r["flags"]) & REC_BLOCKS}


def test_setting_off_reads_nothing_more(tree):
    plain = fake_sysfs.gather(tree, DEVREC_DTYPE)
    recs, reads = viab_host.gather(tree, DEVREC_DTYPE, on=False, count=True)
    assert recs.tobytes() == plain.tobytes()
    assert reads == 0  # no driver or iommu_group read of an entry whose vendor no class has
    fast, _ = viab_host.gather(tree, DEVREC_DTYPE, on=False, fast=True)
    assert fast.tobytes() == plain.tobytes()
    _, reads_on = viab_host.gather(tree, DEVREC_DTYPE, on=True, count=True)
    assert reads_on > 0  # the counting seam sees the reads the setting adds


def test_blockers(tree):
    recs, _ = viab_host.gather(tree, DEVREC_DTYPE, on=True)
    assert _blockers(recs) == {"0000:01:00.1": (10, "snd_hda_intel"), "0000:06:00.0": (14, "nvme"),
                               "0000:08:00.0": (15, "ixgbe")}
    # nothing else moved: the records without the flag are the plain gather's
    plain = fake_sysfs.gather(tree, DEVREC_DTYPE)
    keep = (recs["flags"] & REC_BLOCKS) == 0
    assert recs[keep].tobytes() == plain[keep].tobytes()


def test_viability_drivers(tree):
    recs, _ = viab_host.gather(tree, DEVREC_DTYPE, on=True, drivers=["vfio-pci", "pci-stub", "pcieport", "snd_hda_intel"])
    assert set(_blockers(recs)) == {"0000:06:00.0", "0000:08:00.0"}
    # an empty list: pcieport and pci-stub block, the class driver vfio-pci still does not
    recs, _ = viab_host.gather(tree, DEVREC_DTYPE, on=True, drivers=[])
    assert set(_blockers(recs)) == {"0000:01:00.1", "0000:03:00.0", "0000:04:00.0", "0000:06:00.0", "0000:08:00.0"}


@pytest.mark.parametrize("drivers", [None, []])
def test_walk_equals_fast_gather(tree, drivers):
    walk, _ = viab_host.gather(tree, DEVREC_DTYPE, on=True, drivers=drivers)
    for threads in (1, 4):
        fast, _ = viab_host.gather(tree, DEVREC_DTYPE, on=True, drivers=drivers, fast=True, threads=threads)
        assert fast.tobytes() == walk.tobytes()


def test_many_entries_walk_equals_fast_gather(tmp_path):
    devs = []
    for i in range(300):
        kind = i % 5
        d = dict(bdf="0000:%02x:%02x.%d" % (i >> 8, (i >> 3) & 31, i & 7), group=i // 4)
        if kind == 0:
            d.update(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
        elif kind == 1:
            d.update(driver="snd_hda_intel", **AUDIO)
        elif kind == 2:
            d.update(vendor=b"0x10b5\n", device=b"0xc010\n", driver="pcieport")
        elif kind == 3:
            d.update(vendor=b"0x144d\n", device=b"0xa80a\n", driver="nvme")
        else:
            d.update(vendor=b"0x8086\n", device=b"0x1533\n")
        devs.append(d)
    base = fake_sysfs.make_tree(str(tmp_path), devs)
    walk, _ = viab_host.gather(base, DEVREC_DTYPE, on=True)
    fast, _ = viab_host.gather(base, DEVREC_DTYPE, on=True, fast=True, threads=4)
    assert fast.tobytes() == walk.tobytes()
    assert len(_blockers(walk)) == 120
    assert os.path.isdir(base)
    assert (walk["flags"][np.arange(300) % 5 == 1] & REC_BLOCKS).all()
