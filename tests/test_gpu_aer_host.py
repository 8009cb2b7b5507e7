"""GPU end to end of the host plugin's PCIe AER health (Plugin::aerHealth, refreshAerHealth) on the fake sysfs trees
with AER files written into them: counts over and under the limits, a non-fatal to fatal flip that re-times the taint
with one generation step, the vfio-device-missing and AER taints on one device in table order, PrepareDraDevices
allowed for an AER taint and refused for vfio-device-missing, a rediscover after the counters reset, a vGPU pool
tainted through its parent's files, unknown files that do not taint, and aerHealth off reading nothing."""
import os

import numpy as np
import pytest

import aer_cases as AC
import aer_host as AH
import dra_host as DH
import dra_mdev_host as MH
import fake_mdev
import fake_sysfs
from oracle import aer_oracle as AO
from oracle import dra_taint_oracle as TO
from test_gpu_dra_host import CLASSES, DEVS, DRIVERS
from test_gpu_dra_mdev_host import MDEVS, PARENTS, VDRV, VGPU, _model_name
from test_gpu_dra_taint_host import T0, Watched, mdev_tree, refresh as refresh_dra, tree  # noqa: F401

import test_gpu_dra_taint_host as TH

pytestmark = pytest.mark.gpu


def table(driver):
    return [(driver + "/unhealthy", "vfio-device-missing", "NoSchedule"), (driver + "/pcie-aer", "fatal", "NoSchedule"),
            (driver + "/pcie-aer", "nonfatal", "NoSchedule")]


def _plugin(kx, tree, clock, aer=True, limits=(0, 0)):
    root, base, pciids, cdi = tree
    for d in DEVS:
        AH.write(os.path.join(base, d["bdf"]))
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, classes=CLASSES, dra=DRIVERS, viability=True)
    TH._lib().kxh_set_dra_taints(hp.h, 1)
    TH._lib().kxh_set_clock(hp.h, clock.ctypes.data)
    AH.enable(hp, aer, *limits)
    return hp


def _want(state, gen, rows):
    """the oracle's slices of the NVIDIA pool; rows: group -> [missing, fatal, nonfatal] times"""
    recs = DH.expected_records(state, DEVS, 0)
    recs = recs[recs["iommu_group"] != 20]
    since = np.array([rows.get(str(g), [-1, -1, -1]) for g in recs["iommu_group"]], np.int64)
    return AO.dra_slices_taints(DRIVERS[0], "node-a", "node-a", gen, recs, table(DRIVERS[0]), since)


def test_passthrough_aer_flow(kx, tree, tmp_path):
    clock = np.array([T0], np.int64)
    base = tree[1]
    hp = _plugin(kx, tree, clock, limits=(0, 2))
    try:
        AH.write(os.path.join(base, "0000:c1:00.1"), nonfatal=3)  # the second member of group 214, over the limit 2
        AH.write(os.path.join(base, "0000:41:00.0"), nonfatal=2)  # group 40: at the limit, healthy
        state = hp.init("YAML")
        idx = TH._served(state, "214")
        assert AH.reasons(hp, idx)["214"] == "0000:c1:00.1 reported 3 non-fatal uncorrectable PCIe errors (limit 2)"
        assert AH.health(hp, idx)["214"] == "Unhealthy"
        assert AH.health(hp, TH._served(state, "40"))["40"] == "Healthy"
        blob, offs = DH.slices(hp, 0)
        want, woffs = _want(state, 1, {"214": [-1, -1, T0]})
        assert blob == want and np.array_equal(offs, woffs) and DH.generation(hp) == 1
        assert AH.refresh(hp) == ([], False, False)  # nothing new

        AH.write(os.path.join(base, "0000:c1:00.0"), fatal=2)  # non-fatal to fatal: a new value and a new time
        clock[0] = T0 + 60
        assert AH.refresh(hp) == ([], True, False) and DH.generation(hp) == 2  # still Unhealthy: same ListAndWatch
        assert AH.reasons(hp, idx)["214"] == "0000:c1:00.0 reported 2 fatal uncorrectable PCIe errors (limit 0)"
        assert DH.slices(hp, 0)[0] == _want(state, 2, {"214": [-1, T0 + 60, -1]})[0]
        # an AER taint does not stop a claim that tolerates it, nor Allocate
        assert DH.prepare(hp, DRIVERS[0], "node-a", ["vfio214"]) == [hp.allocate(["214"])["cdi_devices"]]

        w = Watched(hp, tmp_path, idx, [d[0] for d in state["plugins"][idx]["devs"]])
        clock[0] = T0 + 120
        w.remove("214")  # the device node goes too: both taints, in table order
        assert refresh_dra(hp) == (True, False) and DH.generation(hp) == 3
        blob = DH.slices(hp, 0)[0]
        assert blob == _want(state, 3, {"214": [T0 + 120, T0 + 60, -1]})[0]
        assert blob.index(b'"vfio.nvidia.com/unhealthy"') < blob.index(b'"vfio.nvidia.com/pcie-aer"')
        with pytest.raises(RuntimeError, match="device vfio214 is tainted vfio.nvidia.com/unhealthy"):
            DH.prepare(hp, DRIVERS[0], "node-a", ["vfio214"])
        w.create("214")
        assert refresh_dra(hp) == (True, False) and DH.generation(hp) == 4

        # the function was re-enumerated: zeroed counters clear the taint at the next rediscover, one generation step
        AH.write(os.path.join(base, "0000:c1:00.0"))
        AH.write(os.path.join(base, "0000:c1:00.1"))
        state = DH.rediscover(hp)
        assert DH.generation(hp) == 5 and AH.reasons(hp, idx)["214"] == ""
        assert DH.slices(hp, 0)[0] == _want(state, 5, {})[0]
        assert AH.health(hp, idx)["214"] == "Healthy"
        assert AH.refresh(hp) == ([], False, False)
        w.stop()
    finally:
        hp.close()


def test_refresh_reports_listandwatch_changes(kx, tree):
    clock = np.array([T0], np.int64)
    base = tree[1]
    hp = _plugin(kx, tree, clock, limits=(5, 5))
    try:
        state = hp.init("YAML")
        idx = TH._served(state, "80")
        AH.write(os.path.join(base, "0000:81:00.0"), fatal=6)
        assert AH.refresh(hp) == ([idx], True, False) and DH.generation(hp) == 2
        assert AH.health(hp, idx)["80"] == "Unhealthy"
        AH.write(os.path.join(base, "0000:81:00.0"), fatal=5)  # back at the limit
        assert AH.refresh(hp) == ([idx], True, False) and DH.generation(hp) == 3
        assert DH.slices(hp, 0)[0] == _want(state, 3, {})[0]
    finally:
        hp.close()


def test_unknown_files_do_not_taint(kx, tree):
    clock = np.array([T0], np.int64)
    base = tree[1]
    hp = _plugin(kx, tree, clock)
    try:
        AH.write_raw(os.path.join(base, "0000:41:00.0"), b"TOTAL_ERR_FATAL 007\n", b"TOTAL_ERR_NONFATAL 3\r\n")
        os.remove(os.path.join(base, "0000:81:00.0", "aer_dev_fatal"))  # no AER capability
        os.remove(os.path.join(base, "0000:81:00.0", "aer_dev_nonfatal"))
        AH.write_raw(os.path.join(base, "0000:c1:00.0"), AC._pad_to(AC.F, 4097, 9), AC._pad_to(AC.N, 4097, 9))
        state = hp.init("YAML")
        for g in ("40", "80", "214"):
            assert AH.reasons(hp, TH._served(state, g))[g] == ""
        assert DH.slices(hp, 0)[0] == _want(state, 1, {})[0]
        assert AH.reads(hp) > 0
    finally:
        hp.close()


def test_off_reads_nothing(kx, tree):
    clock = np.array([T0], np.int64)
    base = tree[1]
    hp = _plugin(kx, tree, clock, aer=False)
    try:
        AH.write(os.path.join(base, "0000:c1:00.0"), fatal=9, nonfatal=9)
        state = hp.init("YAML")
        idx = TH._served(state, "214")
        assert AH.health(hp, idx)["214"] == "Healthy" and AH.reasons(hp, idx)["214"] == ""
        recs = DH.expected_records(state, DEVS, 0)
        recs = recs[recs["iommu_group"] != 20]
        want = TO.dra_slices_taint(DRIVERS[0], "node-a", "node-a", 1, recs, DRIVERS[0] + "/unhealthy",
                                   "vfio-device-missing", "NoSchedule", np.full(len(recs), -1, np.int64))
        assert DH.slices(hp, 0)[0] == want[0]
        assert AH.refresh(hp) == ([], False, False)
        DH.rediscover(hp)
        assert AH.reads(hp) == 0 and DH.generation(hp) == 1
    finally:
        hp.close()


def test_vgpu_pool_through_parent_files(kx, mdev_tree, oracle, pci_text):  # noqa: F811
    root, base, mbase, pciids, cdi = mdev_tree
    clock = np.array([T0], np.int64)
    for p in PARENTS:
        if os.path.isdir(os.path.join(base, p["bdf"])):
            AH.write(os.path.join(base, p["bdf"]), fatal=1 if p["bdf"] == "0000:c1:00.0" else 0)
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    try:
        DH.configure(hp, node="node-a")
        fake_mdev.set_vgpu(hp, mbase, VGPU)
        MH.set_vgpu_dra(hp, [VDRV])
        TH._lib().kxh_set_dra_taints(hp.h, 1)
        TH._lib().kxh_set_clock(hp.h, clock.ctypes.data)
        AH.enable(hp)
        state = hp.init("YAML")
        recs = MH.expected_records(state, PARENTS, 0, _model_name(oracle, pci_text))
        parent_of = {str(m["group"]): m["parent"] for m in MDEVS}
        rows = {g: [-1, T0, -1] for g, par in parent_of.items() if par == "0000:c1:00.0"}
        since = np.array([rows.get(str(g), [-1, -1, -1]) for g in recs["iommu_group"]], np.int64)
        want = AO.dra_slices_mdev_taints(VDRV, "node-a", "node-a", 1, recs, table(VDRV), since)
        assert MH.slices(hp, 0)[0] == want[0]
        idx = TH._served(state, "300")
        assert AH.reasons(hp, idx)["300"] == "0000:c1:00.0 reported 1 fatal uncorrectable PCIe errors (limit 0)"
        assert DH.prepare(hp, VDRV, "node-a", ["vfio300"]) == [hp.allocate(["300"])["cdi_devices"]]
        AH.write(os.path.join(base, "0000:c1:00.0"))
        assert AH.refresh(hp)[1:] == (False, True) and MH.generation(hp) == 2 and DH.generation(hp) == 1
        assert b"taints" not in MH.slices(hp, 0)[0]
    finally:
        hp.close()
