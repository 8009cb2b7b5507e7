"""GPU end to end of the host plugin's DRA device taints (Plugin::draTaints, refreshDraHealth) on a fake sysfs and a fake
/dev/vfio watched by a running HealthWatcher: a removed device node taints its group at the clock seam's time with one
generation step, the time stays while the group stays unhealthy and across a rediscovery, a recreated node clears it,
PrepareDraDevices refuses the tainted group, a blocked group stays out of the slices, the same flow for a vGPU pool,
and with draTaints off an unhealthy device changes neither the slices nor a generation."""
import ctypes as C
import os

import numpy as np
import pytest

import dra_host as DH
import dra_mdev_host as MH
import fake_mdev
import fake_sysfs
import pcie_host
from oracle import dra_oracle as DO
from oracle import dra_taint_oracle as TO
from test_gpu_dra_host import CLASSES, DEVS, DRIVERS
from test_gpu_dra_mdev_host import MDEVS, PARENTS, VDRV, VGPU, _model_name

pytestmark = pytest.mark.gpu

VALUE, EFFECT = "vfio-device-missing", "NoSchedule"
T0 = 1767225600  # 2026-01-01T00:00:00Z


def _lib():
    L = fake_sysfs.host_lib()
    L.kxh_set_dra_taints.argtypes = [C.c_void_p, C.c_int]
    L.kxh_set_clock.argtypes = [C.c_void_p, C.c_void_p]
    L.kxh_refresh_dra_health.restype = C.c_int
    L.kxh_refresh_dra_health.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_char_p, C.c_size_t]
    L.kxh_set_device_path.restype = C.c_int
    L.kxh_set_device_path.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    return L


def refresh(hp):
    """refreshDraHealth: (passthrough pools moved, vGPU pools moved)"""
    moved, err = C.c_int(-1), C.create_string_buffer(512)
    assert _lib().kxh_refresh_dra_health(hp.h, C.byref(moved), err, len(err)) == 0, err.value
    return bool(moved.value & 1), bool(moved.value & 2)


class Watched:
    """a HealthWatcher (watching creates too) on plugin `idx`, whose devicePath is a fake /dev/vfio holding a file per
    device of the plugin"""

    def __init__(self, hp, tmp_path, idx, groups):
        self.hp, self.dir = hp, tmp_path / "vfio"
        self.dir.mkdir()
        for g in groups:
            (self.dir / g).write_text("")
        L = _lib()
        assert L.kxh_set_device_path(hp.h, idx, (str(self.dir) + "/").encode()) == 0
        err = C.create_string_buffer(512)
        self.w = L.kxh_health_start(hp.h, idx, 1, err, len(err))
        assert self.w, err.value

    def remove(self, g):
        os.remove(self.dir / g)
        assert _lib().kxh_health_poll(self.w, 1000) == 1

    def create(self, g):
        (self.dir / g).write_text("")
        assert _lib().kxh_health_poll(self.w, 1000) == 1

    def stop(self):
        _lib().kxh_health_stop(self.w)


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = pcie_host.make_nested_tree(root, DEVS, relative=True)
    DH.add_numa(root, DEVS)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, clock, taints=True):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, classes=CLASSES, dra=DRIVERS, viability=True)
    _lib().kxh_set_dra_taints(hp.h, int(taints))
    _lib().kxh_set_clock(hp.h, clock.ctypes.data)
    return hp


def _served(state, group):
    return [k for k, p in enumerate(state["plugins"]) if any(d[0] == group for d in p["devs"])][0]


def _want(state, gen, taint):
    """the taint oracle's slices of the NVIDIA pool; taint: group -> time.  Group 20 has a blocker: never published."""
    recs = DH.expected_records(state, DEVS, 0)
    recs = recs[recs["iommu_group"] != 20]
    since = np.array([taint.get(str(g), -1) for g in recs["iommu_group"]], np.int64)
    return TO.dra_slices_taint(DRIVERS[0], "node-a", "node-a", gen, recs, DRIVERS[0] + "/unhealthy", VALUE, EFFECT, since)


def test_passthrough_taint_flow(kx, tree, tmp_path):
    clock = np.array([T0], np.int64)
    hp = _plugin(kx, tree, clock)
    try:
        state = hp.init("YAML")
        idx = _served(state, "214")
        w = Watched(hp, tmp_path, idx, [d[0] for d in state["plugins"][idx]["devs"]])
        blob, offs = DH.slices(hp, 0)
        want, woffs = _want(state, 1, {})
        assert blob == want and np.array_equal(offs, woffs)
        assert b"taints" not in blob and b'"name":"vfio20"' not in blob
        assert refresh(hp) == (False, False) and DH.generation(hp) == 1  # nothing unhealthy yet

        w.remove("214")
        assert refresh(hp) == (True, False) and DH.generation(hp) == 2
        blob, offs = DH.slices(hp, 0)
        want, woffs = _want(state, 2, {"214": T0})
        assert blob == want and np.array_equal(offs, woffs)
        assert b'"taints":[{"key":"vfio.nvidia.com/unhealthy","value":"vfio-device-missing","effect":"NoSchedule",' \
               b'"timeAdded":"2026-01-01T00:00:00Z"}]' in blob
        assert b'"generation":2' in DH.slices(hp, 1)[0]  # one generation for every passthrough pool

        clock[0] = T0 + 3600  # a refresh with nothing new: same generation, same bytes, the time kept
        assert refresh(hp) == (False, False) and DH.generation(hp) == 2
        assert DH.slices(hp, 0)[0] == blob

        with pytest.raises(RuntimeError, match="PrepareDraDevices: device vfio214 is tainted vfio.nvidia.com/unhealthy="
                                               "vfio-device-missing:NoSchedule"):
            DH.prepare(hp, DRIVERS[0], "node-a", ["vfio40", "vfio214"])
        assert DH.prepare(hp, DRIVERS[0], "node-a", ["vfio40"]) == [hp.allocate(["40"])["cdi_devices"]]

        state = DH.rediscover(hp)  # nothing moved in sysfs: health and the taint time carry over
        assert DH.generation(hp) == 2 and DH.slices(hp, 0)[0] == blob

        w.remove("20")  # a blocked group turning unhealthy: not published, so no taint and no new generation
        assert refresh(hp) == (False, False) and DH.generation(hp) == 2
        assert b'"name":"vfio20"' not in DH.slices(hp, 0)[0]

        w.create("214")
        clock[0] = T0 + 7200
        assert refresh(hp) == (True, False) and DH.generation(hp) == 3
        blob, offs = DH.slices(hp, 0)
        want, woffs = _want(state, 3, {})
        assert blob == want and np.array_equal(offs, woffs) and b"taints" not in blob
        assert DH.prepare(hp, DRIVERS[0], "node-a", ["vfio214"]) == [hp.allocate(["214"])["cdi_devices"]]

        w.remove("214")  # turning unhealthy again takes the time of now
        assert refresh(hp) == (True, False) and DH.generation(hp) == 4
        assert DH.slices(hp, 0)[0] == _want(state, 4, {"214": T0 + 7200})[0]
        w.stop()
    finally:
        hp.close()


def test_rediscover_keeps_surviving_and_drops_leaving(kx, tree, tmp_path):
    clock = np.array([T0], np.int64)
    base = tree[1]
    hp = _plugin(kx, tree, clock)
    try:
        state = hp.init("YAML")
        idx = _served(state, "214")
        w = Watched(hp, tmp_path, idx, [d[0] for d in state["plugins"][idx]["devs"]])
        w.remove("214")
        w.remove("40")
        assert refresh(hp) == (True, False) and DH.generation(hp) == 2
        os.remove(os.path.join(base, "0000:41:00.0"))  # group 40 leaves
        clock[0] = T0 + 60
        state = DH.rediscover(hp)
        assert DH.generation(hp) == 3
        blob, offs = DH.slices(hp, 0)
        devs = [d for d in DEVS if d["bdf"] != "0000:41:00.0"]
        recs = DH.expected_records(state, devs, 0)
        recs = recs[recs["iommu_group"] != 20]
        since = np.where(recs["iommu_group"] == 214, T0, -1).astype(np.int64)
        want, woffs = TO.dra_slices_taint(DRIVERS[0], "node-a", "node-a", 3, recs, DRIVERS[0] + "/unhealthy", VALUE, EFFECT,
                                          since)
        assert blob == want and np.array_equal(offs, woffs) and b'"name":"vfio40"' not in blob
        assert refresh(hp) == (False, False) and DH.generation(hp) == 3  # group 214's time survived, 40's is gone
        w.stop()
    finally:
        hp.close()


def test_off_changes_nothing(kx, tree, tmp_path):
    """draTaints off (the default): an unhealthy device moves neither the slices nor either generation, and prepare
    still answers"""
    clock = np.array([T0], np.int64)
    hp = _plugin(kx, tree, clock, taints=False)
    try:
        state = hp.init("YAML")
        before = [DH.slices(hp, c) for c in (0, 1)]
        idx = _served(state, "214")
        w = Watched(hp, tmp_path, idx, [d[0] for d in state["plugins"][idx]["devs"]])
        w.remove("214")
        assert refresh(hp) == (False, False)
        assert DH.generation(hp) == 1 and MH.generation(hp) == 1
        after = [DH.slices(hp, c) for c in (0, 1)]
        for (b0, o0), (b1, o1) in zip(before, after):
            assert b0 == b1 and np.array_equal(o0, o1)
        recs = DH.expected_records(state, DEVS, 0)
        assert before[0][0] == DO.dra_slices(DRIVERS[0], "node-a", "node-a", 1, recs[recs["iommu_group"] != 20])[0]
        assert DH.prepare(hp, DRIVERS[0], "node-a", ["vfio214"]) == [hp.allocate(["214"])["cdi_devices"]]
        w.stop()
    finally:
        hp.close()


@pytest.fixture
def mdev_tree(tmp_path, pci_text):
    root = str(tmp_path)
    base, mbase = MH.make_tree(root, PARENTS, MDEVS)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, mbase, str(tmp_path / "pci.ids"), str(cdi) + "/"


def test_vgpu_taint_flow(kx, mdev_tree, tmp_path, oracle, pci_text):
    root, base, mbase, pciids, cdi = mdev_tree
    clock = np.array([T0], np.int64)
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    try:
        DH.configure(hp, node="node-a")
        fake_mdev.set_vgpu(hp, mbase, VGPU)
        MH.set_vgpu_dra(hp, [VDRV])
        _lib().kxh_set_dra_taints(hp.h, 1)
        _lib().kxh_set_clock(hp.h, clock.ctypes.data)
        state = hp.init("YAML")
        idx = _served(state, "300")
        assert state["plugins"][idx]["vgpu"]
        w = Watched(hp, tmp_path, idx, [d[0] for d in state["plugins"][idx]["devs"]])
        recs = MH.expected_records(state, PARENTS, 0, _model_name(oracle, pci_text))

        def want(gen, taint):
            since = np.array([taint.get(str(g), -1) for g in recs["iommu_group"]], np.int64)
            return TO.dra_slices_mdev_taint(VDRV, "node-a", "node-a", gen, recs, VDRV + "/unhealthy", VALUE, EFFECT, since)

        assert MH.slices(hp, 0)[0] == want(1, {})[0]
        w.remove("300")
        assert refresh(hp) == (False, True) and MH.generation(hp) == 2 and DH.generation(hp) == 1
        blob, offs = MH.slices(hp, 0)
        wb, wo = want(2, {"300": T0})
        assert blob == wb and np.array_equal(offs, wo) and b'"timeAdded":"2026-01-01T00:00:00Z"' in blob
        clock[0] = T0 + 5
        assert refresh(hp) == (False, False) and MH.slices(hp, 0)[0] == blob
        with pytest.raises(RuntimeError, match="device vfio300 is tainted vgpu.nvidia.com/unhealthy"):
            DH.prepare(hp, VDRV, "node-a", ["vfio300"])
        w.create("300")
        assert refresh(hp) == (False, True) and MH.generation(hp) == 3
        assert MH.slices(hp, 0)[0] == want(3, {})[0]
        assert DH.prepare(hp, VDRV, "node-a", ["vfio300"]) == [hp.allocate(["300"])["cdi_devices"]]
        w.stop()
    finally:
        hp.close()
