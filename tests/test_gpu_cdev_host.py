"""GPU end to end of the host plugin with one class served through VFIO cdevs (XpuClass::vfioCdev) and one through group
nodes, on a fake sysfs: the specs, a group with a member without a cdev, Allocate live and from the snapshot, a swap of
cdev numbers across rediscover, the health watcher on cdev nodes, and a restart with resumeIndices and the setting
switched."""
import ctypes as C
import os

import numpy as np
import pytest

import cdev_host as H
import fake_sysfs
import pyref_cdev as PC
import viab_host
from kxpu_b200.binding import CDIDEV_DTYPE

pytestmark = pytest.mark.gpu

NVD = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
AMD = ("1002", "vfio-pci", "amd.com", "amd.com/gpu", "cdi-amd")
DEVS = [dict(bdf="0000:01:00.0", group=40, **NVD),
        dict(bdf="0000:01:00.1", group=40, vendor=b"0x10de\n", device=b"0x22a3\n", driver="vfio-pci"),
        dict(bdf="0000:02:00.0", group=41, **NVD),
        dict(bdf="0000:03:00.0", group=42, **NVD),  # no vfio-dev/: no cdev
        dict(bdf="0000:81:00.0", group=50, vendor=b"0x1002\n", device=b"0x740f\n", driver="vfio-pci")]
CDEVS = {"0000:01:00.0": 3, "0000:01:00.1": 4, "0000:02:00.0": 5, "0000:81:00.0": 6}
WHY = "0000:03:00.0 has no VFIO cdev"


def _spec(recs):
    a = np.zeros(len(recs), CDIDEV_DTYPE)
    for i, (bdf, g, idx, n) in enumerate(recs):
        a[i]["bdf"], a[i]["iommu_group"], a[i]["index"], a[i][PC.CDEV_FIELD] = bdf.encode(), g, idx, n
    return PC.emit(PC.FMT_YAML, b"nvidia.com/gpu", a)


def _plugin(kx, base, pciids, cdi, cdev, gen=None, resume=False):
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    hp.L.kxh_set_classes.argtypes = [C.c_void_p, C.c_char_p]
    assert hp.L.kxh_set_classes(hp.h, H.spec([H.NV_CDEV if cdev else H.NV, AMD])) == 0
    if gen is not None:
        hp.L.kxh_snapshot_enable.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        hp.L.kxh_snapshot_enable(hp.h, gen.ctypes.data, None)
    if resume:
        hp.L.kxh_set_resume.argtypes = [C.c_void_p, C.c_int]
        hp.L.kxh_set_resume(hp.h, 1)
    return hp


def test_cdev_class_end_to_end(tmp_path, kx, pci_text):
    root = str(tmp_path)
    base = fake_sysfs.make_tree(root, DEVS)
    for bdf, n in CDEVS.items():
        H.set_vfio_dev(base, bdf, ["vfio%d" % n])
    (tmp_path / "pci.ids").write_bytes(pci_text)
    pciids = str(tmp_path / "pci.ids")
    cdi = str(tmp_path / "cdi") + "/"
    os.makedirs(cdi)
    nv_file, amd_file = cdi + "cdi-vfio-xxxx.yaml", cdi + "cdi-amd.yaml"

    # group mode for both classes: nothing under vfio-dev/ is read
    off = _plugin(kx, base, pciids, cdi, False)
    a = off.init()
    assert H.cdev_reads(off) == 0
    amd_group_doc, nv_group_doc = open(amd_file, "rb").read(), open(nv_file, "rb").read()
    assert b"/dev/vfio/40\n" in nv_group_doc
    off.close()

    gen = np.array([1], np.uint64)
    hp = _plugin(kx, base, pciids, cdi, True, gen)
    b = hp.init()
    assert H.cdev_reads(hp) == 4  # the four functions of the cdev class
    assert a["pciSnapshot"] == b["pciSnapshot"] and a["iommuMap"] == b["iommuMap"]
    # the cdev spec names each function's node and leaves out group 42; the group-mode file is unchanged
    assert open(nv_file, "rb").read() == _spec([("0000:01:00.0", 40, 0, 3), ("0000:01:00.1", 40, 1, 4), ("0000:02:00.0", 41, 2, 5)])
    assert open(amd_file, "rb").read() == amd_group_doc
    # group 42: Unhealthy with its reason, refused
    assert viab_host.devs(hp, 0) == {"40": ("Healthy", None), "41": ("Healthy", None), "42": ("Healthy", WHY)}
    nodes = H.plugin_nodes(hp, 0)
    assert nodes["path"] == "/dev/vfio/devices/" and nodes["nodes"] == {"40": ["vfio3", "vfio4"], "41": ["vfio5"], "42": []}
    assert H.plugin_nodes(hp, 1)["path"] == "/dev/vfio/" and H.plugin_nodes(hp, 1)["nodes"] == {}
    with pytest.raises(RuntimeError, match="IOMMU group 42 is not viable: " + WHY):
        hp.allocate(["42"])
    assert hp.allocate(["40"])["cdi_devices"] == ["nvidia.com/gpu=0", "nvidia.com/gpu=1"]

    # a changed cdev: the snapshot still answers while the generation stands, the live path refuses
    H.set_vfio_dev(base, "0000:02:00.0", ["vfio9"])
    assert hp.allocate(["41"])["cdi_devices"] == ["nvidia.com/gpu=2"]
    gen[0] = 2
    with pytest.raises(RuntimeError, match="the VFIO cdev of 0000:02:00.0 changed since discovery"):
        hp.allocate(["41"])

    # health: the watcher watches every member's node
    dev = tmp_path / "vfio_nodes"
    dev.mkdir()
    for n in (3, 4, 5, 9):
        (dev / ("vfio%d" % n)).write_bytes(b"")
    hp.L.kxh_set_device_path.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    assert hp.L.kxh_set_device_path(hp.h, 0, str(dev).encode()) == 0
    err = C.create_string_buffer(512)
    w = hp.L.kxh_health_start(hp.h, 0, 0, err, len(err))
    assert w, err.value
    try:
        # 0000:01:00.0 and 0000:02:00.0 swap numbers across a re-bind
        H.set_vfio_dev(base, "0000:01:00.0", ["vfio5"])
        H.set_vfio_dev(base, "0000:02:00.0", ["vfio3"])
        gen[0] = 3
        r = viab_host.rediscover(hp)
        assert r["pciSnapshot"] == b["pciSnapshot"]  # every index kept
        assert 0 in r["report"]["changed"] and nv_file in r["report"]["written"] and amd_file not in r["report"]["written"]
        assert open(nv_file, "rb").read() == _spec([("0000:01:00.0", 40, 0, 5), ("0000:01:00.1", 40, 1, 4),
                                                     ("0000:02:00.0", 41, 2, 3)])
        assert H.plugin_nodes(hp, 0)["nodes"]["40"] == ["vfio5", "vfio4"]
        hp.L.kxh_health_resync.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        assert hp.L.kxh_health_resync(w, err, len(err)) == 0, err.value
        assert hp.allocate(["41"])["cdi_devices"] == ["nvidia.com/gpu=2"]  # the live read matches the new walk
        os.remove(dev / "vfio4")  # a member of group 40
        assert hp.L.kxh_health_poll(w, 1000) >= 1
        assert viab_host.devs(hp, 0)["40"][0] == "Unhealthy" and viab_host.devs(hp, 0)["41"][0] == "Healthy"
    finally:
        hp.L.kxh_health_stop(w)
    snap = r["pciSnapshot"]
    hp.close()

    # restart with resumeIndices and the setting switched off: the cdev spec is read with the other layout
    H.set_vfio_dev(base, "0000:01:00.0", None)
    back = _plugin(kx, base, pciids, cdi, False, resume=True)
    c = back.init()
    # every function the cdev spec named keeps its index; group 42, which it left out, gets one above all of them
    assert [s[4] for s in snap] == [0, 1, 2, 3, 4]
    assert [s[4] for s in c["pciSnapshot"]] == [0, 1, 2, 5, 4]
    doc = open(nv_file, "rb").read()
    assert b"/dev/vfio/42\n" in doc and b"/dev/vfio/devices/" not in doc
    back.close()
    # and on again: the group-mode spec is read with the other layout
    H.set_vfio_dev(base, "0000:01:00.0", ["vfio5"])
    on = _plugin(kx, base, pciids, cdi, True, resume=True)
    d = on.init()
    assert [s[4] for s in d["pciSnapshot"]] == [0, 1, 2, 5, 4]
    assert b"/dev/vfio/devices/vfio5\n" in open(nv_file, "rb").read()
    on.close()
