"""GPU end to end of the host's vGPU classes on a fake sysfs: a passthrough NVIDIA class next to an NVIDIA and an
Intel vGPU class.  The passthrough state must not change; the vGPU resources, CDI files, Allocate answers and
ListAndWatch bytes must equal what the oracles give for the gathered records."""
import ctypes as C
import os

import numpy as np
import pytest

import fake_mdev
import fake_sysfs
from oracle import mdev_oracle as mo
from oracle import xpu_oracle as xo
from test_mdev_host import MDEVS, PARENTS, VGPU

pytestmark = pytest.mark.gpu

PASSTHROUGH = [dict(bdf="0000:c1:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=214),
               dict(bdf="0000:c5:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=215)]


def expected(recs):
    """per vGPU class: the CDI devices (ascending index) and {group: [indices]} from the oracle's classify"""
    rules = [(v.encode(), d.encode()) for v, d, _, _, _ in VGPU]
    res = mo.classify_mdev(rules, recs)
    gclass = {}
    for d in range(res["n_devids"]):
        for g in res["dev_groups"][res["dev_off"][d]:res["dev_off"][d + 1]]:
            gclass[int(g)] = int(res["dev_rule"][d])
    per = [[] for _ in VGPU]
    groups = {}
    for i in np.nonzero(res["accept_index"] != 0xFFFFFFFF)[0]:
        g = int(recs["iommu_group"][i])
        per[gclass[g]].append((recs["uuid"][i], g, recs["parent"][i], int(res["accept_index"][i])))
        groups.setdefault(g, []).append(int(res["accept_index"][i]))
    devs = []
    for c in range(len(VGPU)):
        a = np.zeros(len(per[c]), mo.MDEVCDI_DTYPE)
        for k, t in enumerate(sorted(per[c], key=lambda t: t[3])):
            a[k] = t
        devs.append(a)
    return devs, groups, gclass


def test_host_flow_with_vgpu_classes(tmp_path, kx, pci_text, oracle):
    root = str(tmp_path)
    base = fake_sysfs.make_tree(root, PASSTHROUGH + PARENTS)
    mbase = fake_mdev.make_tree(root, MDEVS)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    # without vGPU classes: the passthrough state
    hp = fake_sysfs.HostPlugin(kx, base, str(tmp_path / "pci.ids"), str(cdi) + "/")
    a = hp.init("YAML")
    a_file = open(a["cdiFile"], "rb").read()
    assert a["mdevMap"] == [] and a["typeMap"] == [] and a["mdevCdiFiles"] == []
    hp.close()
    # with vGPU classes
    hp = fake_sysfs.HostPlugin(kx, base, str(tmp_path / "pci.ids"), str(cdi) + "/")
    fake_mdev.set_vgpu(hp, mbase, VGPU)
    b = hp.init("YAML")
    for k in ("iommuMap", "deviceMap", "cdiFile", "cdiFiles"):
        assert b[k] == a[k], k
    assert open(b["cdiFile"], "rb").read() == a_file
    npt = len(a["plugins"])
    assert b["plugins"][:npt] == a["plugins"]
    recs = fake_mdev.gather(mbase, VGPU)
    devs, groups, gclass = expected(recs)
    vg = b["plugins"][npt:]
    assert [(p["resource"], p["class"], p["vgpu"]) for p in vg] == [("nvidia.com/GRID_T4-1Q", 0, True), ("nvidia.com/GRID_T4-2Q", 0, True),
                                                                     ("intel.com/GVTg_V5_4", 1, True)]
    assert [p["devs"] for p in vg] == [[["300", "Healthy"], ["301", "Healthy"]], [["302", "Healthy"]], [["310", "Healthy"]]]
    assert [os.path.basename(f) for f in b["mdevCdiFiles"]] == ["cdi-mdev-nvidia.yaml", "cdi-mdev-intel.yaml"]
    for c, f in enumerate(b["mdevCdiFiles"]):
        assert open(f, "rb").read() == mo.cdi_emit_mdev(0, VGPU[c][3].encode(), devs[c])
    # Allocate: names and Envs of the group's class
    for g in (300, 302, 310):
        kind = VGPU[gclass[g]][3]
        blob, offs = xo.alloc_names_kind(kind.encode(), np.array(groups[g], np.uint64))
        names = [blob[offs[i]:offs[i + 1]].decode() for i in range(len(groups[g]))]
        assert hp.allocate([str(g)]) == {"envs": {"KUBERNETES_CDI_VENDOR_CLASS": kind}, "cdi_devices": names}
    assert hp.allocate(["214"])["envs"] == {"KUBERNETES_CDI_VENDOR_CLASS": "nvidia.com/gpu"}
    for mixed in (["214", "300"], ["300", "214"], ["300", "310"]):
        with pytest.raises(RuntimeError, match="invalid allocation request: devices of more than one class"):
            hp.allocate(mixed)
    # ListAndWatch bytes, then health flips on /dev/vfio/<group>
    for k, p in enumerate(vg):
        gids = np.array([int(d[0]) for d in p["devs"]], np.uint32)
        assert hp.list_and_watch(npt + k) == oracle.lw_encode(gids)
    vfio = tmp_path / "vfio"
    vfio.mkdir()
    for g in ("300", "301"):
        (vfio / g).write_text("")
    L = hp.L
    L.kxh_set_device_path.restype = C.c_int
    L.kxh_set_device_path.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    assert L.kxh_set_device_path(hp.h, npt, (str(vfio) + "/").encode()) == 0
    err = C.create_string_buffer(512)
    w = L.kxh_health_start(hp.h, npt, 0, err, len(err))
    assert w, err.value
    try:
        os.remove(vfio / "301")
        assert L.kxh_health_poll(w, 1000) == 1
        assert hp.list_and_watch(npt) == oracle.lw_encode(np.array([300, 301], np.uint32), np.array([1, 0], np.uint8))
    finally:
        L.kxh_health_stop(w)
    # an mdev moved to another IOMMU group: Allocate re-reads the link and fails
    link = os.path.join(mbase, MDEVS[2]["uuid"], "iommu_group")
    os.unlink(link)
    os.symlink(os.path.join(root, "iommu_groups", "999"), link)
    with pytest.raises(RuntimeError, match="invalid allocation request: unknown device: " + MDEVS[2]["uuid"]):
        hp.allocate(["302"])
    # JSON: the same files as .json
    st = hp.init("JSON")
    assert [os.path.basename(f) for f in st["mdevCdiFiles"]] == ["cdi-mdev-nvidia.json", "cdi-mdev-intel.json"]
    hp.close()


def test_vgpu_class_kind_or_stem_must_be_unique(tmp_path, kx, pci_text):
    root = str(tmp_path)
    base = fake_sysfs.make_tree(root, PASSTHROUGH)
    mbase = fake_mdev.make_tree(root, [])
    (tmp_path / "pci.ids").write_bytes(pci_text)
    for bad in ([("10de", "vfio_mdev", "nvidia.com", "nvidia.com/gpu", "cdi-mdev-nvidia")],
                [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-vfio-xxxx")],
                [VGPU[0], ("8086", "vfio_mdev", "intel.com", "intel.com/gvt", "cdi-mdev-nvidia")]):
        hp = fake_sysfs.HostPlugin(kx, base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
        fake_mdev.set_vgpu(hp, mbase, bad)
        with pytest.raises(RuntimeError, match="CDI kind and file stem must differ"):
            hp.init("YAML")
        hp.close()
