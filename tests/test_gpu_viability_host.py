"""GPU end to end of the host plugin's IOMMU group viability (Plugin::groupViability) on a fake sysfs with three groups:
a GPU whose HD-audio function is on snd_hda_intel (20), a GPU whose audio function is on vfio-pci (21), and a GPU behind
a pcieport bridge next to an unbound function (22)."""
import ctypes as C
import os

import numpy as np
import pytest

import fake_sysfs
import viab_host

pytestmark = pytest.mark.gpu

GPU = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
AUDIO = dict(vendor=b"0x10de\n", device=b"0x22a3\n")
DEVS = [dict(bdf="0000:01:00.0", group=20, **GPU), dict(bdf="0000:01:00.1", group=20, driver="snd_hda_intel", **AUDIO),
        dict(bdf="0000:02:00.0", group=21, **GPU), dict(bdf="0000:02:00.1", group=21, driver="vfio-pci", **AUDIO),
        dict(bdf="0000:03:00.0", group=22, **GPU),
        dict(bdf="0000:03:00.1", group=22, vendor=b"0x10b5\n", device=b"0xc010\n", driver="pcieport"),
        dict(bdf="0000:03:00.2", group=22, vendor=b"0x8086\n", device=b"0x1533\n")]
GROUPS = np.array([20, 21, 22], np.uint32)
WHY = "0000:01:00.1 is bound to snd_hda_intel"


def _tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = fake_sysfs.make_tree(root, DEVS)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _cdi(cdi):
    return {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}


def test_host_viability_end_to_end(tmp_path, kx, oracle, pci_text):
    root, base, pciids, cdi = _tree(tmp_path, pci_text)
    off = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    a = off.init("YAML")
    lw_off = off.list_and_watch(0)
    cdi_off = _cdi(cdi)
    assert lw_off == oracle.lw_encode(GROUPS, np.ones(3, np.uint8))
    assert viab_host.devs(off, 0) == {"20": ("Healthy", None), "21": ("Healthy", None), "22": ("Healthy", None)}
    assert off.allocate(["20"])["cdi_devices"] == ["nvidia.com/gpu=0"]
    off.close()

    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    viab_host.set_viability(hp, True)
    b = hp.init("YAML")
    for k in ("iommuMap", "deviceMap", "plugins", "cdiFile", "pciSnapshot"):
        assert a[k] == b[k], k  # the verdict lives beside Health: the state the plugin already computed is unchanged
    assert _cdi(cdi) == cdi_off
    assert viab_host.devs(hp, 0) == {"20": ("Healthy", WHY), "21": ("Healthy", None), "22": ("Healthy", None)}
    assert hp.list_and_watch(0) == oracle.lw_encode(GROUPS, np.array([0, 1, 1], np.uint8))
    with pytest.raises(RuntimeError, match="^invalid allocation request: IOMMU group 20 is not viable: " + WHY + "$"):
        hp.allocate(["20"])
    with pytest.raises(RuntimeError, match="IOMMU group 20 is not viable"):
        hp.allocate(["21", "20"])
    assert hp.allocate(["21"])["cdi_devices"] == ["nvidia.com/gpu=1", "nvidia.com/gpu=2"]
    assert hp.allocate(["22"])["cdi_devices"] == ["nvidia.com/gpu=3"]

    # /dev/vfio/20 going and coming back flips Health, never the verdict
    L = viab_host._lib()
    vfio = tmp_path / "vfio"
    vfio.mkdir()
    for g in GROUPS:
        (vfio / str(g)).write_text("")
    assert L.kxh_set_device_path(hp.h, 0, (str(vfio) + "/").encode()) == 0
    err = C.create_string_buffer(512)
    w = hp.L.kxh_health_start(hp.h, 0, 1, err, len(err))
    assert w, err.value
    try:
        os.remove(vfio / "20")
        assert hp.L.kxh_health_poll(w, 1000) == 1
        assert viab_host.devs(hp, 0)["20"] == ("Unhealthy", WHY)
        (vfio / "20").write_text("")
        assert hp.L.kxh_health_poll(w, 1000) == 1
        assert viab_host.devs(hp, 0)["20"] == ("Healthy", WHY)
        assert hp.list_and_watch(0) == oracle.lw_encode(GROUPS, np.array([0, 1, 1], np.uint8))
    finally:
        hp.L.kxh_health_stop(w)

    # the audio function moves to pci-stub (a bind uevent): the rediscovery finds the group viable
    link = os.path.join(root, "devices", "0000:01:00.1", "driver")
    os.remove(link)
    os.makedirs(os.path.join(root, "drivers", "pci-stub"), exist_ok=True)
    os.symlink(os.path.join(root, "drivers", "pci-stub"), link)
    r = viab_host.rediscover(hp)
    assert r["report"]["changed"] == [0] and r["report"]["added"] == []
    assert r["report"]["written"] == [] and _cdi(cdi) == cdi_off
    assert viab_host.devs(hp, 0) == {"20": ("Healthy", None), "21": ("Healthy", None), "22": ("Healthy", None)}
    assert hp.list_and_watch(0) == oracle.lw_encode(GROUPS, np.ones(3, np.uint8))
    assert hp.allocate(["20"])["cdi_devices"] == ["nvidia.com/gpu=0"]
    # and back to snd_hda_intel: unviable again, the plugin counts as changed again
    os.remove(link)
    os.symlink(os.path.join(root, "drivers", "snd_hda_intel"), link)
    r = viab_host.rediscover(hp)
    assert r["report"]["changed"] == [0]
    assert viab_host.devs(hp, 0)["20"] == ("Healthy", WHY)
    hp.close()


def test_host_viability_rebind_to_vfio_pci(tmp_path, kx, oracle, pci_text):
    """The audio function rebound to vfio-pci becomes a member of its group with a fresh index."""
    root, base, pciids, cdi = _tree(tmp_path, pci_text)
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    viab_host.set_viability(hp, True)
    hp.init("YAML")
    link = os.path.join(root, "devices", "0000:01:00.1", "driver")
    os.remove(link)
    os.symlink(os.path.join(root, "drivers", "vfio-pci"), link)
    r = viab_host.rediscover(hp)
    assert 0 in r["report"]["changed"]
    assert r["iommuMap"][0] == ["20", [["0000:01:00.0", 0], ["0000:01:00.1", 4]]]
    assert viab_host.devs(hp, 0)["20"] == ("Healthy", None)
    assert hp.list_and_watch(0) == oracle.lw_encode(GROUPS, np.ones(3, np.uint8))
    assert hp.allocate(["20"])["cdi_devices"] == ["nvidia.com/gpu=0", "nvidia.com/gpu=4"]
    hp.close()
