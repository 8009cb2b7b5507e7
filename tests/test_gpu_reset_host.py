"""GPU end to end of the host plugin's reset check (Plugin::resetCheck) on a fake sysfs tree: groups VFIO cannot reset
between tenants are sent Unhealthy with a reason naming the function, refused by Allocate and PrepareDraDevices and
left out of the CDI spec and the DRA pool; rediscover serves a group again once the function on its bus is rebound to
vfio-pci; with the setting off every output is the default plugin's and no reset file is opened."""
import os
import re

import numpy as np
import pytest

import dra_host as DH
import fake_sysfs
import pcie_host
import reset_host as H
import sriov_host
import viab_host

pytestmark = pytest.mark.gpu

DRIVERS = ["gpu.nvidia.com"]
GPU = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
AUDIO = dict(vendor=b"0x10de\n", device=b"0x22a3\n")
DEVS = [dict(bdf="0000:00:05.0", group=5, path="pci0000:00/0000:00:05.0", **GPU),                     # root bus
        dict(bdf="0000:41:00.0", group=41, path="pci0000:40/0000:40:01.0/0000:41:00.0", **GPU),       # audio on snd
        dict(bdf="0000:41:00.1", group=41, path="pci0000:40/0000:40:01.0/0000:41:00.1", driver="snd_hda_intel", **AUDIO),
        dict(bdf="0000:42:00.0", group=42, path="pci0000:42/0000:42:00.0", **GPU),                    # pm only
        dict(bdf="0000:61:00.0", group=61, path="pci0000:60/0000:60:01.0/0000:61:00.0", **GPU),       # FLR
        dict(bdf="0000:62:00.0", group=62, path="pci0000:60/0000:60:02.0/0000:62:00.0", **GPU),       # bus reset of
        dict(bdf="0000:62:00.1", group=62, path="pci0000:60/0000:60:02.0/0000:62:00.1", driver="vfio-pci", **AUDIO)]
METHODS = ["flr", "af_flr", "bus", "cxl_bus", "device_specific", "acpi"]  # pm left out
WHY = {"5": "0000:00:05.0 has no function reset and sits on a root bus",
       "41": "0000:41:00.0 has no function reset and 0000:41:00.1 on its bus is bound to snd_hda_intel",
       "42": "0000:42:00.0 has no reset method in resetMethods (reset_method: pm)"}
SERVED = ("61", "62")


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = pcie_host.make_nested_tree(root, DEVS, relative=True)
    H.set_method(base, "0000:42:00.0", b"pm\n")
    H.set_method(base, "0000:61:00.0", b"flr\n")
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, on):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, dra=DRIVERS)
    if on is not None:
        H.set_reset(hp, on, METHODS)
    return hp


def _outputs(hp, tree):
    cdi = tree[3]
    specs = {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}
    return specs, hp.list_and_watch(0), DH.slices(hp, 0)[0]


def _plugin_of(state, group):
    return [k for k, p in enumerate(state["plugins"]) for d in p["devs"] if d[0] == group][0]


def test_off_is_the_default_plugin(kx, tree):
    default = _plugin(kx, tree, None)
    try:
        default.init("YAML")
        want = _outputs(default, tree)
        gen = DH.generation(default)
    finally:
        default.close()
    for f in os.listdir(tree[3]):
        os.remove(os.path.join(tree[3], f))
    off = _plugin(kx, tree, False)
    try:
        state = off.init("YAML")
        assert H.reads(off) == 0
        assert _outputs(off, tree) == want and DH.generation(off) == gen
        assert all(d[1] == "Healthy" for p in state["plugins"] for d in p["devs"])
        assert viab_host.devs(off, 0) == {g: ("Healthy", None) for g in ("5", "41", "42", "61", "62")}
        assert off.allocate(["41"])["cdi_devices"]
    finally:
        off.close()


def test_reset_end_to_end(kx, tree):
    root, base = tree[0], tree[1]
    hp = _plugin(kx, tree, True)
    try:
        state = hp.init("YAML")
        assert H.reads(hp) == 10  # reset_method of the six candidates, and reset of the four without one
        devs = viab_host.devs(hp, 0)
        assert devs == dict({g: ("Healthy", WHY[g]) for g in WHY}, **{g: ("Healthy", None) for g in SERVED})
        ids = [d[0] for d in state["plugins"][0]["devs"]]
        want = kx.lw_encode(np.array([int(g) for g in ids], np.uint32), np.array([g in SERVED for g in ids], np.uint8))
        assert hp.list_and_watch(0) == want
        spec = open(os.path.join(tree[3], "cdi-vfio-xxxx.yaml"), "rb").read()
        blob = DH.slices(hp, 0)[0]
        for g in SERVED:
            assert b"/dev/vfio/%s\n" % g.encode() in spec and b'"name":"vfio%s"' % g.encode() in blob
        for g, why in WHY.items():
            assert b"/dev/vfio/%s\n" % g.encode() not in spec and b'"name":"vfio%s"' % g.encode() not in blob
            with pytest.raises(RuntimeError, match="IOMMU group %s is not viable: %s" % (g, re.escape(why))):
                hp.allocate([g])
            with pytest.raises(RuntimeError, match="not viable"):
                DH.prepare(hp, DRIVERS[0], "node-a", ["vfio" + g])
        for g in SERVED:
            assert hp.allocate([g])["cdi_devices"]
            assert DH.prepare(hp, DRIVERS[0], "node-a", ["vfio" + g])[0]
        reads = H.reads(hp)
        hp.allocate(["61"])
        assert H.reads(hp) == reads  # Allocate reads no reset file
        # the audio function rebound to vfio-pci: its bus-reset set is closed by group 41, which rediscover serves again
        gen = DH.generation(hp)
        sriov_host.rebind(root, base, "0000:41:00.1", "vfio-pci")
        r = viab_host.rediscover(hp)
        assert r["report"]["changed"] and DH.generation(hp) == gen + 1
        assert H.reads(hp) == reads + 12  # the walk again, and the audio function is a candidate now
        assert viab_host.devs(hp, 0)["41"] == ("Healthy", None)
        cdi = hp.allocate(["41"])["cdi_devices"]
        assert len(cdi) == 2
        assert b"/dev/vfio/41\n" in open(os.path.join(tree[3], "cdi-vfio-xxxx.yaml"), "rb").read()
        assert b'"name":"vfio41"' in DH.slices(hp, 0)[0]
        assert DH.prepare(hp, DRIVERS[0], "node-a", ["vfio41"])[0] == cdi
        # in another group instead: withheld again, naming it
        os.remove(os.path.join(os.path.realpath(os.path.join(base, "0000:41:00.1")), "iommu_group"))
        os.makedirs(os.path.join(root, "iommu_groups", "43"))
        os.symlink(os.path.join(root, "iommu_groups", "43"), os.path.join(os.path.realpath(os.path.join(base, "0000:41:00.1")), "iommu_group"))
        r = viab_host.rediscover(hp)
        devs = viab_host.devs(hp, 0)
        devs.update(viab_host.devs(hp, _plugin_of(r, "43")))  # the audio function's group is a plugin of its own
        assert devs["41"] == ("Healthy", "0000:41:00.0 has no function reset and 0000:41:00.1 on its bus is in IOMMU group 43")
        assert devs["43"] == ("Healthy", "0000:41:00.1 has no function reset and 0000:41:00.0 on its bus is in IOMMU group 41")
    finally:
        hp.close()
