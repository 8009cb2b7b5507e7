"""GPU end to end of the host plugin with SR-IOV VFs (Plugin::sriovAware) on a fake sysfs tree: VFs under a PF on a host
driver are served and a preferred allocation keeps a request on one PF; a PF on vfio-pci with VFs enabled and its VFs are
withheld everywhere; a PF rebound after discovery makes Allocate's live path refuse its VF; a changed sriov_numvfs keeps
the surviving VFs' indices; with the setting off every output is the default plugin's and nothing new is read."""
import os

import numpy as np
import pytest

import dra_host as DH
import fake_sysfs
import pcie_host
import sriov_host as H
import topo_host
import viab_host

pytestmark = pytest.mark.gpu

CLASSES = H.NV
DRIVERS = ["gpu.nvidia.com"]
PF = dict(vendor=b"0x10de\n", device=b"0x2330\n")
VF = dict(vendor=b"0x10de\n", device=b"0x2331\n", driver="vfio-pci")
DOWN = "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0"  # one switch down port above everything
DEVS = [dict(bdf="0000:03:00.0", group=30, driver="nvidia", path=DOWN + "/0000:03:00.0", **PF),   # PF A, host driver
        dict(bdf="0000:03:00.1", group=40, driver="nvidia", path=DOWN + "/0000:03:00.1", **PF),   # PF B, host driver
        dict(bdf="0000:03:10.0", group=31, path=DOWN + "/0000:03:10.0", **VF),                    # A's VFs
        dict(bdf="0000:03:10.1", group=32, path=DOWN + "/0000:03:10.1", **VF),
        dict(bdf="0000:03:11.0", group=41, path=DOWN + "/0000:03:11.0", **VF),                    # B's VFs
        dict(bdf="0000:03:11.1", group=42, path=DOWN + "/0000:03:11.1", **VF),
        dict(bdf="0000:05:00.0", group=50, driver="vfio-pci", path="pci0000:00/0000:00:02.0/0000:05:00.0", **PF),  # PF C
        dict(bdf="0000:05:10.0", group=51, path="pci0000:00/0000:00:02.0/0000:05:10.0", **VF),
        dict(bdf="0000:05:10.1", group=52, path="pci0000:00/0000:00:02.0/0000:05:10.1", **VF)]
WHY_50 = "0000:05:00.0 has 2 VFs enabled"
WHY_51 = "0000:05:10.0 needs the VF token of 0000:05:00.0 (bound to vfio-pci)"
WHY_52 = "0000:05:10.1 needs the VF token of 0000:05:00.0 (bound to vfio-pci)"


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = pcie_host.make_nested_tree(root, DEVS, relative=True)
    H.link_vfs(base, "0000:03:00.0", ["0000:03:10.0", "0000:03:10.1"], b"2\n")
    H.link_vfs(base, "0000:03:00.1", ["0000:03:11.0", "0000:03:11.1"], b"2\n")
    H.link_vfs(base, "0000:05:00.0", ["0000:05:10.0", "0000:05:10.1"], b"2\n")
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, sriov, pcie=False):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, classes=CLASSES, dra=DRIVERS, pcie=pcie)
    if sriov is not None:
        H.set_sriov(hp, sriov)
    return hp


def _outputs(hp, tree):
    cdi = tree[3]
    specs = {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}
    return specs, [hp.list_and_watch(i) for i in range(2)], DH.slices(hp, 0)[0]


def _plugin_of(state, group):
    return [k for k, p in enumerate(state["plugins"]) for d in p["devs"] if d[0] == group][0]


def test_off_is_the_default_plugin(kx, tree):
    default = _plugin(kx, tree, None)
    try:
        default.init("YAML")
        want = _outputs(default, tree)
    finally:
        default.close()
    for f in os.listdir(tree[3]):
        os.remove(os.path.join(tree[3], f))
    off = _plugin(kx, tree, False)
    try:
        state = off.init("YAML")
        assert H.reads(off) == 0
        assert _outputs(off, tree) == want
        assert all(d[1] == "Healthy" for p in state["plugins"] for d in p["devs"])
        assert off.allocate(["51"])["cdi_devices"]  # served as any function
    finally:
        off.close()


def test_sriov_end_to_end(kx, tree):
    root, base = tree[0], tree[1]
    hp = _plugin(kx, tree, True, pcie=True)
    try:
        state = hp.init("YAML")
        assert H.reads(hp) == 7  # the seven vfio-pci functions; the PFs on nvidia are no candidates
        vfp, pfp = _plugin_of(state, "31"), _plugin_of(state, "50")
        devs = viab_host.devs(hp, vfp)
        assert {g: devs[g] for g in ("31", "32", "41", "42")} == {g: ("Healthy", None) for g in ("31", "32", "41", "42")}
        assert devs["51"] == ("Healthy", WHY_51) and devs["52"] == ("Healthy", WHY_52)
        assert viab_host.devs(hp, pfp) == {"50": ("Healthy", WHY_50)}
        # ListAndWatch: the withheld groups Unhealthy
        for k in (vfp, pfp):
            ids = [d[0] for d in state["plugins"][k]["devs"]]
            want = kx.lw_encode(np.array([int(g) for g in ids], np.uint32),
                                np.array([g not in ("50", "51", "52") for g in ids], np.uint8))
            assert hp.list_and_watch(k) == want
        # refused by Allocate and PrepareDraDevices, absent from the spec and the DRA pool
        for g, why in (("50", WHY_50), ("51", WHY_51), ("52", WHY_52)):
            with pytest.raises(RuntimeError, match="IOMMU group %s is not viable: %s" % (g, why.replace("(", r"\(").replace(")", r"\)"))):
                hp.allocate([g])
            with pytest.raises(RuntimeError, match="not viable"):
                DH.prepare(hp, DRIVERS[0], "node-a", ["vfio" + g])
        spec = open(os.path.join(tree[3], "cdi-vfio-xxxx.yaml"), "rb").read()
        for g in ("31", "32", "41", "42"):
            assert b"/dev/vfio/%s\n" % g.encode() in spec
        for g in ("50", "51", "52"):
            assert b"/dev/vfio/%s\n" % g.encode() not in spec
        blob = DH.slices(hp, 0)[0]
        assert b'"name":"vfio31"' in blob and all(b'"name":"vfio%s"' % g not in blob for g in (b"50", b"51", b"52"))
        assert DH.prepare(hp, DRIVERS[0], "node-a", ["vfio41"]) == [["nvidia.com/gpu=%d" % _index(state, "0000:03:11.0")]]
        # the same request on a plugin without PFs in the forest mixes the two PFs
        plain = _plugin(kx, tree, False, pcie=True)
        try:
            plain.init("YAML")
            assert topo_host.preferred_allocation(plain, vfp, [(["31", "41", "42"], [], 2)])[0] == ["31", "41"]
        finally:
            plain.close()
        # a 2-VF request over VFs of both PFs under one down port stays on the PF that holds two (without PFs in the
        # forest the best fit is the down port, and position order would take 31 and 41)
        got = topo_host.preferred_allocation(hp, vfp, [(["31", "41", "42"], [], 2)])
        assert got[0] == ["41", "42"]
        got = topo_host.preferred_allocation(hp, vfp, [(["31", "41", "32"], ["41"], 2)])
        assert got[0] == ["41", "31"] or got[0] == ["41", "32"]
        # PF A rebound to vfio-pci after discovery: the live path refuses its VF
        assert hp.allocate(["31"])["cdi_devices"]
        H.rebind(root, base, "0000:03:00.0", "vfio-pci")
        with pytest.raises(RuntimeError, match=r"0000:03:10.0 needs the VF token of 0000:03:00.0 \(bound to vfio-pci\)"):
            hp.allocate(["31"])
        H.rebind(root, base, "0000:03:00.0", "nvidia")
        assert hp.allocate(["31"])["cdi_devices"]
        # VFs enabled on a served function since discovery: refused naming it
        open(os.path.join(base, "0000:03:11.1", "sriov_numvfs"), "wb").write(b"1\n")
        with pytest.raises(RuntimeError, match="0000:03:11.1 has 1 VFs enabled"):
            hp.allocate(["42"])
        os.remove(os.path.join(base, "0000:03:11.1", "sriov_numvfs"))
    finally:
        hp.close()


def _index(state, bdf):
    return [m[1] for _, ms in state["iommuMap"] for m in ms if m[0] == bdf][0]


def test_rediscover_after_numvfs_change(kx, tree):
    root, base = tree[0], tree[1]
    hp = _plugin(kx, tree, True)
    try:
        a = hp.init("YAML")
        gen = DH.generation(hp)
        # PF B goes from 2 to 3 VFs, and PF C's VFs are disabled (echo 0 > sriov_numvfs)
        new = dict(bdf="0000:03:11.2", group=43, path=DOWN + "/0000:03:11.2", **VF)
        os.makedirs(os.path.join(root, "devices", new["path"]))
        tgt = os.path.join(root, "devices", new["path"])
        for f in ("vendor", "device"):
            open(os.path.join(tgt, f), "wb").write(new[f])
        os.symlink(os.path.join(root, "drivers", "vfio-pci"), os.path.join(tgt, "driver"))
        os.makedirs(os.path.join(root, "iommu_groups", "43"))
        os.symlink(os.path.join(root, "iommu_groups", "43"), os.path.join(tgt, "iommu_group"))
        os.symlink(os.path.join("../../../devices", new["path"]), os.path.join(base, new["bdf"]))
        os.symlink("../0000:03:00.1", os.path.join(tgt, "physfn"))
        open(os.path.join(base, "0000:03:00.1", "sriov_numvfs"), "wb").write(b"3\n")
        for vf in ("0000:05:10.0", "0000:05:10.1"):
            os.remove(os.path.join(base, vf))
        open(os.path.join(base, "0000:05:00.0", "sriov_numvfs"), "wb").write(b"0\n")
        r = viab_host.rediscover(hp)
        before = {m[0]: m[1] for _, ms in a["iommuMap"] for m in ms}
        after = {m[0]: m[1] for _, ms in r["iommuMap"] for m in ms}
        for bdf in ("0000:03:10.0", "0000:03:10.1", "0000:03:11.0", "0000:03:11.1", "0000:05:00.0"):
            assert after[bdf] == before[bdf]
        assert after["0000:03:11.2"] > max(before.values())
        assert r["report"]["changed"]
        assert DH.generation(hp) == gen + 1
        # PF C has no VFs now: served
        assert viab_host.devs(hp, _plugin_of(r, "50"))["50"] == ("Healthy", None)
        assert hp.allocate(["50"])["cdi_devices"] == ["nvidia.com/gpu=%d" % before["0000:05:00.0"]]
        assert b"/dev/vfio/50\n" in open(os.path.join(tree[3], "cdi-vfio-xxxx.yaml"), "rb").read()
    finally:
        hp.close()
