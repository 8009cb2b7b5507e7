"""GPU end to end of the host plugin serving vGPUs that live on SR-IOV VFs (XpuClass::vfVgpu) on a fake sysfs tree: one
PF on the vGPU manager's driver and eight VFs, three of type A, two of type B and three free ones that list both names.
Two plugins named by the type keys and one spec file with five devices; the PF and the free VFs are never offered;
nothing is withheld with sriovAware; a changed type is refused by Allocate and moves the VF to the other plugin with a
fresh index at rediscover; learned names keep both resources when every VF is taken; a restart on that full GPU serves
them only with vgpuTypeNames; with the setting off the outputs are unchanged."""
import os

import pytest

import dra_host as DH
import fake_sysfs
import sriov_host as SH
import vf_vgpu_host as H
import viab_host

pytestmark = pytest.mark.gpu

VF = dict(vendor=b"0x10de\n", device=b"0x2331\n", driver="nvidia")
PF = "0000:03:00.0"
VFS = ["0000:03:00.%d" % k for k in range(1, 8)] + ["0000:03:01.0"]
GROUP = {PF: 30, **{bdf: 31 + k for k, bdf in enumerate(VFS)}}
TYPE = {VFS[0]: 557, VFS[1]: 557, VFS[2]: 557, VFS[3]: 558, VFS[4]: 558}  # VFS[5:] are free
LIST = H.HEADER + b"557   : NVIDIA H100-4C\n558   : NVIDIA H100-8C\n"
A, B = "NVIDIA_H100-4C", "NVIDIA_H100-8C"
NAMES = {557: "NVIDIA H100-4C", 558: "NVIDIA H100-8C"}


@pytest.fixture
def tree(tmp_path, pci_text):
    devs = [dict(bdf=PF, group=30, vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia")]
    devs += [dict(bdf=bdf, group=GROUP[bdf], **VF) for bdf in VFS]
    base = fake_sysfs.make_tree(str(tmp_path), devs)
    SH.link_vfs(base, PF, VFS, b"8\n")
    for bdf in VFS:
        t = TYPE.get(bdf, 0)
        H.set_files(base, bdf, b"%d\n" % t, H.HEADER if t else LIST)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return str(tmp_path), base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, on=True, names=None, sriov=False):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    assert hp.L.kxh_set_classes(hp.h, H.CLASSES.encode()) == 0
    if on is not None:
        H.set_vf_vgpu(hp, 1, on, names)
    SH.set_sriov(hp, sriov)
    return hp


def _vgpu_plugins(state):
    """{type key: {group id: CDI index}} of the vGPU class's plugins"""
    index = {str(g): ms[0][1] for g, ms in state["iommuMap"]}
    return {p["name"]: {d[0]: index[d[0]] for d in p["devs"]} for p in state["plugins"]
            if p["resource"].startswith("nvidia.com/NVIDIA_H100")}


def _spec(tree):
    return open(os.path.join(tree[3], "cdi-vgpu-vf.yaml"), "rb").read()


def _offered(state):
    return {d[0] for p in state["plugins"] for d in p["devs"]}


def test_end_to_end(kx, tree):
    root, base = tree[0], tree[1]
    hp = _plugin(kx, tree)
    try:
        state = hp.init("YAML")
        assert H.reads(hp) == 16  # two files for each of the eight VFs; the PF is never read
        plugins = _vgpu_plugins(state)
        assert sorted(plugins) == [A, B]
        assert set(plugins[A]) == {"31", "32", "33"} and set(plugins[B]) == {"34", "35"}
        assert [p["resource"] for p in state["plugins"] if p["name"] in (A, B)] == ["nvidia.com/" + A, "nvidia.com/" + B]
        assert _offered(state) == {"31", "32", "33", "34", "35"}  # neither the PF (30) nor the free VFs (36-38)
        spec = _spec(tree)
        assert spec.count(b"  - name:") == 5
        for g in range(30, 39):
            assert (b"/dev/vfio/%d\n" % g in spec) == (31 <= g <= 35)
        assert hp.allocate(["31"])["cdi_devices"] == ["nvidia.com/vgpu=%d" % plugins[A]["31"]]
        assert H.learned(hp) == {557: A, 558: B}
        # a type change sends no uevent: Allocate re-reads it, and rediscover moves the VF with a fresh index
        before = max(i for p in plugins.values() for i in p.values())
        H.set_files(base, VFS[0], b"558\n")
        with pytest.raises(RuntimeError, match="0000:03:00.1 carries vGPU type 558, not type 557 as discovered"):
            hp.allocate(["31"])
        state = DH.rediscover(hp)
        plugins = _vgpu_plugins(state)
        assert set(plugins[A]) == {"32", "33"} and set(plugins[B]) == {"31", "34", "35"}
        assert plugins[B]["31"] > before
        assert state["report"]["pci"]["n_changed"] == 1
        assert any(f.endswith("cdi-vgpu-vf.yaml") for f in state["report"]["written"])
        assert b"nvidia.com/vgpu=%d" % plugins[B]["31"] in _spec(tree)
        assert hp.allocate(["31"])["cdi_devices"] == ["nvidia.com/vgpu=%d" % plugins[B]["31"]]
        # every free VF taken: no list names a type any more, the learned names keep both resources
        for bdf in VFS[5:]:
            H.set_files(base, bdf, b"557\n")
        for bdf in VFS:
            H.set_files(base, bdf, creatable=H.HEADER)
        state = DH.rediscover(hp)
        plugins = _vgpu_plugins(state)
        assert set(plugins[A]) == {"32", "33", "36", "37", "38"} and set(plugins[B]) == {"31", "34", "35"}
    finally:
        hp.close()
    # a new plugin on the full GPU: only vgpuTypeNames name the types
    bare = _plugin(kx, tree)
    try:
        assert _vgpu_plugins(bare.init("YAML")) == {}
    finally:
        bare.close()
    named = _plugin(kx, tree, names=NAMES)
    try:
        plugins = _vgpu_plugins(named.init("YAML"))
        assert set(plugins[A]) == {"32", "33", "36", "37", "38"} and set(plugins[B]) == {"31", "34", "35"}
    finally:
        named.close()


def test_nothing_withheld_with_sriov(kx, tree):
    hp = _plugin(kx, tree, sriov=True)
    try:
        state = hp.init("YAML")
        for k, p in enumerate(state["plugins"]):
            if p["name"] in (A, B):
                assert all(blocker is None for _, blocker in viab_host.devs(hp, k).values())
        assert _spec(tree).count(b"  - name:") == 5
        assert hp.allocate(["34"])["cdi_devices"]
    finally:
        hp.close()


def test_off_outputs_unchanged(kx, tree):
    outs = []
    for on in (None, False):
        for f in os.listdir(tree[3]):
            os.remove(os.path.join(tree[3], f))
        hp = _plugin(kx, tree, on=on)
        try:
            state = hp.init("YAML")
            assert H.reads(hp) == 0
            specs = {f: open(os.path.join(tree[3], f), "rb").read() for f in sorted(os.listdir(tree[3]))}
            outs.append((state, specs, [hp.list_and_watch(k) for k in range(len(state["plugins"]))]))
        finally:
            hp.close()
    assert outs[0] == outs[1]
    state = outs[0][0]
    # without the setting the class is a passthrough class on the manager's driver: the PF and every VF under one id
    assert _offered(state) == {str(g) for g in range(30, 39)}
