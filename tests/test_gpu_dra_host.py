"""GPU end to end of the host plugin's DRA ResourceSlices (XpuClass::draDriver) on a fake sysfs whose entries link into
devices/pci.../<bdf> and carry numa_node files: an NVIDIA class and an AMD class, ResourceSlices against the oracle run
on records built from the tree, a blocked group left out, PrepareDraDevices against Allocate and the CDI spec, the
generation after a rediscovery, the configuration errors, and a plugin without a DRA driver that reads and writes
exactly what it did before."""
import os

import numpy as np
import pytest

import dra_host as DH
import fake_sysfs
import pcie_host
from oracle import dra_oracle as DO

pytestmark = pytest.mark.gpu

CLASSES = "10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-xxxx;1002,vfio-pci,amd.com,amd.com/gpu,cdi-amd"
NV = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
AMD = dict(vendor=b"0x1002\n", device=b"0x74a1\n", driver="vfio-pci")
AUDIO = dict(vendor=b"0x10de\n", device=b"0x22a3\n")
DEVS = [
    dict(bdf="0000:21:00.0", group=20, path="pci0000:20/0000:20:01.0/0000:21:00.0", numa=b"0\n", **NV),
    dict(bdf="0000:21:00.1", group=20, path="pci0000:20/0000:20:01.0/0000:21:00.1", driver="snd_hda_intel", **AUDIO),
    dict(bdf="0000:41:00.0", group=40, path="pci0000:40/0000:40:01.0/0000:41:00.0", numa=b"0\n", **NV),
    dict(bdf="0000:81:00.0", group=80, path="pci0000:80/0000:80:01.0/0000:81:00.0", **NV),
    dict(bdf="0000:c1:00.0", group=214, path="pci0000:c0/0000:c0:01.0/0000:c1:00.0", numa=b"1\n", **NV),
    dict(bdf="0000:c1:00.1", group=214, path="pci0000:c0/0000:c0:01.0/0000:c1:00.1", numa=b"1\n", driver="vfio-pci",
         **AUDIO),
    dict(bdf="0000:e1:00.0", group=300, path="pci0000:e0/0000:e0:01.0/0000:e1:00.0", numa=b"-1\n", **AMD),
    dict(bdf="0000:e2:00.0", group=301, path="pci0000:e0/0000:e0:02.0/0000:e2:00.0", numa=b"1\n", **AMD),
]
DRIVERS = ["vfio.nvidia.com", "vfio.amd.com"]


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = pcie_host.make_nested_tree(root, DEVS, relative=True)
    DH.add_numa(root, DEVS)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, **cfg):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, classes=CLASSES, **cfg)
    return hp


def _cdi(cdi):
    return {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}


@pytest.mark.parametrize("topo", [False, True])
@pytest.mark.parametrize("pcie", [False, True])
@pytest.mark.parametrize("viability", [False, True])
def test_slices_match_oracle(kx, tree, topo, pcie, viability):
    hp = _plugin(kx, tree, dra=DRIVERS, topo=topo, pcie=pcie, viability=viability)
    try:
        state = hp.init("YAML")
        assert DH.generation(hp) == 1
        for cls, driver in enumerate(DRIVERS):
            want = DH.expected_records(state, DEVS, cls)
            if viability:
                want = want[want["iommu_group"] != 20]  # 0000:21:00.1 is bound to snd_hda_intel
            blob, offs = DH.slices(hp, cls)
            wblob, woffs = DO.dra_slices(driver, "node-a", "node-a", 1, want)
            assert blob == wblob and np.array_equal(offs, woffs)
            assert (b'"name":"vfio20"' in blob) == (cls == 0 and not viability)
        nv = DH.slices(hp, 0)[0]
        assert b'"numaNode":{"int":1}' in nv and b'"resource.kubernetes.io/pcieRoot":{"string":"pci0000:c0"}' in nv
    finally:
        hp.close()


def test_prepare_matches_allocate_and_spec(kx, tree):
    hp = _plugin(kx, tree, dra=DRIVERS)
    cdi = tree[3]
    try:
        hp.init("YAML")
        for driver, groups, kind in ((DRIVERS[0], ["214", "40", "80", "20"], "nvidia.com/gpu"), (DRIVERS[1], ["300", "301"], "amd.com/gpu")):
            got = DH.prepare(hp, driver, "node-a", ["vfio" + g for g in groups])
            assert got == [hp.allocate([g])["cdi_devices"] for g in groups]
            specs = b"".join(_cdi(cdi).values())
            for names in got:
                for name in names:
                    k, idx = name.split("=")
                    assert k == kind and b'kind: ' + kind.encode() in specs and b'- name: "%s"' % idx.encode() in specs
        with pytest.raises(RuntimeError, match="unknown DRA driver vfio.other.com"):
            DH.prepare(hp, "vfio.other.com", "node-a", ["vfio214"])
        with pytest.raises(RuntimeError, match="unknown pool node-b"):
            DH.prepare(hp, DRIVERS[0], "node-b", ["vfio214"])
        with pytest.raises(RuntimeError, match="unknown device vfio300 "):  # an AMD group under the NVIDIA driver
            DH.prepare(hp, DRIVERS[0], "node-a", ["vfio214", "vfio300"])
        with pytest.raises(RuntimeError, match="unknown device gpu214 "):
            DH.prepare(hp, DRIVERS[0], "node-a", ["gpu214"])
    finally:
        hp.close()


def test_blocked_group_refused_by_prepare(kx, tree):
    hp = _plugin(kx, tree, dra=DRIVERS, viability=True)
    try:
        hp.init("YAML")
        with pytest.raises(RuntimeError, match="IOMMU group 20 is not viable: 0000:21:00.1 is bound to snd_hda_intel"):
            DH.prepare(hp, DRIVERS[0], "node-a", ["vfio20"])
    finally:
        hp.close()


def test_rediscover_bumps_generation(kx, tree):
    root, base = tree[0], tree[1]
    hp = _plugin(kx, tree, dra=DRIVERS)
    try:
        hp.init("YAML")
        assert b'"name":"vfio40"' in DH.slices(hp, 0)[0]
        DH.rediscover(hp)  # nothing moved
        assert DH.generation(hp) == 1
        os.remove(os.path.join(base, "0000:41:00.0"))
        state = DH.rediscover(hp)
        assert DH.generation(hp) == 2
        blob, offs = DH.slices(hp, 0)
        assert b'"name":"vfio40"' not in blob and b'"generation":2' in blob
        want = DH.expected_records(state, [d for d in DEVS if d["bdf"] != "0000:41:00.0"], 0)
        wblob, woffs = DO.dra_slices(DRIVERS[0], "node-a", "node-a", 2, want)
        assert blob == wblob and np.array_equal(offs, woffs)
        assert b'"generation":2' in DH.slices(hp, 1)[0]  # one generation for every class's pool
    finally:
        hp.close()


def test_configuration_errors(kx, tree):
    hp = _plugin(kx, tree, dra=DRIVERS, node="")
    try:
        assert DH.initiate(hp) == "DRA driver vfio.nvidia.com is set but the node name is empty (NODE_NAME)"
    finally:
        hp.close()
    hp = _plugin(kx, tree, dra=[DRIVERS[0], DRIVERS[0]])
    try:
        assert DH.initiate(hp) == "DRA driver vfio.nvidia.com is set on two classes (0 and 1)"
    finally:
        hp.close()
    hp = _plugin(kx, tree, dra=DRIVERS)
    try:
        assert DH.initiate(hp) is None
        with pytest.raises(RuntimeError, match="class 2 has no DRA driver"):
            DH.slices(hp, 2)
    finally:
        hp.close()


def test_without_dra_driver_nothing_changes(kx, tree, oracle):
    """A plugin with the default settings, under counting seams, reads no numa_node and no entry link, and every
    output equals a plugin's built without touching the feature; with a DRA driver the reads happen and the
    device-plugin outputs still do not change."""
    cdi = tree[3]
    outs = []
    for dra in (None, ["", ""], DRIVERS):
        hp = _plugin(kx, tree, dra=dra)
        count = DH.Counter(hp) if dra is not None else None
        try:
            state = hp.init("YAML")
            n_plugins = len(state["plugins"])
            outs.append((state, [hp.list_and_watch(i) for i in range(n_plugins)], _cdi(cdi),
                         [hp.allocate([g]) for g in ("214", "40", "300")]))
            reads = count.reads() if count else None
        finally:
            hp.close()
        if dra == ["", ""]:
            assert reads == (0, 0)
        if dra == DRIVERS:
            assert reads[0] > 0 and reads[1] == len(DEVS)
    assert outs[0] == outs[1] == outs[2]
