"""GPU end to end of the host plugin's vGPU DRA ResourceSlices (a draDriver on a vGPU class) on a fake sysfs whose
mdev entries link under pci<domain>:<bus> components and whose parent GPUs carry `device` and `numa_node` files: the
slices against the oracle run on records built from the tree, the failed reads that drop only their attribute, a
passthrough pool beside a vGPU pool, PrepareDraDevices for both drivers, the start-up refusals, the generations after
rediscovery, and a plugin without a vGPU DRA driver that reads and writes exactly what it did before."""
import os

import numpy as np
import pytest

import dra_host as DH
import dra_mdev_host as MH
import fake_mdev
import fake_sysfs
from oracle import dra_mdev_oracle as DMO
from oracle import dra_oracle as DO

pytestmark = pytest.mark.gpu

VGPU = [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")]
NV = dict(vendor=b"0x10de\n", driver="nvidia")
PARENTS = [
    dict(bdf="0000:c1:00.0", group=40, path="pci0000:c0/0000:c0:01.0/0000:c1:00.0", device=b"0x2330\n", numa=b"1\n", **NV),
    # no numa_node file: numaNode left out
    dict(bdf="0000:41:00.0", group=41, path="pci0000:40/0000:40:01.0/0000:41:00.0", device=b"0x2330\n", **NV),
    # no device file: parentDeviceID and productName left out
    dict(bdf="0000:e1:00.0", group=42, path="pci0000:e0/0000:e0:01.0/0000:e1:00.0", numa=b"0\n", **NV),
    # a link without a pci... component: the root is unknown
    dict(bdf="0000:d1:00.0", group=43, path="platform/0000:d1:00.0", device=b"0xfffe\n", numa=b"0\n", **NV),
    # a passthrough GPU of the NVIDIA class
    dict(bdf="0000:81:00.0", group=80, path="pci0000:80/0000:80:01.0/0000:81:00.0", vendor=b"0x10de\n", device=b"0x2330\n",
         driver="vfio-pci", numa=b"0\n"),
]
U = ["0b2ad9a2-6e2c-4a55-9d41-%012x" % k for k in range(8)]
MDEVS = [
    dict(uuid=U[1], parent="0000:c1:00.0", group=300),
    dict(uuid=U[2], parent="0000:c1:00.0", group=301, type_id="nvidia-1121", name=b"NVIDIA H100XM-2-20C\n"),
    dict(uuid=U[3], parent="0000:41:00.0", group=302),
    dict(uuid=U[4], parent="0000:e1:00.0", group=303),
    dict(uuid=U[5], parent="0000:d1:00.0", group=304),
]
VDRV, PDRV = "vgpu.nvidia.com", "vfio.nvidia.com"


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base, mbase = MH.make_tree(root, PARENTS, MDEVS)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, mbase, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, vdra=None, pdra=None, node="node-a", topo=False):
    root, base, mbase, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, dra=pdra, node=node, topo=topo)
    fake_mdev.set_vgpu(hp, mbase, VGPU)
    if vdra is not None:
        MH.set_vgpu_dra(hp, vdra, node)
    return hp


def _model_name(oracle, pci_text):
    return lambda vendor, device: oracle.lookup_many(pci_text, [int(vendor, 16) << 16 | int(device, 16)])[1][0]


def _attrs(blob):
    import json
    return {d["name"]: d["attributes"] for line in blob.splitlines() for d in json.loads(line)["spec"]["devices"]}


@pytest.mark.parametrize("topo", [False, True])
def test_slices_match_oracle(kx, tree, oracle, pci_text, topo):
    hp = _plugin(kx, tree, vdra=[VDRV], pdra=[PDRV], topo=topo)
    try:
        state = hp.init("YAML")
        assert MH.generation(hp) == 1 and DH.generation(hp) == 1
        want = MH.expected_records(state, PARENTS, 0, _model_name(oracle, pci_text))
        assert len(want) == 5
        blob, offs = MH.slices(hp, 0)
        wblob, woffs = DMO.dra_slices_mdev(VDRV, "node-a", "node-a", 1, want)
        assert blob == wblob and np.array_equal(offs, woffs)
        a = _attrs(blob)
        assert a["vfio300"]["productName"] == {"string": "GH100_H100_SXM5_80GB"} and a["vfio300"]["numaNode"] == {"int": 1}
        assert a["vfio300"]["resource.kubernetes.io/pcieRoot"] == {"string": "pci0000:c0"}
        assert a["vfio301"]["mdevType"] == {"string": "NVIDIA_H100XM-2-20C"} and a["vfio301"]["uuid"] == {"string": U[2]}
        # each failed read drops its attribute and nothing else
        assert "numaNode" not in a["vfio302"] and a["vfio302"]["parentDeviceID"] == {"string": "2330"}
        assert "parentDeviceID" not in a["vfio303"] and "productName" not in a["vfio303"] and a["vfio303"]["numaNode"] == {"int": 0}
        assert "resource.kubernetes.io/pcieRoot" not in a["vfio304"] and a["vfio304"]["parentAddress"] == {"string": "0000:d1:00.0"}
        # the passthrough pool beside it
        pblob, poffs = DH.slices(hp, 0)
        pwant = DH.expected_records(state, PARENTS, 0)
        assert len(pwant) == 1
        pw, pwoffs = DO.dra_slices(PDRV, "node-a", "node-a", 1, pwant)
        assert pblob == pw and np.array_equal(poffs, pwoffs)
        with pytest.raises(RuntimeError, match="vGPU class 1 has no DRA driver"):
            MH.slices(hp, 1)
    finally:
        hp.close()


def test_vgpu_pool_alone(kx, tree, oracle, pci_text):
    """a DRA driver on the vGPU class only: the passthrough class is not published"""
    hp = _plugin(kx, tree, vdra=[VDRV])
    try:
        state = hp.init("YAML")
        want = MH.expected_records(state, PARENTS, 0, _model_name(oracle, pci_text))
        assert MH.slices(hp, 0)[0] == DMO.dra_slices_mdev(VDRV, "node-a", "node-a", 1, want)[0]
        with pytest.raises(RuntimeError, match="class 0 has no DRA driver"):
            DH.slices(hp, 0)
    finally:
        hp.close()


def test_prepare_both_drivers(kx, tree):
    hp = _plugin(kx, tree, vdra=[VDRV], pdra=[PDRV])
    try:
        hp.init("YAML")
        groups = ["300", "304", "302"]
        assert DH.prepare(hp, VDRV, "node-a", ["vfio" + g for g in groups]) == [hp.allocate([g])["cdi_devices"] for g in groups]
        assert all(n.startswith("nvidia.com/vgpu=") for g in groups for n in hp.allocate([g])["cdi_devices"])
        assert DH.prepare(hp, PDRV, "node-a", ["vfio80"]) == [hp.allocate(["80"])["cdi_devices"]]
        with pytest.raises(RuntimeError, match="unknown device vfio80 "):  # a passthrough group under the vGPU driver
            DH.prepare(hp, VDRV, "node-a", ["vfio300", "vfio80"])
        with pytest.raises(RuntimeError, match="unknown device vfio300 "):  # a vGPU group under the passthrough driver
            DH.prepare(hp, PDRV, "node-a", ["vfio300"])
        with pytest.raises(RuntimeError, match="unknown pool node-b"):
            DH.prepare(hp, VDRV, "node-b", ["vfio300"])
        with pytest.raises(RuntimeError, match="unknown DRA driver vgpu.other.com"):
            DH.prepare(hp, "vgpu.other.com", "node-a", ["vfio300"])
    finally:
        hp.close()


def test_startup_refusals(kx, tree):
    hp = _plugin(kx, tree, vdra=[PDRV], pdra=[PDRV])
    try:
        assert DH.initiate(hp) == "DRA driver vfio.nvidia.com is set on two classes (0 and vGPU 0)"
    finally:
        hp.close()
    hp = _plugin(kx, tree, vdra=[VDRV], node="")
    try:
        assert DH.initiate(hp) == "DRA driver vgpu.nvidia.com is set but the node name is empty (NODE_NAME)"
    finally:
        hp.close()
    hp = _plugin(kx, tree, vdra=[VDRV], pdra=[PDRV])
    try:
        assert DH.initiate(hp) is None
    finally:
        hp.close()


def test_rediscover_generations(kx, tree, oracle, pci_text):
    root, base, mbase = tree[0], tree[1], tree[2]
    hp = _plugin(kx, tree, vdra=[VDRV], pdra=[PDRV])
    try:
        hp.init("YAML")
        DH.rediscover(hp)  # nothing moved
        assert (MH.generation(hp), DH.generation(hp)) == (1, 1)
        new = dict(uuid=U[6], parent="0000:41:00.0", group=305)
        MH.add_mdev(root, PARENTS, new)
        state = DH.rediscover(hp)
        assert (MH.generation(hp), DH.generation(hp)) == (2, 1)
        blob, offs = MH.slices(hp, 0)
        assert b'"name":"vfio305"' in blob and b'"generation":2' in blob
        want = MH.expected_records(state, PARENTS, 0, _model_name(oracle, pci_text))
        wblob, woffs = DMO.dra_slices_mdev(VDRV, "node-a", "node-a", 2, want)
        assert blob == wblob and np.array_equal(offs, woffs)
        os.remove(os.path.join(mbase, U[1]))  # vGPU 300 destroyed
        DH.rediscover(hp)
        assert (MH.generation(hp), DH.generation(hp)) == (3, 1)
        assert b'"name":"vfio300"' not in MH.slices(hp, 0)[0]
        os.remove(os.path.join(base, "0000:81:00.0"))  # the passthrough GPU leaves
        DH.rediscover(hp)
        assert (MH.generation(hp), DH.generation(hp)) == (3, 2)
        assert b'"generation":3' in MH.slices(hp, 0)[0] and b'"generation":2' in DH.slices(hp, 0)[0]
    finally:
        hp.close()


def test_without_vgpu_dra_nothing_changes(kx, tree):
    """Under counting seams: with no vGPU DRA driver nothing new is read; with one, the mdev walk reads each entry's
    parent numa_node, link and device once and the PCI walk nothing new; every device-plugin output stays the same."""
    cdi = tree[4]
    outs = []
    for vdra in (None, [""], [VDRV]):
        hp = _plugin(kx, tree, vdra=vdra)
        count, dev = DH.Counter(hp), MH.DeviceReads(hp)
        try:
            state = hp.init("YAML")
            outs.append((state, [hp.list_and_watch(i) for i in range(len(state["plugins"]))],
                         {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))},
                         [hp.allocate([g]) for g in ("300", "304", "80")]))
            reads = count.reads() + (dev.reads(),)
        finally:
            hp.close()
        assert reads == ((len(MDEVS),) * 3 if vdra == [VDRV] else (0, 0, 0)), (vdra, reads)
    assert outs[0] == outs[1] == outs[2]
