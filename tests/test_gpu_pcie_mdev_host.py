"""GPU end to end of the host plugin's vGPU PCIe topology (Plugin::vgpuPcieTopologyAware) on a fake sysfs whose vGPU
parents sit behind switches: with the setting off no mdev link is read and a vGPU plugin's answer is
kxpu_preferred_allocation's (also with pcieTopologyAware on); with it on, requests are packed under one parent GPU, then
one switch, a must-include vGPU pulls the rest from its GPU, unknown paths give the NUMA answer, and a rediscovery after
an mdev moved to another parent moves its node."""
import numpy as np
import pytest

import dra_host
import fake_mdev
import fake_sysfs
import pcie_host
import pcie_mdev_host as MH
import topo_host

pytestmark = pytest.mark.gpu

VGPU = [("10de", "nvidia-vgpu", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")]
# GPUs A and B behind one switch (root port 00:01.0); C and D each behind a root port of their own
GPUS = {"0000:03:00.0": "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0",
        "0000:04:00.0": "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:01.0/0000:04:00.0",
        "0000:07:00.0": "pci0000:00/0000:00:02.0/0000:05:00.0/0000:06:00.0/0000:07:00.0",
        "0000:0a:00.0": "pci0000:00/0000:00:03.0/0000:08:00.0/0000:09:00.0/0000:0a:00.0"}
ORDER = list(GPUS)
# 16 vGPUs of one type, 4 per GPU; lexical UUID order (the walk order) deals them out round robin over the GPUs
MDEVS = [dict(uuid="%08x-0000-4000-8000-%012x" % (k, k), parent=ORDER[k % 4], group=300 + k, driver="nvidia-vgpu",
              type_id="nvidia-471", name=b"GRID A100-10C\n") for k in range(16)]
GPU_OF = {str(m["group"]): m["parent"] for m in MDEVS}
IDS = [str(300 + k) for k in range(16)]


def _plugin(tmp_path, kx, pci_text, vgpu_pcie, pcie=False, topo=False, gpus=GPUS):
    """A host plugin over the fake tree (built on first use, parents placed by gpus) with one vGPU class"""
    root = str(tmp_path)
    if not (tmp_path / "bus" / "mdev").exists():
        fake_sysfs.make_tree(root, [])
        MH.make_tree(root, gpus, MDEVS)
        (tmp_path / "pci.ids").write_bytes(pci_text)
        (tmp_path / "cdi").mkdir()
    hp = fake_sysfs.HostPlugin(kx, str(tmp_path / "bus" / "pci" / "devices"), str(tmp_path / "pci.ids"),
                               str(tmp_path / "cdi") + "/")
    fake_mdev.set_vgpu(hp, str(tmp_path / "bus" / "mdev" / "devices"), VGPU)
    MH.set_vgpu_pcie(hp, vgpu_pcie)
    pcie_host.set_pcie(hp, pcie)
    topo_host.set_topology(hp, topo)
    count = dra_host.Counter(hp)
    state = hp.init("YAML")
    return hp, state, count


def _vgpu_plugin(state):
    k = [i for i, p in enumerate(state["plugins"]) if p["vgpu"]]
    assert len(k) == 1
    return k[0]


def _numa_answer(kx, hp, plugin, reqs):
    """kxpu_preferred_allocation over the plugin's devices (their NUMA masks), as IDs"""
    numa = topo_host.devs_numa(hp, plugin)
    ids = list(numa)
    pos = {d: i for i, d in enumerate(ids)}
    dev_numa = np.array([numa[d] for d in ids], np.uint64)
    out = kx.preferred_allocation(dev_numa, [([pos[a] for a in av], [pos[m] for m in mu], s) for av, mu, s in reqs])
    return [[ids[p] for p in q] for q in out]


REQS = [(IDS, [], 4), (IDS, ["306"], 4), (IDS, [], 6), (IDS, ["300", "301"], 2), (IDS[::3], [], 3)]


def test_setting_off_reads_nothing_and_keeps_the_numa_answer(tmp_path, kx, pci_text):
    for pcie in (False, True):
        hp, state, count = _plugin(tmp_path, kx, pci_text, vgpu_pcie=False, pcie=pcie, topo=True)
        assert count.reads()[1] == 0  # no entry link read: the PCI walk is empty and the mdev walk reads none
        k = _vgpu_plugin(state)
        assert set(pcie_host.devs_pcie(hp, k).values()) == {0xFFFFFFFF}
        got = topo_host.preferred_allocation(hp, k, REQS)
        assert got == _numa_answer(kx, hp, k, REQS)
        assert [GPU_OF[d] for d in got[0]] == ORDER  # walk order: one vGPU of every GPU
        hp.close()
    hp, state, count = _plugin(tmp_path, kx, pci_text, vgpu_pcie=False)
    assert topo_host.options(hp)["GetPreferredAllocationAvailable"] is False
    assert topo_host.preferred_allocation(hp, _vgpu_plugin(state), REQS) == []  # the reference's empty answer
    hp.close()


def test_setting_on_packs_under_one_gpu_then_one_switch(tmp_path, kx, pci_text):
    hp, state, count = _plugin(tmp_path, kx, pci_text, vgpu_pcie=True)
    assert count.reads()[1] == len(MDEVS)  # one link read per mdev
    assert topo_host.options(hp)["GetPreferredAllocationAvailable"] is True
    k = _vgpu_plugin(state)
    nodes = pcie_host.devs_pcie(hp, k)
    assert len({nodes[d] for d in IDS}) == 4 and all(v != 0xFFFFFFFF for v in nodes.values())
    for gpu in ORDER:  # the vGPUs of one GPU share its node
        assert len({nodes[d] for d in IDS if GPU_OF[d] == gpu}) == 1
    a, b, c, d, e = topo_host.preferred_allocation(hp, k, REQS)
    assert len({GPU_OF[x] for x in a}) == 1  # 4 of 4 free on each GPU: one GPU
    assert "306" in b and {GPU_OF[x] for x in b} == {GPU_OF["306"]}  # the must-include vGPU's GPU
    assert {GPU_OF[x] for x in c} == {ORDER[0], ORDER[1]}  # 6: the two GPUs behind one switch, not C and D
    assert d == ["300", "301"]
    assert {GPU_OF[x] for x in e} <= {ORDER[0], ORDER[1]}  # 3 of A, B, C, D's 2, 1, 1, 2: the switch holding 3
    hp.close()


def test_unknown_paths_give_the_numa_answer(tmp_path, kx, pci_text):
    flat = {a: "platform/" + a for a in GPUS}  # links with no component that begins with "pci": every path unknown
    hp, state, count = _plugin(tmp_path, kx, pci_text, vgpu_pcie=True, gpus=flat)
    assert count.reads()[1] == len(MDEVS)
    k = _vgpu_plugin(state)
    assert set(pcie_host.devs_pcie(hp, k).values()) == {0xFFFFFFFF}
    assert topo_host.preferred_allocation(hp, k, REQS) == _numa_answer(kx, hp, k, REQS)
    hp.close()


def test_rediscover_moves_the_node(tmp_path, kx, pci_text):
    hp, state, _ = _plugin(tmp_path, kx, pci_text, vgpu_pcie=True)
    k = _vgpu_plugin(state)
    before = pcie_host.devs_pcie(hp, k)
    # vGPU 300 leaves GPU A for GPU D (destroyed on one, created with the same UUID and group on the other)
    MH.move(str(tmp_path), MDEVS[0]["uuid"], GPUS[ORDER[0]], GPUS[ORDER[3]])
    rep = dra_host.rediscover(hp)
    assert rep is not None
    after = pcie_host.devs_pcie(hp, k)
    # node ordinals are first-seen, so they renumber; what holds is which vGPUs share a node
    assert before["300"] == before["304"] != before["303"]
    assert after["300"] == after["303"] != after["304"]
    moved = dict(GPU_OF, **{"300": ORDER[3]})
    for a in IDS:
        for b in IDS:
            assert (after[a] == after[b]) == (moved[a] == moved[b]), (a, b)
    got = topo_host.preferred_allocation(hp, k, [(IDS, ["300"], 5)])[0]
    assert {GPU_OF[x] for x in got if x != "300"} == {ORDER[3]}  # 300 and D's four
    hp.close()
