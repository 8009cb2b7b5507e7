"""GPU end to end of the host plugin's NUMA topology (Plugin::topologyAware) on a fake two-node sysfs: the device
masks, the ListAndWatch bytes (decoded with the protobuf runtime), GetPreferredAllocation, and an unchanged state with
the setting off."""
import numpy as np
import pytest

import fake_mdev
import fake_sysfs
import pyref_topo as P
import topo_host

pytestmark = pytest.mark.gpu

# two slots on node 0 (groups 10, 11), two on node 1 (groups 20, 21), one with no numa_node (30), one group spanning
# both nodes (40: functions on node 0 and node 1)
DEVS = [("0000:01:00.0", 10, b"0\n"), ("0000:02:00.0", 11, b"0\n"), ("0000:81:00.0", 20, b"1\n"),
        ("0000:82:00.0", 21, b"1\n"), ("0000:90:00.0", 30, None), ("0000:a0:00.0", 40, b"0\n"), ("0000:a0:00.1", 40, b"1\n")]
MASKS = {"10": 1, "11": 1, "20": 2, "21": 2, "30": 0, "40": 3}


def _tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = fake_sysfs.make_tree(root, [dict(bdf=b, vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=g)
                                       for b, g, _ in DEVS])
    topo_host.add_numa(root, {b: raw for b, _, raw in DEVS if raw is not None})
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def test_host_topology_end_to_end(tmp_path, kx, pci_text):
    base, pciids, cdi = _tree(tmp_path, pci_text)
    off = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    a = off.init("YAML")
    lw_off = off.list_and_watch(0)
    assert topo_host.devs_numa(off, 0) == {g: 0 for g in MASKS}
    assert topo_host.options(off)["GetPreferredAllocationAvailable"] is False
    assert topo_host.preferred_allocation(off, 0, [(["10", "20"], [], 1)]) == []
    off.close()

    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    topo_host.set_topology(hp, True)
    b = hp.init("YAML")
    for k in ("iommuMap", "deviceMap", "plugins", "cdiFile"):
        assert a[k] == b[k], k  # the setting changes nothing the plugin already computed
    assert topo_host.devs_numa(hp, 0) == MASKS
    assert topo_host.options(hp) == dict(PreStartRequired=False, GetPreferredAllocationAvailable=True)
    lw = hp.list_and_watch(0)
    ids = [d[0] for d in P.lw_parse(lw)]
    assert P.lw_parse(lw) == [(g, "Healthy", [k for k in range(2) if (MASKS[g] >> k) & 1]) for g in ids]
    assert [(i, h) for i, h, _ in P.lw_parse(lw)] == [(i, h) for i, h, _ in P.lw_parse(lw_off)]
    # 2 of 4 with one must-include device: the other device comes from the same node
    assert topo_host.preferred_allocation(hp, 0, [(["10", "11", "20", "21"], ["20"], 2)]) == [["20", "21"]]
    assert topo_host.preferred_allocation(hp, 0, [(["10", "20", "11", "21"], ["11"], 2), (["30", "21", "20"], [], 2),
                                                  (["10", "20"], [], 0)]) == [["11", "10"], ["20", "21"], []]
    with pytest.raises(RuntimeError, match="unknown device: 99"):
        topo_host.preferred_allocation(hp, 0, [(["10", "99"], [], 1)])
    with pytest.raises(RuntimeError, match="kxpu_preferred_allocation"):
        topo_host.preferred_allocation(hp, 0, [(["10", "11"], ["20"], 2)])  # must-include not available
    hp.close()


def test_host_topology_mdev(tmp_path, kx, pci_text):
    root = str(tmp_path)
    parents = {"0000:01:00.0": b"0x10de\n", "0000:81:00.0": b"0x10de\n"}
    mdevs = [dict(uuid="%08x-0000-4000-8000-%012x" % (i, i), parent=p, group=300 + i)
             for i, p in enumerate(["0000:01:00.0", "0000:01:00.0", "0000:81:00.0", "0000:81:00.0"])]
    base = fake_sysfs.make_tree(root, [])
    mbase = fake_mdev.make_tree(root, mdevs, parents=parents)
    topo_host.add_numa(root, {"0000:01:00.0": b"0\n", "0000:81:00.0": b"1\n"})
    (tmp_path / "pci.ids").write_bytes(pci_text)
    (tmp_path / "cdi").mkdir()
    hp = fake_sysfs.HostPlugin(kx, base, str(tmp_path / "pci.ids"), str(tmp_path / "cdi") + "/")
    fake_mdev.set_vgpu(hp, mbase, [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-vgpu")])
    topo_host.set_topology(hp, True)
    st = hp.init("YAML")
    idx = [i for i, p in enumerate(st["plugins"]) if p["vgpu"]][0]
    assert topo_host.devs_numa(hp, idx) == {"300": 1, "301": 1, "302": 2, "303": 2}
    assert P.lw_parse(hp.list_and_watch(idx))[2] == ("302", "Healthy", [1])
    assert topo_host.preferred_allocation(hp, idx, [(["300", "302", "301", "303"], ["303"], 2)]) == [["303", "302"]]
    hp.close()
