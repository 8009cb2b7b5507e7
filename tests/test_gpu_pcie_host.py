"""GPU end to end of the host plugin's PCIe topology (Plugin::pcieTopologyAware) on the worked example's fake sysfs: the
nodes the Devices carry, the options, GetPreferredAllocation on the example's table, and a rediscovery after one GPU's
link moved under the other switch."""
import ctypes as C
import json

import pytest

import fake_sysfs
import pcie_example as EX
import pcie_host
import topo_host

pytestmark = pytest.mark.gpu
NV = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")


def _plugin(tmp_path, kx, pci_text):
    root = str(tmp_path)
    devs = [dict(bdf=bdf, path=path, group=g, **NV) for (bdf, path), g in zip(EX.gpu_paths(), EX.GROUPS)]
    base = pcie_host.make_nested_tree(root, devs, relative=True)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    (tmp_path / "cdi").mkdir()
    return fake_sysfs.HostPlugin(kx, base, str(tmp_path / "pci.ids"), str(tmp_path / "cdi") + "/")


def _rediscover(hp):
    hp.L.kxh_rediscover.restype = C.c_int
    hp.L.kxh_rediscover.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(1 << 20)
    assert hp.L.kxh_rediscover(hp.h, b"YAML", buf, len(buf)) >= 0, buf.value
    return json.loads(buf.value.decode())


def _ids(groups):
    return [str(g) for g in groups]


def test_host_pcie_end_to_end(tmp_path, kx, pci_text):
    off = _plugin(tmp_path, kx, pci_text)
    a = off.init("YAML")
    assert topo_host.options(off)["GetPreferredAllocationAvailable"] is False
    assert set(pcie_host.devs_pcie(off, 0).values()) == {0xFFFFFFFF}
    off.close()

    hp = fake_sysfs.HostPlugin(kx, str(tmp_path / "bus" / "pci" / "devices"), str(tmp_path / "pci.ids"),
                               str(tmp_path / "cdi") + "/")
    pcie_host.set_pcie(hp, True)
    topo_host.set_topology(hp, True)  # both settings on together
    b = hp.init("YAML")
    for k in ("iommuMap", "deviceMap", "plugins", "cdiFile"):
        assert a[k] == b[k], k
    assert topo_host.options(hp) == dict(PreStartRequired=False, GetPreferredAllocationAvailable=True)
    assert pcie_host.devs_pcie(hp, 0) == dict(zip(_ids(EX.GROUPS), [3, 4, 7, 8, 12, 13, 16, 17]))
    assert topo_host.devs_numa(hp, 0) == dict(zip(_ids(EX.GROUPS), [0] * 8))  # no numa_node files in this tree
    reqs = [(_ids(av), _ids(mu), size) for av, mu, size, _ in EX.TABLE]
    assert topo_host.preferred_allocation(hp, 0, reqs) == [_ids(ans) for _, _, _, ans in EX.TABLE]
    with pytest.raises(RuntimeError, match="unknown device: 99"):
        topo_host.preferred_allocation(hp, 0, [(["10", "99"], [], 1)])

    # GPU 10 (0000:03:00.0) moves under the second switch of socket 0: a third down port of 0000:05:00.0
    before = topo_host.preferred_allocation(hp, 0, [(_ids([10, 11, 12, 13]), ["12"], 2), (_ids([10, 11, 12, 13]), [], 1)])
    assert before == [["12", "13"], ["10"]]
    pcie_host.move_link(str(tmp_path), "0000:03:00.0",
                        "pci0000:00/0000:00:02.0/0000:05:00.0/0000:06:02.0/0000:03:00.0")
    rep = _rediscover(hp)
    assert rep is not None
    assert pcie_host.devs_pcie(hp, 0) == dict(zip(_ids(EX.GROUPS), [3, 6, 7, 8, 12, 13, 16, 17]))
    after = topo_host.preferred_allocation(hp, 0, [(_ids([10, 11, 12, 13]), ["12"], 2), (_ids([10, 11, 12, 13]), [], 1)])
    assert after == [["12", "10"], ["11"]]
    hp.close()
