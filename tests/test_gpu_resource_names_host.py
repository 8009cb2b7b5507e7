"""GPU end to end of XpuClass::resourceNames on fake sysfs trees: {"*": "pgpu"} over three H100 variants serves one
nvidia.com/pgpu plugin with every group in walk order; two ids with one pci.ids name (GH100) share one plugin; the CDI
spec, Allocate's CDI names and the DRA slices (productName the model name) are byte-identical with and without the
names, and so is ListAndWatch where the plugins correspond; GetPreferredAllocation packs by NUMA node across the merged
ids; rediscover adds a new id to pgpu in place; the metrics carry the alias."""
import os

import pytest

import dra_host as DH
import fake_sysfs
import metrics_host as MH
import test_resource_names as T
import topo_host

pytestmark = pytest.mark.gpu
NV = dict(vendor=b"0x10de\n", driver="vfio-pci")
MIXED = [("0000:03:00.0", 10, b"0x2331\n"), ("0000:04:00.0", 11, b"0x2330\n"), ("0000:05:00.0", 12, b"0x2321\n"),
         ("0000:06:00.0", 13, b"0x2330\n"), ("0000:07:00.0", 14, b"0x2331\n")]
NUMA = {"0000:03:00.0": b"0\n", "0000:04:00.0": b"1\n", "0000:05:00.0": b"0\n", "0000:06:00.0": b"1\n",
        "0000:07:00.0": b"1\n"}


def _tree(tmp_path, pci_text, devs, name="t"):
    root = tmp_path / name
    root.mkdir()
    base = fake_sysfs.make_tree(str(root), [dict(bdf=b, group=g, device=d, **NV) for b, g, d in devs])
    (root / "pci.ids").write_bytes(pci_text)
    (root / "cdi").mkdir()
    return str(root), base, str(root / "pci.ids"), str(root / "cdi") + "/"


def _plugin(kx, tree, names=None, dra=True, topo=False):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, dra=["gpu.nvidia.com"] if dra else None, topo=topo)
    if names:
        T.set_names(hp, 0, names)
    return hp


def _plugins(state):
    return [(p["resource"], [d[0] for d in p["devs"]]) for p in state["plugins"]]


def _slices(hp):
    blob, off = DH.slices(hp, 0)
    return bytes(blob), [int(x) for x in off]


def _spec(tree):
    cdi = tree[3]
    return {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}


def test_one_pgpu_plugin(kx, tmp_path, pci_text):
    tree = _tree(tmp_path, pci_text, MIXED)
    off = _plugin(kx, tree)
    a = off.init("YAML")
    spec_off, alloc_off, slices_off = _spec(tree), off.allocate(["10", "12", "14"]), _slices(off)
    assert len(a["plugins"]) == 3
    off.close()
    hp = _plugin(kx, tree, {"*": "pgpu"})
    b = hp.init("YAML")
    assert _plugins(b) == [("nvidia.com/pgpu", ["10", "11", "12", "13", "14"])]
    assert b["iommuMap"] == a["iommuMap"] and b["cdiFile"] == a["cdiFile"]
    assert _spec(tree) == spec_off
    assert hp.allocate(["10", "12", "14"]) == alloc_off
    assert _slices(hp) == slices_off  # productName stays the model name of each group
    assert b"GH100_H100_SXM5_80GB" in slices_off[0] and b"pgpu" not in slices_off[0]
    hp.close()


def test_listed_ids_and_star(kx, tmp_path, pci_text):
    tree = _tree(tmp_path, pci_text, MIXED)
    hp = _plugin(kx, tree, {"2321": "h100l", "*": "pgpu"})
    assert _plugins(hp.init("YAML")) == [("nvidia.com/pgpu", ["10", "11", "13", "14"]), ("nvidia.com/h100l", ["12"])]
    hp.close()


def test_same_pci_ids_name_shares_one_plugin(kx, tmp_path, pci_text):
    tree = _tree(tmp_path, pci_text, [("0000:03:00.0", 10, b"0x2302\n"), ("0000:04:00.0", 11, b"0x2343\n"),
                                      ("0000:05:00.0", 12, b"0x22a3\n")])
    off = _plugin(kx, tree, dra=False)
    a = off.init("YAML")
    assert [p["name"] for p in a["plugins"]].count("GH100") == 2  # two plugins, one socket: the collision
    off.close()
    hp = _plugin(kx, tree, {"22a3": "nvswitch"}, dra=False)
    b = hp.init("YAML")
    assert _plugins(b) == [("nvidia.com/GH100", ["10", "11"]), ("nvidia.com/nvswitch", ["12"])]
    hp.close()


def test_list_and_watch_bytes(kx, tmp_path, pci_text):
    tree = _tree(tmp_path, pci_text, [d for d in MIXED if d[2] == b"0x2330\n"])
    off = _plugin(kx, tree)
    off.init("YAML")
    lw, spec, sl = off.list_and_watch(0), _spec(tree), _slices(off)
    off.close()
    hp = _plugin(kx, tree, {"*": "pgpu"})
    assert _plugins(hp.init("YAML")) == [("nvidia.com/pgpu", ["11", "13"])]
    assert hp.list_and_watch(0) == lw and _spec(tree) == spec and _slices(hp) == sl
    hp.close()


def test_preferred_allocation_across_ids(kx, tmp_path, pci_text):
    tree = _tree(tmp_path, pci_text, MIXED)
    topo_host.add_numa(tree[0], NUMA)
    hp = _plugin(kx, tree, {"*": "pgpu"}, topo=True)
    hp.init("YAML")
    assert topo_host.devs_numa(hp, 0) == {"10": 1, "11": 2, "12": 1, "13": 2, "14": 2}
    # node 1 holds three of the five (2330, 2330, 2331): a request of 3 stays there
    assert topo_host.preferred_allocation(hp, 0, [(["10", "11", "12", "13", "14"], [], 3)]) == [["11", "13", "14"]]
    assert topo_host.preferred_allocation(hp, 0, [(["10", "11", "12", "13", "14"], ["12"], 2)]) == [["12", "10"]]
    hp.close()


def test_rediscover_joins_in_place(kx, tmp_path, pci_text):
    tree = _tree(tmp_path, pci_text, MIXED[:2])
    hp = _plugin(kx, tree, {"*": "pgpu"})
    assert _plugins(hp.init("YAML")) == [("nvidia.com/pgpu", ["10", "11"])]
    root, bdf = tree[0], "0000:05:00.0"  # a third variant appears, as make_tree builds an entry
    d = os.path.join(root, "devices", bdf)
    os.makedirs(d)
    open(os.path.join(d, "vendor"), "wb").write(b"0x10de\n")
    open(os.path.join(d, "device"), "wb").write(b"0x2321\n")
    os.symlink(os.path.join(root, "drivers", "vfio-pci"), os.path.join(d, "driver"))
    os.makedirs(os.path.join(root, "iommu_groups", "12"))
    os.symlink(os.path.join(root, "iommu_groups", "12"), os.path.join(d, "iommu_group"))
    os.symlink(d, os.path.join(tree[1], bdf))
    r = DH.rediscover(hp)
    assert r["report"]["added"] == [] and r["report"]["changed"] == [0]
    assert _plugins(r) == [("nvidia.com/pgpu", ["10", "11", "12"])]
    hp.close()


def test_metrics_carry_the_alias(kx, tmp_path, pci_text):
    tree = _tree(tmp_path, pci_text, MIXED)
    hp = _plugin(kx, tree, {"*": "pgpu"})
    hp.init("YAML")
    st = MH.state(hp)
    MH.scrape(hp, tree[3], MH.document(st))
    assert all(p["resource"] == "nvidia.com/pgpu" for p in st["plugins"])
    hp.close()
