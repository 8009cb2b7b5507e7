"""GPU end to end of Plugin::draPcieDomain on a fake tree: pcie_example's eight GPUs in one class and, in a second
class with its own DRA driver, a NIC PF on its vendor driver below the first switch of each socket with VFs on
vfio-pci.  With the setting the GPU and NIC-VF pools publish equal pcieSwitch values exactly where they share a switch;
with sriovPfAware too a VF carries its PF and its ports; a rediscovery that moves a GPU under another switch moves the
generation and one that changes nothing does not; the read counters do not depend on the setting; with the setting
empty every output and generation is as without it."""
import os

import pytest

import dra_host as DH
import dra_pcie_host as H
import dra_pf_host as PFH
import fake_sysfs
import pcie_example as EX
import pcie_host
import sriov_host as SH

pytestmark = pytest.mark.gpu


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = H.make_tree(root)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    (tmp_path / "cdi").mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(tmp_path / "cdi") + "/"


def _plugin(kx, tree, domain=None, sriov=False):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, classes=H.CLASSES, dra=H.DRIVERS)
    if sriov:
        SH.set_sriov(hp, True)
        PFH.enable(hp, True)
    if domain is not None:
        H.set_domain(hp, domain)
    return hp


def _clear(cdi):
    for f in os.listdir(cdi):
        os.remove(os.path.join(cdi, f))


def _outputs(hp, tree, state):
    cdi = tree[3]
    return dict(lw=[hp.list_and_watch(k) for k in range(len(state["plugins"]))],
                specs={f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))},
                slices=[DH.slices(hp, c) for c in range(2)], gen=DH.generation(hp), state=state)


def _run(kx, tree, domain=None, sriov=False):
    _clear(tree[3])
    hp = _plugin(kx, tree, domain, sriov)
    counter = DH.Counter(hp)
    try:
        out = _outputs(hp, tree, hp.init("YAML"))
        out["reads"] = counter.reads()
        return out
    finally:
        hp.close()


def _same_slices(a, b):
    for (x, xo), (y, yo) in zip(a, b):
        assert x == y and list(xo) == list(yo)


def test_empty_changes_nothing(kx, tree):
    unset, empty = _run(kx, tree), _run(kx, tree, "")
    _same_slices(unset.pop("slices"), empty.pop("slices"))
    assert unset == empty
    assert not any(H.RP in d["attributes"] for d in H.devices_of(_run(kx, tree)["slices"][0][0]).values())


def test_pools_share_switches(kx, tree):
    off, on = _run(kx, tree), _run(kx, tree, H.DOMAIN)
    for k in ("lw", "specs", "gen", "reads"):  # only the slices differ; no new file or link is read
        assert on[k] == off[k], k
    gpu, nic = H.devices_of(on["slices"][0][0]), H.devices_of(on["slices"][1][0])
    gpu_off, nic_off = H.devices_of(off["slices"][0][0]), H.devices_of(off["slices"][1][0])
    assert set(gpu) == {"vfio%d" % g for g in EX.GROUPS} and set(nic) == {"vfio71", "vfio72", "vfio81"}
    want = dict(zip(EX.GROUPS, [("0000:00:01.0", "0000:01:00.0")] * 2 + [("0000:00:02.0", "0000:05:00.0")] * 2 +
                    [("0000:80:01.0", "0000:81:00.0")] * 2 + [("0000:80:02.0", "0000:85:00.0")] * 2))
    for g, (rp, sw) in want.items():
        a = dict(gpu["vfio%d" % g]["attributes"])
        assert a.pop(H.RP) == {"string": rp} and a.pop(H.SW) == {"string": sw}
        assert a == gpu_off["vfio%d" % g]["attributes"]
    for name, (rp, sw) in (("vfio71", want[10]), ("vfio72", want[10]), ("vfio81", want[20])):
        a = dict(nic[name]["attributes"])
        assert a.pop(H.RP) == {"string": rp} and a.pop(H.SW) == {"string": sw}
        assert a == nic_off[name]["attributes"]
    # a claim matching pcieSwitch across the two pools: exactly the GPUs below the NIC VF's switch
    for name in nic:
        sw = nic[name]["attributes"][H.SW]
        same = sorted(int(d[4:]) for d, v in gpu.items() if v["attributes"][H.SW] == sw)
        assert same == ([10, 11] if name != "vfio81" else [20, 21])


def test_with_sriov_pf_aware(kx, tree):
    off, on = _run(kx, tree, sriov=True), _run(kx, tree, H.DOMAIN, sriov=True)
    nic, nic_off = H.devices_of(on["slices"][1][0]), H.devices_of(off["slices"][1][0])
    for name, pf in (("vfio71", H.PF_A), ("vfio72", H.PF_A), ("vfio81", H.PF_B)):
        a = dict(nic[name]["attributes"])
        assert a["physfnAddress"] == {"string": pf} and a["physfnDeviceID"] == {"string": "101e"}
        assert a.pop(H.RP)["string"] in ("0000:00:01.0", "0000:80:01.0") and H.SW in a
        a.pop(H.SW)
        assert a == nic_off[name]["attributes"]
    assert on["reads"] == off["reads"] and on["gen"] == off["gen"]


def test_rediscover(kx, tree):
    root = tree[0]
    _clear(tree[3])
    hp = _plugin(kx, tree, H.DOMAIN)
    try:
        hp.init("YAML")
        gen, blob = DH.generation(hp), DH.slices(hp, 0)[0]
        DH.rediscover(hp)  # nothing changed: same bytes, same generation
        assert DH.generation(hp) == gen and DH.slices(hp, 0)[0] == blob
        # GPU 10 (0000:03:00.0) moves below socket 0's second switch
        pcie_host.move_link(root, "0000:03:00.0", "pci0000:00/0000:00:02.0/0000:05:00.0/0000:06:02.0/0000:03:00.0")
        DH.rediscover(hp)
        assert DH.generation(hp) == gen + 1
        a = H.devices_of(DH.slices(hp, 0)[0])["vfio10"]["attributes"]
        assert a[H.RP] == {"string": "0000:00:02.0"} and a[H.SW] == {"string": "0000:05:00.0"}
        DH.rediscover(hp)
        assert DH.generation(hp) == gen + 1
    finally:
        hp.close()
    # without the setting the same move does not move the generation: nothing it publishes changed
    _clear(tree[3])
    pcie_host.move_link(root, "0000:03:00.0", EX.gpu_paths()[0][1])
    hp = _plugin(kx, tree)
    try:
        hp.init("YAML")
        gen = DH.generation(hp)
        pcie_host.move_link(root, "0000:03:00.0", "pci0000:00/0000:00:02.0/0000:05:00.0/0000:06:02.0/0000:03:00.0")
        DH.rediscover(hp)
        assert DH.generation(hp) == gen
    finally:
        hp.close()
