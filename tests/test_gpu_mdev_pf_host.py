"""GPU end to end of Plugin::vgpuSriovAware on a fake tree: an H100 PF 0000:41:00.0 with two VFs carrying three mdevs,
and a second H100 0000:c1:00.0 whose mdev sits on the PF itself.  A fatal count in the PF's aer_dev_fatal makes every
vGPU on its VFs Unhealthy with a reason naming the PF, taints them pcie-aer=fatal, and shows in the metrics; a later
refreshAerHealth after the counter is back to 0 clears both; the PF's files are read once per refresh; the vGPU pool
carries physfnAddress, physfnDeviceID and the PF's model name; the start-up refusal; and with the setting off the same
tree gives the bytes, specs, slices, metrics and counters it gave before, with no physfn read."""
import json
import os

import pytest

import aer_host as AH
import dra_host as DH
import dra_mdev_host as MH
import fake_mdev
import fake_sysfs
import mdev_pf_host as PH
import metrics_host as MX
from oracle import oracle as O
from test_gpu_dra_taint_host import T0, _lib as taint_lib
from test_metrics import host_metrics

pytestmark = pytest.mark.gpu

VGPU = [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")]
NV = dict(vendor=b"0x10de\n", driver="nvidia")
PF, VF4, VF5, PF2 = "0000:41:00.0", "0000:41:00.4", "0000:41:00.5", "0000:c1:00.0"
PARENTS = [
    dict(bdf=PF, group=40, path="pci0000:40/0000:40:01.0/" + PF, device=b"0x2330\n", numa=b"0\n", **NV),
    dict(bdf=VF4, group=44, path="pci0000:40/0000:40:01.0/" + VF4, device=b"0x2331\n", numa=b"0\n", **NV),
    dict(bdf=VF5, group=45, path="pci0000:40/0000:40:01.0/" + VF5, device=b"0x2331\n", numa=b"0\n", **NV),
    dict(bdf=PF2, group=41, path="pci0000:c0/0000:c0:01.0/" + PF2, device=b"0x2330\n", numa=b"1\n", **NV),
]
U = ["0b2ad9a2-6e2c-4a55-9d41-%012x" % k for k in range(8)]
MDEVS = [dict(uuid=U[1], parent=VF4, group=300), dict(uuid=U[2], parent=VF4, group=301),
         dict(uuid=U[3], parent=VF5, group=302), dict(uuid=U[4], parent=PF2, group=303)]
VDRV = "vgpu.nvidia.com"
ON_VFS = {"300", "301", "302"}
FATAL = PF + " reported 1 fatal uncorrectable PCIe errors (limit 0)"


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base, mbase = PH.make_tree(root, PARENTS, MDEVS, [(VF4, PF), (VF5, PF)])
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, mbase, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, on=True, taints=False, clock=None):
    root, base, mbase, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    fake_mdev.set_vgpu(hp, mbase, VGPU)
    MH.set_vgpu_dra(hp, [VDRV], "node-a")
    PH.enable(hp, on)
    AH.enable(hp, True)
    if taints:
        taint_lib().kxh_set_dra_taints(hp.h, 1)
        taint_lib().kxh_set_clock(hp.h, clock)
    return hp


def _start(hp):
    err = DH.initiate(hp)
    assert err is None, err
    return MX.state(hp)


def _vgpu_plugin(state):
    return next(k for k, p in enumerate(state["plugins"]) if p["vgpu"])


def _devices(blob):
    return {d["name"]: d for line in blob.splitlines() for d in json.loads(line)["spec"]["devices"]}


def _clear(cdi):
    for f in os.listdir(cdi):
        os.remove(os.path.join(cdi, f))


def test_pf_aer_on_the_vfs_vgpus(kx, tree):
    import ctypes as C
    base = tree[1]
    clock = C.c_int64(T0)
    hp = _plugin(kx, tree, taints=True, clock=C.byref(clock))
    try:
        state = _start(hp)
        k = _vgpu_plugin(state)
        assert PH.reads(hp) == 4  # one physfn read per grouped mdev
        assert set(AH.health(hp, k).values()) == {"Healthy"}
        a0 = AH.reads(hp)
        AH.write(os.path.join(base, PF), fatal=1)
        changed, _, vmoved = AH.refresh(hp)
        # each mdev's parent files, then the PF's two files once for its three vGPU groups
        assert AH.reads(hp) - a0 == 2 * 4 + 2
        assert changed == [k] and vmoved and MH.generation(hp) == 2
        assert AH.reasons(hp, k) == {g: FATAL for g in ON_VFS} | {"303": ""}
        assert AH.health(hp, k) == {g: "Unhealthy" for g in ON_VFS} | {"303": "Healthy"}
        devs = _devices(MH.slices(hp, 0)[0])
        taint = dict(key=VDRV + "/pcie-aer", value="fatal", effect="NoSchedule", timeAdded="2026-01-01T00:00:00Z")
        assert all(devs["vfio" + g]["taints"] == [taint] for g in ON_VFS) and "taints" not in devs["vfio303"]
        text = host_metrics(hp).decode()
        for g in ON_VFS:  # the PF's count is the group's fatal maximum, and its reason a sample
            assert any(ln.startswith("kata_xpu_pcie_aer_errors{") and 'device="%s"' % g in ln and
                       ln.endswith(',severity="fatal"} 1') for ln in text.splitlines()), text
            assert any(ln.startswith("kata_xpu_device_unhealthy_reason{") and 'device="%s"' % g in ln and FATAL in ln
                       for ln in text.splitlines()), text
        # the PF re-enumerated: its counters start at 0 again
        AH.write(os.path.join(base, PF), fatal=0)
        clock.value = T0 + 60
        changed, _, vmoved = AH.refresh(hp)
        assert changed == [k] and vmoved and MH.generation(hp) == 3
        assert set(AH.reasons(hp, k).values()) == {""} and set(AH.health(hp, k).values()) == {"Healthy"}
        assert all("taints" not in d for d in _devices(MH.slices(hp, 0)[0]).values())
    finally:
        hp.close()


def test_pool_carries_the_pf(kx, tree, pci_text):
    hp = _plugin(kx, tree)
    try:
        _start(hp)
        devs = _devices(MH.slices(hp, 0)[0])
        model = O.lookup_many(pci_text, [0x10de2330])[1][0]
        model = (model if isinstance(model, bytes) else model.encode()).decode()
        for g in ON_VFS:
            a = devs["vfio" + g]["attributes"]
            assert a["physfnAddress"] == {"string": PF} and a["physfnDeviceID"] == {"string": "2330"}
            assert a["productName"] == {"string": model} and a["parentAddress"]["string"] in (VF4, VF5)
            assert a["parentDeviceID"] == {"string": "2331"}
        a = devs["vfio303"]["attributes"]
        assert "physfnAddress" not in a and "physfnDeviceID" not in a and a["parentAddress"] == {"string": PF2}
    finally:
        hp.close()


def test_refused_without_a_vgpu_class(kx, tree):
    root, base, mbase, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    PH.enable(hp, True)
    try:
        assert DH.initiate(hp) == "vgpuSriovAware is set but no vGPU class is configured"
    finally:
        hp.close()


def test_off_changes_nothing(kx, tree):
    """the same tree with the setting off: no physfn read, and every output as without the feature; on, only the
    mdev-on-a-VF devices' attributes and AER differ"""
    base, cdi = tree[1], tree[4]
    runs = {}
    for on in (False, True):
        _clear(cdi)
        hp = _plugin(kx, tree, on=on)
        try:
            state = _start(hp)
            a0 = AH.reads(hp)
            AH.write(os.path.join(base, PF), fatal=1)
            AH.refresh(hp)
            specs = {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}
            runs[on] = dict(lw=[hp.list_and_watch(k) for k in range(len(state["plugins"]))], specs=specs,
                            slices=MH.slices(hp, 0)[0], metrics=host_metrics(hp), counters=MX.counters(hp),
                            reads=PH.reads(hp), aer=AH.reads(hp) - a0, gen=(MH.generation(hp), DH.generation(hp)))
            os.remove(os.path.join(base, PF, "aer_dev_fatal"))
            os.remove(os.path.join(base, PF, "aer_dev_nonfatal"))
        finally:
            hp.close()
    off, on = runs[False], runs[True]
    assert off["reads"] == 0 and on["reads"] == 4
    assert off["specs"] == on["specs"]
    assert off["aer"] + 2 == on["aer"]  # a refresh reads the PF's two files once more
    assert off["lw"] != on["lw"] and off["slices"] != on["slices"]
    off_devs = _devices(off["slices"])
    assert all("physfnAddress" not in d["attributes"] for d in off_devs.values())
    assert off_devs["vfio303"] == _devices(on["slices"])["vfio303"]
