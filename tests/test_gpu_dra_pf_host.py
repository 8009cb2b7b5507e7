"""GPU end to end of Plugin::sriovPfAware on a fake tree: PF A (0000:4d:00.0, on its vendor driver) with three VFs on
vfio-pci, PF B with two, and a plain function with none, all of one passthrough class.  With the setting on each VF's
slice device carries its PF's address and device id, and the plain function's bytes do not change; a fatal count in PF
A's aer_dev_fatal makes exactly its three VFs Unhealthy with a reason naming the PF, taints them pcie-aer=fatal and shows
in the metrics, while PF B's VFs stay Healthy; each PF's files are read once per refresh; the setting is refused
without sriovAware; a rediscovery after PF A's VFs are re-created keeps every CDI index and moves the pool generation
when what a VF publishes about its PF changed.  With the setting off every output is as without it."""
import ctypes as C
import json
import os

import pytest

import aer_host as AH
import dra_host as DH
import dra_pf_host as H
import fake_sysfs
import metrics_host as MX
import sriov_host as SH
from test_gpu_dra_taint_host import T0, _lib as taint_lib
from test_metrics import host_metrics

pytestmark = pytest.mark.gpu

FATAL = H.PF_A + " reported 1 fatal uncorrectable PCIe errors (limit 0)"
SERVED = 6  # the five VFs and the plain function


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = H.make_tree(root)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, on=True, clock=None):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, classes=H.CLASSES, dra=[H.DRIVER])
    SH.set_sriov(hp, True)
    if on is not None:
        H.enable(hp, on)
    AH.enable(hp, True)
    if clock is not None:
        taint_lib().kxh_set_dra_taints(hp.h, 1)
        taint_lib().kxh_set_clock(hp.h, clock)
    return hp


def _devices(blob):
    return {d["name"]: d for line in blob.splitlines() for d in json.loads(line)["spec"]["devices"]}


def _clear(cdi):
    for f in os.listdir(cdi):
        os.remove(os.path.join(cdi, f))


def _indices(state):
    return {m[0]: m[1] for _, ms in state["iommuMap"] for m in ms}


def _outputs(hp, tree, state):
    cdi = tree[3]
    return dict(lw=[hp.list_and_watch(k) for k in range(len(state["plugins"]))],
                specs={f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))},
                slices=DH.slices(hp, 0)[0], metrics=host_metrics(hp), gen=DH.generation(hp))


def test_off_changes_nothing(kx, tree):
    """the setting left alone and the setting set off: the same bytes, counters and reads, a fatal PF error included"""
    base = tree[1]
    AH.write(os.path.join(base, H.PF_A), fatal=1)
    runs = []
    for on in (None, False):
        _clear(tree[3])
        clock = C.c_int64(T0)
        hp = _plugin(kx, tree, on=on, clock=C.byref(clock))
        try:
            state = hp.init("YAML")
            a0 = AH.reads(hp)
            AH.refresh(hp)
            runs.append(dict(_outputs(hp, tree, state), aer=AH.reads(hp) - a0, counters=MX.counters(hp)))
        finally:
            hp.close()
    assert runs[0] == runs[1]
    assert runs[0]["aer"] == 2 * SERVED  # the PFs are no members: never read
    assert all("physfnAddress" not in d["attributes"] for d in _devices(runs[0]["slices"]).values())


def test_pool_carries_the_pf(kx, tree):
    _clear(tree[3])
    off = _plugin(kx, tree, on=False)
    try:
        out_off = _outputs(off, tree, off.init("YAML"))
        want = _devices(out_off["slices"])
    finally:
        off.close()
    _clear(tree[3])
    hp = _plugin(kx, tree)
    try:
        out_on = _outputs(hp, tree, hp.init("YAML"))
        for k in ("lw", "specs", "gen"):  # only the slices differ
            assert out_on[k] == out_off[k], k
        devs = _devices(DH.slices(hp, 0)[0])
        assert set(devs) == set(want)
        for groups, pf in ((H.GROUPS_A, H.PF_A), (H.GROUPS_B, H.PF_B)):
            for g in groups:
                a = dict(devs["vfio" + g]["attributes"])
                assert a.pop("physfnAddress") == {"string": pf} and a.pop("physfnDeviceID") == {"string": "56c0"}
                assert a == want["vfio" + g]["attributes"]  # every other attribute as without the setting
        assert devs["vfio60"] == want["vfio60"]
    finally:
        hp.close()


def test_pf_aer_on_its_vfs(kx, tree):
    base = tree[1]
    clock = C.c_int64(T0)
    hp = _plugin(kx, tree, clock=C.byref(clock))
    try:
        state = hp.init("YAML")
        assert len(state["plugins"]) == 1
        assert set(AH.health(hp, 0).values()) == {"Healthy"}
        gen = DH.generation(hp)
        a0 = AH.reads(hp)
        AH.write(os.path.join(base, H.PF_A), fatal=1)
        changed, moved, _ = AH.refresh(hp)
        assert AH.reads(hp) - a0 == 2 * (SERVED + 2)  # each served function, then each distinct PF once
        assert changed == [0] and moved and DH.generation(hp) == gen + 1
        others = {g: "" for g in H.GROUPS_B + ["60"]}
        assert AH.reasons(hp, 0) == {g: FATAL for g in H.GROUPS_A} | others
        assert AH.health(hp, 0) == {g: "Unhealthy" for g in H.GROUPS_A} | {g: "Healthy" for g in others}
        devs = _devices(DH.slices(hp, 0)[0])
        taint = dict(key=H.DRIVER + "/pcie-aer", value="fatal", effect="NoSchedule", timeAdded="2026-01-01T00:00:00Z")
        assert all(devs["vfio" + g]["taints"] == [taint] for g in H.GROUPS_A)
        assert all("taints" not in devs["vfio" + g] for g in others)
        text = host_metrics(hp).decode()
        for g in H.GROUPS_A:  # the PF's count is the group's fatal maximum, and its reason a sample
            assert any(ln.startswith("kata_xpu_pcie_aer_errors{") and 'device="%s"' % g in ln and
                       ln.endswith(',severity="fatal"} 1') for ln in text.splitlines()), text
            assert any(ln.startswith("kata_xpu_device_unhealthy_reason{") and 'device="%s"' % g in ln and FATAL in ln
                       for ln in text.splitlines()), text
        for g in others:
            assert not any(ln.startswith("kata_xpu_device_unhealthy_reason{") and 'device="%s"' % g in ln
                           for ln in text.splitlines()), text
        # a second refresh reads the same files again and moves nothing
        a1 = AH.reads(hp)
        changed, moved, _ = AH.refresh(hp)
        assert AH.reads(hp) - a1 == 2 * (SERVED + 2) and changed == [] and not moved
        # the PF re-enumerated: its counters start at 0 again
        AH.write(os.path.join(base, H.PF_A), fatal=0)
        clock.value = T0 + 60
        changed, moved, _ = AH.refresh(hp)
        assert changed == [0] and moved and set(AH.health(hp, 0).values()) == {"Healthy"}
        assert all("taints" not in d for d in _devices(DH.slices(hp, 0)[0]).values())
    finally:
        hp.close()


def test_refused_without_sriov_aware(kx, tree):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    DH.configure(hp, classes=H.CLASSES, dra=[H.DRIVER])
    H.enable(hp, True)
    try:
        assert DH.initiate(hp) == "sriovPfAware is set but sriovAware is off"
    finally:
        hp.close()


def _recreate_vfs(base, pf, vfs, numvfs, physfn_of=None):
    """echo 0 > sriov_numvfs, then numvfs again: the VFs' physfn / virtfn links go and come back (physfn_of: a VF -> the
    PF its new link names, for a link that moved)"""
    p = os.path.realpath(os.path.join(base, pf))
    for k, vf in enumerate(vfs):
        os.remove(os.path.join(os.path.realpath(os.path.join(base, vf)), "physfn"))
        os.remove(os.path.join(p, "virtfn%d" % k))
    for vf in vfs:
        target = (physfn_of or {}).get(vf, pf)
        v = os.path.realpath(os.path.join(base, vf))
        os.symlink(os.path.relpath(os.path.realpath(os.path.join(base, target)), v), os.path.join(v, "physfn"))
    for k, vf in enumerate(vfs):
        os.symlink(os.path.relpath(os.path.realpath(os.path.join(base, vf)), p), os.path.join(p, "virtfn%d" % k))
    open(os.path.join(p, "sriov_numvfs"), "wb").write(numvfs)


def test_rediscover_after_vfs_recreated(kx, tree):
    base = tree[1]
    hp = _plugin(kx, tree)
    try:
        before = _indices(hp.init("YAML"))
        gen = DH.generation(hp)
        blob = DH.slices(hp, 0)[0]
        # the same VFs again: same addresses and groups, same PF: indices and bytes kept, nothing to republish
        _recreate_vfs(base, H.PF_A, H.VFS_A, b"3\n")
        assert _indices(DH.rediscover(hp)) == before
        assert DH.generation(hp) == gen and DH.slices(hp, 0)[0] == blob
        # PF A now reports another device id (a PF personality switch) and its VFs come back: the VFs publish the new
        # id, so the pool moves; every index is kept
        open(os.path.join(base, H.PF_A, "device"), "wb").write(b"0x56c1\n")
        _recreate_vfs(base, H.PF_A, H.VFS_A, b"3\n")
        assert _indices(DH.rediscover(hp)) == before
        assert DH.generation(hp) == gen + 1
        devs = _devices(DH.slices(hp, 0)[0])
        assert all(devs["vfio" + g]["attributes"]["physfnDeviceID"] == {"string": "56c1"} for g in H.GROUPS_A)
        assert all(devs["vfio" + g]["attributes"]["physfnDeviceID"] == {"string": "56c0"} for g in H.GROUPS_B)
        # one VF's link names PF B after the re-creation: its physfnAddress follows, the pool moves again
        _recreate_vfs(base, H.PF_A, H.VFS_A, b"3\n", physfn_of={H.VFS_A[2]: H.PF_B})
        assert _indices(DH.rediscover(hp)) == before
        assert DH.generation(hp) == gen + 2
        devs = _devices(DH.slices(hp, 0)[0])
        assert devs["vfio43"]["attributes"]["physfnAddress"] == {"string": H.PF_B}
        assert devs["vfio41"]["attributes"]["physfnAddress"] == {"string": H.PF_A}
    finally:
        hp.close()
