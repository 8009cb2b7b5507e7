"""GPU end to end of the host plugin publishing vGPUs on SR-IOV VFs as DRA ResourceSlices (XpuClass::vgpuDraDriver,
Plugin::VfVgpuResourceSlices) on a fake sysfs tree: a PF on the vGPU manager's driver with eight VFs, three of type 557,
two of type 558, one of a type no list names and two free ones, next to a passthrough function of a class with a
draDriver.  The pool holds exactly the five named VFs, beside the passthrough pool; prepare answers Allocate's CDI names
(also with vfioCdev and resumeIndices) and refuses a VF whose type changed; rediscover after a type change moves the
generation and the device's vgpuType; health and AER taints reach the pool; with the field unset the reads, slices and
generation are those of the plugin without it."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import aer_host as AH
import cdev_host as CH
import dra_host as DH
import dra_vf_vgpu_cases as VC
import dra_vf_vgpu_host as VH
import dra_vf_vgpu_oracle as VO
import fake_sysfs
import sriov_host as SH
import vf_vgpu_host as H
from oracle import oracle as O
from test_gpu_dra_taint_host import T0, Watched, _lib as taint_lib, refresh

pytestmark = pytest.mark.gpu

VDRV, PDRV = "vgpu-vf.nvidia.com", "vfio.nvidia.com"
PT = dict(bdf="0000:c1:00.0", group=214, vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
VF = dict(vendor=b"0x10de\n", device=b"0x2331\n", driver="nvidia")
PF = "0000:03:00.0"
VFS = ["0000:03:00.%d" % k for k in range(1, 8)] + ["0000:03:01.0"]
GROUP = {PF: 30, **{bdf: 31 + k for k, bdf in enumerate(VFS)}}
TYPE = {VFS[0]: 557, VFS[1]: 557, VFS[2]: 557, VFS[3]: 558, VFS[4]: 558, VFS[5]: 999}  # VFS[6:] are free
LIST = H.HEADER + b"557   : NVIDIA H100-4C\n558   : NVIDIA H100-8C\n"
KEY = {557: b"NVIDIA_H100-4C", 558: b"NVIDIA_H100-8C"}
PUBLISHED = ["vfio%d" % g for g in range(31, 36)]


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    devs = [PT, dict(bdf=PF, group=30, vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia")]
    devs += [dict(bdf=bdf, group=GROUP[bdf], **VF) for bdf in VFS]
    base = fake_sysfs.make_tree(root, devs)
    SH.link_vfs(base, PF, VFS, b"8\n")
    for k, d in enumerate(devs):
        CH.set_vfio_dev(base, d["bdf"], ["vfio%d" % (200 + k)])
        open(os.path.join(root, "devices", d["bdf"], "numa_node"), "wb").write(b"1\n")
    for bdf in VFS:
        t = TYPE.get(bdf, 0)
        H.set_files(base, bdf, b"%d\n" % t, H.HEADER if t else LIST)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return root, base, str(tmp_path / "pci.ids"), str(cdi) + "/"


def _plugin(kx, tree, vdrv=VDRV, pdrv=PDRV, cdev=False, resume=False):
    root, base, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    assert hp.L.kxh_set_classes(hp.h, (H.CLASSES + (",cdev" if cdev else "")).encode()) == 0
    H.set_vf_vgpu(hp, 1)
    DH.configure(hp, dra=[pdrv or "", ""])
    if vdrv:
        VH.set_driver(hp, 1, vdrv)
    hp.L.kxh_set_resume.argtypes = [C.c_void_p, C.c_int]
    hp.L.kxh_set_resume(hp.h, int(resume))
    return hp


def _start(hp):
    """InitiateDevicePlugin with its configuration checks, then the plugin's state"""
    err = DH.initiate(hp)
    assert err is None, err
    hp.L.kxh_state.restype = C.c_int
    hp.L.kxh_state.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(1 << 22)
    assert hp.L.kxh_state(hp.h, buf, len(buf)) >= 0
    return json.loads(buf.value.decode())


def _devices(blob):
    return {d["name"]: d for line in blob.splitlines() for d in json.loads(line)["spec"]["devices"]}


def _product(pci_text):
    name = O.lookup_many(pci_text, [0x10de2330])[1][0]
    return name if isinstance(name, bytes) else name.encode()


def _expected(pci_text, types=None):
    """the records the pool publishes, from the test's own tree description"""
    types = types or TYPE
    recs = [VC.rec(group=GROUP[bdf], type_key=KEY[types[bdf]], type_id=types[bdf], bdf=bdf.encode(), parent=PF.encode(),
                   root=b"", vendor=b"10de", device=b"2330", product=_product(pci_text), numa=1 << 1)
            for bdf in VFS[:5]]
    return np.concatenate(recs)


def _served(state, name):
    return next(k for k, p in enumerate(state["plugins"]) if p["name"] == name)


def test_pool_holds_the_vgpu_vfs(kx, tree, pci_text):
    hp = _plugin(kx, tree)
    try:
        _start(hp)
        blob, offs = VH.slices(hp, 1)
        want, woffs = VO.dra_slices_vf_vgpu(VDRV, "node-a", "node-a", 1, _expected(pci_text))
        assert blob == want and np.array_equal(offs, woffs)
        devs = _devices(blob)
        assert list(devs) == PUBLISHED  # neither the PF (30), the unnamed VF (36) nor the free VFs (37, 38)
        a = devs["vfio31"]["attributes"]
        assert a["parentAddress"] == {"string": PF} and a["pciAddress"] == {"string": VFS[0]}
        assert a["parentDeviceID"] == {"string": "2330"} and a["numaNode"] == {"int": 1}
        assert a["vgpuType"] == {"string": "NVIDIA_H100-4C"} and a["vgpuTypeID"] == {"int": 557}
        # the passthrough pool beside it: its class's group only, same generation
        pblob, _ = DH.slices(hp, 0)
        assert list(_devices(pblob)) == ["vfio214"]
        assert DH.generation(hp) == 1 and b'"generation":1,' in pblob
        with pytest.raises(RuntimeError, match="VfVgpuResourceSlices: class 0 has no vGPU DRA driver"):
            VH.slices(hp, 0)
    finally:
        hp.close()


@pytest.mark.parametrize("cdev", [False, True])
@pytest.mark.parametrize("resume", [False, True])
def test_prepare_answers_allocate(kx, tree, cdev, resume):
    hp = _plugin(kx, tree, cdev=cdev, resume=resume)
    try:
        _start(hp)
        got = DH.prepare(hp, VDRV, "node-a", ["vfio31", "vfio35"])
        assert got == [hp.allocate(["31"])["cdi_devices"], hp.allocate(["35"])["cdi_devices"]]
        assert all(n.startswith("nvidia.com/vgpu=") for ids in got for n in ids)
        assert DH.prepare(hp, PDRV, "node-a", ["vfio214"]) == [hp.allocate(["214"])["cdi_devices"]]
        for name in ("vfio30", "vfio36", "vfio37", "vfio214"):
            with pytest.raises(RuntimeError, match="unknown device %s in pool node-a" % name):
                DH.prepare(hp, VDRV, "node-a", [name])
        with pytest.raises(RuntimeError, match="unknown pool node-b"):
            DH.prepare(hp, VDRV, "node-b", ["vfio31"])
    finally:
        hp.close()


def test_type_change(kx, tree, pci_text):
    root, base = tree[0], tree[1]
    hp = _plugin(kx, tree)
    try:
        _start(hp)
        H.set_files(base, VFS[0], b"558\n")  # no uevent: prepare's Allocate re-reads the type
        with pytest.raises(RuntimeError, match="0000:03:00.1 carries vGPU type 558, not type 557 as discovered"):
            DH.prepare(hp, VDRV, "node-a", ["vfio31"])
        assert DH.generation(hp) == 1
        DH.rediscover(hp)
        assert DH.generation(hp) == 2  # the VF moved to the other type's plugin
        blob, _ = VH.slices(hp, 1)
        want, _ = VO.dra_slices_vf_vgpu(VDRV, "node-a", "node-a", 2, _expected(pci_text, {**TYPE, VFS[0]: 558}))
        assert blob == want
        a = _devices(blob)["vfio31"]["attributes"]
        assert a["vgpuType"] == {"string": "NVIDIA_H100-8C"} and a["vgpuTypeID"] == {"int": 558}
        assert DH.prepare(hp, VDRV, "node-a", ["vfio31"]) == [hp.allocate(["31"])["cdi_devices"]]
        DH.rediscover(hp)
        assert DH.generation(hp) == 2  # nothing changed
    finally:
        hp.close()


def test_taints(kx, tree, tmp_path):
    root, base = tree[0], tree[1]
    hp = _plugin(kx, tree)
    taint_lib().kxh_set_dra_taints(hp.h, 1)
    clock = C.c_int64(T0)
    taint_lib().kxh_set_clock(hp.h, C.byref(clock))
    AH.enable(hp, True)
    w = None
    try:
        state = _start(hp)
        assert DH.generation(hp) == 1
        blob, offs = VH.slices(hp, 1)
        assert b'"taints"' not in blob and len(offs) == 2  # 64 devices per slice with draTaints
        w = Watched(hp, tmp_path, _served(state, "NVIDIA_H100-4C"), ["31", "32", "33"])
        w.remove("32")
        assert refresh(hp) == (True, False) and DH.generation(hp) == 2
        devs = _devices(VH.slices(hp, 1)[0])
        assert devs["vfio32"]["taints"] == [{"key": VDRV + "/unhealthy", "value": "vfio-device-missing",
                                             "effect": "NoSchedule", "timeAdded": "2026-01-01T00:00:00Z"}]
        assert "taints" not in devs["vfio31"] and b'"taints"' not in DH.slices(hp, 0)[0]
        with pytest.raises(RuntimeError, match="device vfio32 is tainted " + VDRV + "/unhealthy=vfio-device-missing"):
            DH.prepare(hp, VDRV, "node-a", ["vfio32"])
        clock.value = T0 + 60
        AH.write(os.path.join(base, VFS[3]), fatal=1)
        assert AH.refresh(hp)[1:] == (True, False) and DH.generation(hp) == 3
        devs = _devices(VH.slices(hp, 1)[0])
        assert devs["vfio34"]["taints"] == [{"key": VDRV + "/pcie-aer", "value": "fatal", "effect": "NoSchedule",
                                             "timeAdded": "2026-01-01T00:01:00Z"}]
        assert DH.prepare(hp, VDRV, "node-a", ["vfio34"]) == [hp.allocate(["34"])["cdi_devices"]]
        w.create("32")
        assert refresh(hp) == (True, False) and DH.generation(hp) == 4
        assert "taints" not in _devices(VH.slices(hp, 1)[0])["vfio32"]
    finally:
        if w:
            w.stop()
        hp.close()


def test_unset_changes_nothing(kx, tree):
    """without a vgpuDraDriver every read, the passthrough slices and the generation are those of the plugin that only
    publishes the passthrough class; with neither driver nothing NUMA or path related is read at all"""
    runs = []
    for vdrv, pdrv in ((None, PDRV), (VDRV, PDRV), (None, None)):
        for f in os.listdir(tree[3]):
            os.remove(os.path.join(tree[3], f))
        hp = _plugin(kx, tree, vdrv=vdrv, pdrv=pdrv)
        counter = DH.Counter(hp)
        try:
            state = _start(hp)
            specs = {f: open(os.path.join(tree[3], f), "rb").read() for f in sorted(os.listdir(tree[3]))}
            lw = [hp.list_and_watch(k) for k in range(len(state["plugins"]))]
            DH.rediscover(hp)
            runs.append(dict(reads=counter.reads(), vf=H.reads(hp), gen=DH.generation(hp), state=state, specs=specs, lw=lw,
                             slices=DH.slices(hp, 0)[0] if pdrv else None))
        finally:
            hp.close()
    unset, both, none = runs
    assert unset["reads"] == both["reads"] and unset["reads"][0] > 0 and unset["reads"][1] > 0
    assert none["reads"] == (0, 0)
    for k in ("vf", "gen", "state", "specs", "lw", "slices"):
        assert unset[k] == both[k], k
    for k in ("vf", "gen", "specs", "lw"):
        assert unset[k] == none[k], k
