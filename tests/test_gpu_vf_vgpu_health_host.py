"""GPU end to end of Plugin::vfVgpuHealth on the fake tree of test_gpu_dra_vf_vgpu_host (a PF with eight VFs, five of
them carrying named vGPU types, next to a passthrough function): a cleared, restored, unreadable and changed vGPU type
through refreshVfVgpuTypes, then rediscover; the PF's AER counts on every served VF group, each PF file read once; the
fourth taint of the VF-vGPU pool, its generation and PrepareDraDevices' refusal; and with the setting off, nothing more
read and the same bytes."""
import ctypes as C
import os

import pytest

import aer_host as AH
import dra_host as DH
import dra_vf_vgpu_host as VH
import fake_sysfs
import vf_vgpu_host as H
from test_gpu_dra_taint_host import T0, _lib as taint_lib
from test_gpu_dra_vf_vgpu_host import PF, VDRV, VFS, _devices, _plugin, _served, _start, tree  # noqa: F401

pytestmark = pytest.mark.gpu

CHANGED_TAINT = dict(key=VDRV + "/vgpu-type", value="changed", effect="NoSchedule")


def _lib():
    L = fake_sysfs.host_lib()
    L.kxh_set_vf_vgpu_health.argtypes = [C.c_void_p, C.c_int]
    L.kxh_refresh_vf_vgpu_types.restype = C.c_int
    L.kxh_refresh_vf_vgpu_types.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int),
                                            C.c_char_p, C.c_size_t]
    L.kxh_devs_drift.restype = C.c_int
    L.kxh_devs_drift.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    return L


def _health_plugin(kx, tree, on=True, **kw):
    hp = _plugin(kx, tree, **kw)
    _lib().kxh_set_vf_vgpu_health(hp.h, int(on))
    return hp


def refresh(hp):
    """refreshVfVgpuTypes: (changed plugins, passthroughMoved, typesMoved)"""
    changed, n, moved, err = (C.c_size_t * 64)(), C.c_size_t(0), C.c_int(-1), C.create_string_buffer(512)
    assert _lib().kxh_refresh_vf_vgpu_types(hp.h, changed, 64, C.byref(n), C.byref(moved), err, len(err)) == 0, err.value
    return list(changed[:n.value]), bool(moved.value & 1), bool(moved.value & 2)


def drift(hp, idx):
    buf = C.create_string_buffer(1 << 16)
    assert _lib().kxh_devs_drift(hp.h, idx, buf, len(buf)) >= 0
    return dict(kv.split("=", 1) for kv in buf.value.decode().split(",") if kv)


def test_cleared_restored_changed_then_rediscover(kx, tree):
    base = tree[1]
    hp = _health_plugin(kx, tree)
    try:
        state = _start(hp)
        p4, p8 = _served(state, "NVIDIA_H100-4C"), _served(state, "NVIDIA_H100-8C")
        r0 = H.reads(hp)
        assert refresh(hp) == ([], False, False)
        assert H.reads(hp) - r0 == 5  # the five served VFs, not the free, unnamed or PF functions
        assert AH.health(hp, p4) == {"31": "Healthy", "32": "Healthy", "33": "Healthy"}
        H.set_files(base, VFS[0], b"0\n")
        assert refresh(hp) == ([p4], False, False)
        assert drift(hp, p4) == {"31": "0000:03:00.1 now carries vGPU type 0 (was 557)", "32": "", "33": ""}
        assert AH.health(hp, p4) == {"31": "Unhealthy", "32": "Healthy", "33": "Healthy"}
        assert refresh(hp) == ([], False, False)  # still cleared: nothing new to send
        H.set_files(base, VFS[0], b"557\n")
        assert refresh(hp) == ([p4], False, False)
        assert AH.health(hp, p4)["31"] == "Healthy" and drift(hp, p4)["31"] == ""
        os.remove(os.path.join(os.path.realpath(os.path.join(base, VFS[3])), "nvidia", "current_vgpu_type"))
        assert refresh(hp) == ([p8], False, False)
        assert drift(hp, p8)["34"] == "0000:03:00.4 has an unreadable vGPU type (was 558)"
        H.set_files(base, VFS[3], b"558\n")
        before = hp.allocate(["31"])["cdi_devices"]
        H.set_files(base, VFS[0], b"558\n")
        assert refresh(hp) == ([p4, p8], False, True)  # p8 recovered, p4 drifted to another type
        assert drift(hp, p4)["31"] == "0000:03:00.1 now carries vGPU type 558 (was 557)"
        assert AH.health(hp, p4)["31"] == "Unhealthy"
        rep = DH.rediscover(hp)["report"]
        assert p4 in rep["changed"] and p8 in rep["changed"]
        assert AH.health(hp, p4) == {"32": "Healthy", "33": "Healthy"}
        assert AH.health(hp, p8) == {"31": "Healthy", "34": "Healthy", "35": "Healthy"}
        assert all(v == "" for k in (p4, p8) for v in drift(hp, k).values())
        after = hp.allocate(["31"])["cdi_devices"]
        assert after != before and len(after) == 1  # the VF has a fresh CDI index under its new type
        assert refresh(hp) == ([], False, False)
    finally:
        hp.close()


def test_pf_aer_on_every_served_vf_group(kx, tree):
    base = tree[1]
    counts = {}
    for on in (False, True):
        hp = _health_plugin(kx, tree, on=on)
        AH.enable(hp, True)
        try:
            state = _start(hp)
            p4, p8 = _served(state, "NVIDIA_H100-4C"), _served(state, "NVIDIA_H100-8C")
            a0 = AH.reads(hp)
            AH.write(os.path.join(base, PF), fatal=1)
            changed = AH.refresh(hp)[0]
            counts[on] = AH.reads(hp) - a0
            want = "0000:03:00.0 reported 1 fatal uncorrectable PCIe errors (limit 0)"
            if on:
                assert changed == [p4, p8]
                assert AH.reasons(hp, p4) == {"31": want, "32": want, "33": want}
                assert AH.reasons(hp, p8) == {"34": want, "35": want}
                assert set(AH.health(hp, p4).values()) == set(AH.health(hp, p8).values()) == {"Unhealthy"}
            else:
                assert changed == [] and set(AH.health(hp, p4).values()) == {"Healthy"}
            os.remove(os.path.join(base, PF, "aer_dev_fatal"))
            os.remove(os.path.join(base, PF, "aer_dev_nonfatal"))
        finally:
            hp.close()
    assert counts[True] == counts[False] + 2  # the PF's two files, once for its five VF groups


def test_dra_type_taint(kx, tree, pci_text):
    base = tree[1]
    blobs = {}
    for on in (False, True):
        for f in os.listdir(tree[3]):
            os.remove(os.path.join(tree[3], f))
        hp = _health_plugin(kx, tree, on=on)
        taint_lib().kxh_set_dra_taints(hp.h, 1)
        clock = C.c_int64(T0)
        taint_lib().kxh_set_clock(hp.h, C.byref(clock))
        AH.enable(hp, True)
        try:
            _start(hp)
            blobs[on] = (VH.slices(hp, 1)[0], DH.slices(hp, 0)[0])
            if not on:
                continue
            H.set_files(base, VFS[1], b"0\n")
            assert refresh(hp)[1] is True and DH.generation(hp) == 2
            clock.value = T0 + 60
            assert refresh(hp)[1] is False and DH.generation(hp) == 2  # unchanged taints: no bump, same timeAdded
            blob = VH.slices(hp, 1)[0]
            devs = _devices(blob)
            assert devs["vfio32"]["taints"] == [dict(CHANGED_TAINT, timeAdded="2026-01-01T00:00:00Z")]
            assert all("taints" not in d for k, d in devs.items() if k != "vfio32")
            # the passthrough pool keeps its bytes; only the generation it shares with the VF-vGPU pool moved
            assert DH.slices(hp, 0)[0] == blobs[False][1].replace(b'"generation":1,', b'"generation":2,')
            with pytest.raises(RuntimeError, match="device vfio32 no longer carries its published vGPU type: "
                                                   "0000:03:00.2 now carries vGPU type 0"):
                DH.prepare(hp, VDRV, "node-a", ["vfio32"])
            assert DH.prepare(hp, VDRV, "node-a", ["vfio31"]) == [hp.allocate(["31"])["cdi_devices"]]
            # the PF's AER taint reuses the pcie-aer entry, next to the type taint
            AH.write(os.path.join(base, PF), fatal=1)
            clock.value = T0 + 120
            assert AH.refresh(hp)[1] is True and DH.generation(hp) == 3
            devs = _devices(VH.slices(hp, 1)[0])
            aer = dict(key=VDRV + "/pcie-aer", value="fatal", effect="NoSchedule", timeAdded="2026-01-01T00:02:00Z")
            assert devs["vfio32"]["taints"] == [aer, dict(CHANGED_TAINT, timeAdded="2026-01-01T00:00:00Z")]
            assert devs["vfio31"]["taints"] == [aer]
            os.remove(os.path.join(base, PF, "aer_dev_fatal"))
            os.remove(os.path.join(base, PF, "aer_dev_nonfatal"))
            H.set_files(base, VFS[1], b"557\n")
            assert refresh(hp)[1] is True and DH.generation(hp) == 4
        finally:
            hp.close()
    assert blobs[True] == blobs[False]  # nothing drifted yet: the fourth entry adds no byte


def test_off_reads_nothing_and_changes_nothing(kx, tree):
    base = tree[1]
    runs = []
    for on in (False, True):
        for f in os.listdir(tree[3]):
            os.remove(os.path.join(tree[3], f))
        hp = _health_plugin(kx, tree, on=on)
        AH.enable(hp, True)
        try:
            state = _start(hp)
            r0, a0 = H.reads(hp), AH.reads(hp)
            H.set_files(base, VFS[0], b"0\n")
            res = refresh(hp)
            reads = (H.reads(hp) - r0, AH.reads(hp) - a0)
            lw = [hp.list_and_watch(k) for k in range(len(state["plugins"]))]
            runs.append(dict(res=res, reads=reads, lw=lw, slices=VH.slices(hp, 1)[0], gen=DH.generation(hp)))
            H.set_files(base, VFS[0], b"557\n")
        finally:
            hp.close()
    off, on = runs
    assert off["res"] == ([], False, False) and off["reads"] == (0, 0)
    assert on["reads"] == (5, 0)
    assert off["slices"] == on["slices"] and off["gen"] == on["gen"] == 1  # without draTaints no taint is published
    assert off["lw"] != on["lw"]  # only the drifted VF's health differs
