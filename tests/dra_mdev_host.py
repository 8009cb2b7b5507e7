"""Fake-sysfs helpers for the host plugin's vGPU DRA ResourceSlices (a draDriver on a vGPU class,
Plugin::VgpuResourceSlices): a tree whose parent GPUs sit under devices/pci<domain>:<bus>/... with `device` and
`numa_node` files and whose mdev entries link below them like real sysfs, the settings, the slices and generation,
and the records a test builds from its own tree description."""
import ctypes as C
import os

import numpy as np

import dra_host as DH
import pcie_host
from fake_sysfs import host_lib
from oracle.dra_mdev_oracle import DRAMDEV_DTYPE


def make_tree(root, parents, mdevs):
    """parents: dicts(bdf, path, vendor, device=None, numa=None, driver, group) -- PCI entries at devices/<path>, linked
    from bus/pci/devices (pcie_host.make_nested_tree, relative links), each with a numa_node file when numa is given;
    mdevs: dicts(uuid, parent (a bdf), group, type_id='nvidia-1120', name=b'NVIDIA H100XM-1-10C\\n', driver='vfio_mdev')
    -- directories devices/<parent path>/<uuid> linked from bus/mdev/devices/<uuid> as ../../../devices/... .  Returns
    (PCI base, mdev base)."""
    base = pcie_host.make_nested_tree(root, parents, relative=True)
    DH.add_numa(root, parents)
    mbase = os.path.join(root, "bus", "mdev", "devices")
    os.makedirs(mbase)
    for m in mdevs:
        add_mdev(root, parents, m)
    return base, mbase


def add_mdev(root, parents, m):
    """one mdev of make_tree's layout (a vGPU created after the tree)"""
    path = {p["bdf"]: p["path"] for p in parents}[m["parent"]]
    rel = os.path.join(path, m["uuid"])
    target = os.path.join(root, "devices", rel)
    os.makedirs(target)
    tdir = os.path.join(root, "devices", path, "mdev_supported_types", m.get("type_id", "nvidia-1120"))
    os.makedirs(tdir, exist_ok=True)
    open(os.path.join(tdir, "name"), "wb").write(m.get("name", b"NVIDIA H100XM-1-10C\n"))
    os.symlink(tdir, os.path.join(target, "mdev_type"))
    drv = os.path.join(root, "drivers", m.get("driver", "vfio_mdev"))
    os.makedirs(drv, exist_ok=True)
    os.symlink(drv, os.path.join(target, "driver"))
    grp = os.path.join(root, "iommu_groups", str(m["group"]))
    os.makedirs(grp, exist_ok=True)
    os.symlink(grp, os.path.join(target, "iommu_group"))
    os.symlink(os.path.join("../../../devices", rel), os.path.join(root, "bus", "mdev", "devices", m["uuid"]))


def _lib():
    L = host_lib()
    L.kxh_set_vgpu_dra.restype = C.c_int
    L.kxh_set_vgpu_dra.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.kxh_vgpu_resource_slices.restype = C.c_int
    L.kxh_vgpu_resource_slices.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p,
                                           C.c_size_t, C.POINTER(C.c_size_t)]
    L.kxh_dra_vgpu_generation.restype = C.c_uint64
    L.kxh_dra_vgpu_generation.argtypes = [C.c_void_p]
    L.kxh_count_id_reads.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_uint64)]
    return L


def set_vgpu_dra(hp, drivers, node="node-a"):
    """the draDriver of every vGPU class (a list, "" = none) and the node name"""
    assert _lib().kxh_set_vgpu_dra(hp.h, ",".join(drivers).encode(), node.encode()) == 0


def slices(hp, cls):
    """(bytes, slice_off) of VgpuResourceSlices(cls); RuntimeError with the message on failure"""
    L = _lib()
    ln, ns = C.c_size_t(0), C.c_size_t(0)
    out, offs = np.zeros(1 << 16, np.uint8), np.zeros(1024, np.uint64)
    rc = L.kxh_vgpu_resource_slices(hp.h, cls, out.ctypes.data, out.size, C.byref(ln), offs.ctypes.data, offs.size, C.byref(ns))
    if rc == -1:
        raise RuntimeError(out.tobytes().split(b"\0", 1)[0].decode())
    assert rc == 0, rc
    return out[:ln.value].tobytes(), offs[:ns.value + 1]


def generation(hp):
    return _lib().kxh_dra_vgpu_generation(hp.h)


class DeviceReads:
    """readIDFromFile reads of "../device" (the parents' device ids of the mdev walk)"""

    def __init__(self, hp):
        self.n = C.c_uint64(0)
        _lib().kxh_count_id_reads(hp.h, b"../device", C.byref(self.n))

    def reads(self):
        return self.n.value


def expected_records(state, parents, cls, model_name):
    """the kxpu_dramdev records VgpuResourceSlices(cls) publishes, built from the test's own tree description and the
    plugin's state (kxh_init's dump): one per mdevMap group of the class in walk order, from its first mdev.
    model_name(vendor, device) -> the sanitised pci.ids name or None."""
    by_bdf = {p["bdf"]: p for p in parents}
    key_of = {g: key for key, groups in state["typeMap"] for g in groups}
    recs = []
    for (gid, members), c in zip(state["mdevMap"], state["mdevClass"]):
        if c != cls:
            continue
        uuid, parent = members[0][0], members[0][1]
        p = by_bdf[parent]
        r = np.zeros(1, DRAMDEV_DTYPE)
        r["mdev_type"], r["uuid"], r["iommu_group"], r["parent"] = key_of[gid].encode(), uuid.encode(), int(gid), parent.encode()
        first = p["path"].split("/")[0]
        r["pcie_root"] = first.encode() if first.startswith("pci") else b""
        vendor = p["vendor"][2:].strip()
        device = p["device"][2:].strip() if p.get("device") is not None else b""
        r["vendor"], r["device"] = vendor, device
        numa = p.get("numa")
        r["numa_mask"] = 1 << int(numa) if numa is not None and numa.strip().isdigit() and int(numa) < 64 else 0
        if device:
            name = (model_name(vendor, device) or device)[:64]
            r["product"][0, :len(name)] = np.frombuffer(name, np.uint8)
            r["product_len"] = len(name)
        recs.append(r)
    return np.concatenate(recs) if recs else np.zeros(0, DRAMDEV_DTYPE)
