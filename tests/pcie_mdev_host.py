"""Fake-sysfs helpers for the host plugin's vGPU PCIe topology (Plugin::vgpuPcieTopologyAware): an mdev tree whose
parents sit in a PCIe hierarchy (devices/pci0000:00/.../<parent>/<uuid>, links relative as on real sysfs), moving an
mdev to another parent, and the setting."""
import ctypes as C
import os
import shutil

import fake_mdev
from fake_sysfs import host_lib


def make_tree(root, gpus, mdevs):
    """gpus: {parent address: its path from devices/, e.g. "pci0000:00/0000:00:01.0/0000:03:00.0"}; mdevs: fake_mdev
    dicts whose parent is an address of gpus.  Every parent has vendor 10de.  Returns the mdev base path."""
    nested = [dict(m, parent=gpus[m["parent"]]) for m in mdevs]
    base = fake_mdev.make_tree(root, nested, parents={p: b"0x10de\n" for p in gpus.values()})
    for m in nested:
        link = os.path.join(base, m["uuid"])
        os.remove(link)
        os.symlink(os.path.join("../../../devices", m["parent"], m["uuid"]), link)
    return base


def move(root, uuid, old_parent_path, new_parent_path):
    """The mdev uuid now lives below another parent (its directory and link move there)."""
    src = os.path.join(root, "devices", old_parent_path, uuid)
    dst = os.path.join(root, "devices", new_parent_path, uuid)
    shutil.move(src, dst)
    tdir = os.path.join(root, "devices", new_parent_path, "mdev_supported_types")
    if not os.path.isdir(tdir):
        shutil.copytree(os.path.join(root, "devices", old_parent_path, "mdev_supported_types"), tdir)
    mt = os.path.join(dst, "mdev_type")
    t = os.path.basename(os.readlink(mt))
    os.remove(mt)
    os.symlink(os.path.join(tdir, t), mt)
    link = os.path.join(root, "bus", "mdev", "devices", uuid)
    os.remove(link)
    os.symlink(os.path.join("../../../devices", new_parent_path, uuid), link)


def set_vgpu_pcie(hp, on):
    L = host_lib()
    L.kxh_set_vgpu_pcie_topology.argtypes = [C.c_void_p, C.c_int]
    L.kxh_set_vgpu_pcie_topology(hp.h, int(on))
