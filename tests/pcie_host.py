"""Fake-sysfs helpers for the host plugin's PCIe topology (Plugin::pcieTopologyAware): a tree whose entries link into
devices/pci.../.../<bdf> like real sysfs, the gathers with a counting readPciPath seam, the setting and the nodes the
Devices carry."""
import ctypes as C
import os

import numpy as np

from fake_sysfs import host_lib
from kxpu_b200.binding import PCIPATH_DTYPE


def make_nested_tree(root, devices, relative=False):
    """fake_sysfs.make_tree's layout with each entry's directory at devices/<path> instead of devices/<bdf>.
    devices: dicts(bdf, path, vendor, device, driver, group) -- path e.g. "pci0000:00/0000:00:01.0/0000:03:00.0", None
    for a plain directory entry; relative: links as "../../../devices/<path>" (real sysfs) instead of absolute ones."""
    base = os.path.join(root, "bus", "pci", "devices")
    os.makedirs(base)
    os.makedirs(os.path.join(root, "drivers"), exist_ok=True)
    os.makedirs(os.path.join(root, "iommu_groups"), exist_ok=True)
    for d in devices:
        target = os.path.join(base, d["bdf"]) if d.get("path") is None else os.path.join(root, "devices", d["path"])
        os.makedirs(target, exist_ok=True)
        for f in ("vendor", "device"):
            if d.get(f) is not None:
                open(os.path.join(target, f), "wb").write(d[f])
        if d.get("driver") is not None:
            drv = os.path.join(root, "drivers", d["driver"])
            os.makedirs(drv, exist_ok=True)
            os.symlink(drv, os.path.join(target, "driver"))
        if d.get("group") is not None:
            grp = os.path.join(root, "iommu_groups", str(d["group"]))
            os.makedirs(grp, exist_ok=True)
            os.symlink(grp, os.path.join(target, "iommu_group"))
        if d.get("path") is not None:
            link = os.path.join(base, d["bdf"])
            os.symlink(os.path.join("../../../devices", d["path"]) if relative else target, link)
    return base


def move_link(root, bdf, new_path):
    """Point <base>/<bdf> at devices/<new_path> (the device's directory moves there)."""
    base = os.path.join(root, "bus", "pci", "devices")
    link = os.path.join(base, bdf)
    target = os.readlink(link)
    new = os.path.join(root, "devices", new_path)
    os.makedirs(os.path.dirname(new), exist_ok=True)
    os.rename(os.path.normpath(os.path.join(base, target)), new)
    os.remove(link)
    os.symlink(new if os.path.isabs(target) else os.path.join("../../../devices", new_path), link)


def _lib():
    L = host_lib()
    L.kxh_gather_pcie.restype = C.c_int
    L.kxh_gather_pcie.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_uint, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p,
                                  C.c_size_t]
    L.kxh_set_pcie_topology.argtypes = [C.c_void_p, C.c_int]
    L.kxh_devs_pcie.restype = C.c_int
    L.kxh_devs_pcie.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    return L


def gather(base, dtype, pcie, fast=False, threads=0, count=False, cap=4096):
    """(records, paths, readPciPath calls) of the PCI gather with pcieTopologyAware = pcie; count installs the
    counting seam (which sends the fast gather down the walk)."""
    L = _lib()
    recs = np.zeros(cap, dtype=dtype)
    paths = np.zeros(cap, dtype=PCIPATH_DTYPE)
    n, np_, reads = C.c_size_t(0), C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_pcie(base.encode(), int(pcie), int(fast), threads, int(count), recs.ctypes.data, paths.ctypes.data,
                           cap, C.byref(n), C.byref(np_), C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], paths[:np_.value], reads.value


def set_pcie(hp, on):
    _lib().kxh_set_pcie_topology(hp.h, int(on))


def devs_pcie(hp, plugin_index):
    buf = C.create_string_buffer(1 << 16)
    assert _lib().kxh_devs_pcie(hp.h, plugin_index, buf, len(buf)) >= 0
    return {k: int(v) for k, v in (x.split("=") for x in buf.value.decode().split(",") if x)}
