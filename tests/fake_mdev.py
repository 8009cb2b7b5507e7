"""Fake /sys/bus/mdev/devices tree next to a fake_sysfs PCI tree: every <uuid> entry is a SYMLINK into a directory
under its parent PCI device's directory, holding `mdev_type` (a link to the parent's mdev_supported_types/<type-id>,
which has a `name` file) and the links `driver` and `iommu_group`, like real sysfs."""
import ctypes as C
import os

import numpy as np

from fake_sysfs import host_lib
from oracle.mdev_oracle import MDEVREC_DTYPE


def make_tree(root, mdevs, parents=None):
    """mdevs: dicts(uuid, parent, type_id='nvidia-222', name=b'GRID T4-1Q\\n'|None, driver='vfio_mdev'|None,
    group=300|None, kind='link'|'dir'|'file', mdev_type=True).  parents: {address: vendor bytes} for parent devices
    that the PCI tree does not hold.  Returns the mdev base path."""
    base = os.path.join(root, "bus", "mdev", "devices")
    os.makedirs(base)
    for a, vendor in (parents or {}).items():
        os.makedirs(os.path.join(root, "devices", a), exist_ok=True)
        open(os.path.join(root, "devices", a, "vendor"), "wb").write(vendor)
    for m in mdevs:
        kind = m.get("kind", "link")
        if kind == "file":
            open(os.path.join(base, m["uuid"]), "w").write("x")
            continue
        if kind == "dir":
            os.makedirs(os.path.join(base, m["uuid"]))
            continue
        pdir = os.path.join(root, "devices", m["parent"])
        target = os.path.join(pdir, m["uuid"])
        os.makedirs(target)
        tdir = os.path.join(pdir, "mdev_supported_types", m.get("type_id", "nvidia-222"))
        os.makedirs(tdir, exist_ok=True)
        if m.get("name", b"GRID T4-1Q\n") is not None:
            open(os.path.join(tdir, "name"), "wb").write(m.get("name", b"GRID T4-1Q\n"))
        if m.get("mdev_type", True):
            os.symlink(tdir, os.path.join(target, "mdev_type"))
        if m.get("driver", "vfio_mdev") is not None:
            drv = os.path.join(root, "drivers", m.get("driver", "vfio_mdev"))
            os.makedirs(drv, exist_ok=True)
            os.symlink(drv, os.path.join(target, "driver"))
        if m.get("group") is not None:
            grp = os.path.join(root, "iommu_groups", str(m["group"]))
            os.makedirs(grp, exist_ok=True)
            os.symlink(grp, os.path.join(target, "iommu_group"))
        os.symlink(target, os.path.join(base, m["uuid"]))
    return base


def expected_record(m, vendor):
    """The kxpu_mdevrec the gather must produce for mdev dict m whose parent's vendor file holds `vendor`."""
    r = np.zeros(1, MDEVREC_DTYPE)[0]
    u = m["uuid"].encode()
    if len(u) == 36:
        r["uuid"] = u
    kind = m.get("kind", "link")
    if kind == "dir":
        r["flags"] = 16
        return r
    if kind == "file" or len(u) != 36:
        return r
    r["parent"] = m["parent"].encode()
    r["parent_vendor_txt"][:len(vendor)] = np.frombuffer(vendor, np.uint8)
    r["vendor_len"] = len(vendor)
    if m.get("driver", "vfio_mdev") is None:
        r["flags"] = 2
        return r
    r["driver"] = m.get("driver", "vfio_mdev").encode()
    if m.get("group") is None:
        r["flags"] = 4
        return r
    r["iommu_group"] = m["group"]
    name = m.get("name", b"GRID T4-1Q\n")
    if name is None or not m.get("mdev_type", True) or len(name) > 40:
        r["flags"] = 32
        return r
    r["type_name"][:len(name)] = np.frombuffer(name, np.uint8)
    r["name_len"] = len(name)
    return r


def gather(mdev_base, classes, cap=4096):
    """The raw mdev gather (Plugin::gatherMdevRecords) under [(vendor, driver, namespace, kind, stem)]."""
    L = host_lib()
    L.kxh_gather_mdev.restype = C.c_int
    L.kxh_gather_mdev.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
    recs = np.zeros(cap, dtype=MDEVREC_DTYPE)
    n = C.c_size_t(0)
    err = C.create_string_buffer(512)
    spec = ";".join(",".join(c) for c in classes).encode()
    rc = L.kxh_gather_mdev(mdev_base.encode(), spec, recs.ctypes.data, cap, C.byref(n), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value]


def set_vgpu(hp, mdev_base, classes):
    """Point a fake_sysfs.HostPlugin at an mdev tree and give it vGPU classes."""
    hp.L.kxh_set_vgpu_classes.restype = C.c_int
    hp.L.kxh_set_vgpu_classes.argtypes = [C.c_void_p, C.c_char_p]
    hp.L.kxh_set_mdev_base.argtypes = [C.c_void_p, C.c_char_p]
    hp.L.kxh_set_mdev_base(hp.h, mdev_base.encode())
    assert hp.L.kxh_set_vgpu_classes(hp.h, ";".join(",".join(c) for c in classes).encode()) == 0
