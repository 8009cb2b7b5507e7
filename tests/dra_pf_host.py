"""Fake-sysfs helpers for Plugin::sriovPfAware (passthrough SR-IOV VFs held to their PF): a tree of two PFs on their
vendor driver with VFs on vfio-pci and a plain function, and the setting."""
import ctypes as C

import fake_sysfs
import sriov_host as SH

CLASSES = "8086,vfio-pci,intel.com,intel.com/gpu,cdi-vfio-intel"
DRIVER = "gpu.intel.com"
INTEL = dict(vendor=b"0x8086\n", device=b"0x56c0\n")
PF_A, PF_B, PLAIN = "0000:4d:00.0", "0000:9a:00.0", "0000:c1:00.0"
VFS_A = ["0000:4d:00.1", "0000:4d:00.2", "0000:4d:00.3"]
VFS_B = ["0000:9a:00.1", "0000:9a:00.2"]
DEVS = [dict(bdf=PF_A, group=40, driver="i915", **INTEL),   # PF A on its vendor driver: no class candidate
        dict(bdf=VFS_A[0], group=41, driver="vfio-pci", **INTEL),
        dict(bdf=VFS_A[1], group=42, driver="vfio-pci", **INTEL),
        dict(bdf=VFS_A[2], group=43, driver="vfio-pci", **INTEL),
        dict(bdf=PF_B, group=50, driver="i915", **INTEL),   # PF B
        dict(bdf=VFS_B[0], group=51, driver="vfio-pci", **INTEL),
        dict(bdf=VFS_B[1], group=52, driver="vfio-pci", **INTEL),
        dict(bdf=PLAIN, group=60, driver="vfio-pci", **INTEL)]  # a function with no VFs
GROUPS_A, GROUPS_B = ["41", "42", "43"], ["51", "52"]


def make_tree(root):
    """the tree of DEVS with PF A's three VFs and PF B's two linked to their PFs; returns the PCI base"""
    base = fake_sysfs.make_tree(root, DEVS)
    SH.link_vfs(base, PF_A, VFS_A, b"3\n")
    SH.link_vfs(base, PF_B, VFS_B, b"2\n")
    return base


def enable(hp, on=True):
    hp.L.kxh_set_sriov_pf.argtypes = [C.c_void_p, C.c_int]
    hp.L.kxh_set_sriov_pf(hp.h, int(on))
