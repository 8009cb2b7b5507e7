"""Fake-sysfs helpers for Plugin::vgpuSriovAware (mdev vGPUs on SR-IOV VFs): dra_mdev_host's tree with `physfn` links
from VFs to their PF, the setting, and the read counter."""
import ctypes as C
import os

import dra_mdev_host as MH
from fake_sysfs import host_lib


def make_tree(root, parents, mdevs, vfs):
    """MH.make_tree, then for every (vf, pf) of vfs a link <vf>/physfn -> ../<pf>, as the kernel makes it.  Returns
    (PCI base, mdev base)."""
    base, mbase = MH.make_tree(root, parents, mdevs)
    for vf, pf in vfs:
        os.symlink(os.path.join("..", pf), os.path.join(os.path.realpath(os.path.join(base, vf)), "physfn"))
    return base, mbase


def _lib():
    L = host_lib()
    L.kxh_set_vgpu_sriov.argtypes = [C.c_void_p, C.c_int]
    L.kxh_mdev_physfn_reads.restype = C.c_uint64
    L.kxh_mdev_physfn_reads.argtypes = [C.c_void_p]
    return L


def enable(hp, on=True):
    _lib().kxh_set_vgpu_sriov(hp.h, int(on))


def reads(hp):
    return _lib().kxh_mdev_physfn_reads(hp.h)
