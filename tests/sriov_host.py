"""Fake-sysfs helpers for the host plugin's SR-IOV handling (Plugin::sriovAware): physfn / virtfnN links and sriov_numvfs
files in a fake tree, driver rebinds, the gather with its side records, the setting and the read counter."""
import ctypes as C
import os

import numpy as np

from fake_sysfs import host_lib
from kxpu_b200.binding import SRIOVREC_DTYPE

NV = "10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-xxxx"


def _dir(base, bdf):
    return os.path.realpath(os.path.join(base, bdf))


def link_vfs(base, pf, vfs, numvfs=None):
    """<vf>/physfn -> ../<pf> and <pf>/virtfn<k> -> ../<vf> (relative, as sysfs has them); numvfs: the bytes of
    <pf>/sriov_numvfs (None: no file)."""
    p = _dir(base, pf)
    for k, vf in enumerate(vfs):
        v = _dir(base, vf)
        os.symlink(os.path.relpath(p, v), os.path.join(v, "physfn"))
        os.symlink(os.path.relpath(v, p), os.path.join(p, "virtfn%d" % k))
    if numvfs is not None:
        open(os.path.join(p, "sriov_numvfs"), "wb").write(numvfs)


def rebind(root, base, bdf, driver):
    """Point <bdf>/driver at drivers/<driver> (None: unbind)."""
    link = os.path.join(_dir(base, bdf), "driver")
    if os.path.islink(link):
        os.remove(link)
    if driver is not None:
        drv = os.path.join(root, "drivers", driver)
        os.makedirs(drv, exist_ok=True)
        os.symlink(drv, link)


def gather(base, dtype, on, classes=NV, fast=False, threads=0, cap=1024):
    """(records, side records, sriovReads) of the PCI gather with sriovAware = on."""
    L = host_lib()
    L.kxh_gather_sriov.restype = C.c_int
    L.kxh_gather_sriov.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t,
                                   C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    recs, srs = np.zeros(cap, dtype), np.zeros(cap, SRIOVREC_DTYPE)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_sriov(base.encode(), classes.encode(), int(on), int(fast), threads, recs.ctypes.data, srs.ctypes.data,
                            cap, C.byref(n), C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], srs[:n.value], reads.value


def set_sriov(hp, on):
    hp.L.kxh_set_sriov.argtypes = [C.c_void_p, C.c_int]
    hp.L.kxh_set_sriov(hp.h, int(on))


def reads(hp):
    hp.L.kxh_sriov_reads.restype = C.c_uint64
    hp.L.kxh_sriov_reads.argtypes = [C.c_void_p]
    return hp.L.kxh_sriov_reads(hp.h)
