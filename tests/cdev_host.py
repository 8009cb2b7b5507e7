"""Fake-sysfs helpers for passthrough classes served through VFIO cdevs (XpuClass::vfioCdev): vfio-dev/ entries in the
fake tree, the gather with its cdev side array, the vGPU-class check and a plugin's cdev nodes."""
import ctypes as C
import json
import os

import numpy as np

from fake_sysfs import host_lib

NV = ("10de", "vfio-pci", "nvidia.com", "nvidia.com/gpu", "cdi-vfio-xxxx")
NV_CDEV = NV + ("cdev",)


def spec(classes):
    return ";".join(",".join(c) for c in classes).encode()


def set_vfio_dev(base, bdf, entries):
    """<base>/<bdf>/vfio-dev/ holding these entry names (directories, as in sysfs); None removes vfio-dev/."""
    d = os.path.join(base, bdf, "vfio-dev")
    if os.path.isdir(d):
        for e in os.listdir(d):
            os.rmdir(os.path.join(d, e))
        os.rmdir(d)
    if entries is None:
        return
    os.makedirs(d)
    for e in entries:
        os.makedirs(os.path.join(d, e))


def gather(base, dtype, classes, fast=False, threads=0, cap=1024):
    """(records, cdevs, vfio-dev reads) of the gather under a class list."""
    L = host_lib()
    L.kxh_gather_cdev.restype = C.c_int
    L.kxh_gather_cdev.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    recs = np.zeros(cap, dtype)
    cdevs = np.zeros(cap, np.int64)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_cdev(base.encode(), spec(classes), int(fast), threads, recs.ctypes.data, cdevs.ctypes.data, cap,
                           C.byref(n), C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], cdevs[:n.value], reads.value


def check_vgpu_classes(classes, vgpu_classes):
    L = host_lib()
    L.kxh_check_vgpu_classes.restype = C.c_int
    L.kxh_check_vgpu_classes.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]
    err = C.create_string_buffer(512)
    rc = L.kxh_check_vgpu_classes(spec(classes), spec(vgpu_classes), err, 512)
    return None if rc == 0 else err.value.decode()


def plugin_nodes(hp, idx):
    hp.L.kxh_plugin_nodes.restype = C.c_int
    hp.L.kxh_plugin_nodes.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(1 << 16)
    assert hp.L.kxh_plugin_nodes(hp.h, idx, buf, len(buf)) >= 0
    return json.loads(buf.value.decode())


def cdev_reads(hp):
    hp.L.kxh_cdev_reads.restype = C.c_uint64
    hp.L.kxh_cdev_reads.argtypes = [C.c_void_p]
    return hp.L.kxh_cdev_reads(hp.h)
