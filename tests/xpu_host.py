"""Fake-sysfs helpers for the accelerator class list of the host plugin (Plugin::xpuClasses): the raw gather and
the InitiateDevicePlugin / Allocate flow under a list of classes.  Builds on fake_sysfs."""
import ctypes as C

import numpy as np

import fake_sysfs
from fake_sysfs import host_lib


def class_spec(classes):
    """[(vendor, driver, namespace, kind, file stem)] -> the "v,d,ns,kind,stem;..." string of kxh_set_classes."""
    return ";".join(",".join(c) for c in classes).encode()


def gather_classes(base, dtype, classes, fast=False, threads=0, cap=4096):
    """The raw gather under a class list (Plugin::xpuClasses)."""
    L = host_lib()
    L.kxh_gather_classes.restype = C.c_int
    L.kxh_gather_classes.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_uint, C.c_void_p, C.c_size_t,
                                     C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
    recs = np.zeros(cap, dtype=dtype)
    n = C.c_size_t(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_classes(base.encode(), class_spec(classes), 1 if fast else 0, threads, recs.ctypes.data, cap,
                              C.byref(n), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value]


class HostPlugin(fake_sysfs.HostPlugin):
    """fake_sysfs.HostPlugin serving the classes [(vendor, driver, namespace, kind, file stem)]."""

    def __init__(self, kx, base, pciids, cdi_dir, classes):
        super().__init__(kx, base, pciids, cdi_dir)
        self.L.kxh_set_classes.restype = C.c_int
        self.L.kxh_set_classes.argtypes = [C.c_void_p, C.c_char_p]
        assert self.L.kxh_set_classes(self.h, class_spec(classes)) == 0
