"""Fake-sysfs helpers for the host plugin's reset check (Plugin::resetCheck): reset_method / reset files in a fake tree,
the gather with its reset reads, the setting and the read counter."""
import ctypes as C
import os

import numpy as np

from fake_sysfs import host_lib
from kxpu_b200.binding import PCIPATH_DTYPE, RESETREC_DTYPE

NV = "10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-xxxx"


def set_method(base, bdf, text=None, legacy=False):
    """<bdf>/reset_method holding text (None: no file), and with legacy an empty <bdf>/reset"""
    d = os.path.realpath(os.path.join(base, bdf))
    for f in ("reset_method", "reset"):
        if os.path.exists(os.path.join(d, f)):
            os.remove(os.path.join(d, f))
    if text is not None:
        open(os.path.join(d, "reset_method"), "wb").write(text)
    if legacy:
        open(os.path.join(d, "reset"), "wb").close()


def gather(base, dtype, on, classes=NV, fast=False, threads=0, cap=1024):
    """(records, paths, side records, resetReads) of the PCI gather and the reset reads with resetCheck = on."""
    L = host_lib()
    L.kxh_gather_reset.restype = C.c_int
    L.kxh_gather_reset.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    recs, paths, rrs = np.zeros(cap, dtype), np.zeros(cap, PCIPATH_DTYPE), np.zeros(cap, RESETREC_DTYPE)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_reset(base.encode(), classes.encode(), int(on), int(fast), threads, recs.ctypes.data,
                            paths.ctypes.data, rrs.ctypes.data, cap, C.byref(n), C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], paths[:n.value], rrs[:n.value], reads.value


def set_reset(hp, on, methods=None):
    """resetCheck = on; methods: a list of names for resetMethods (None keeps the default)"""
    hp.L.kxh_set_reset.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    hp.L.kxh_set_reset(hp.h, int(on), None if methods is None else ",".join(methods).encode())


def reads(hp):
    hp.L.kxh_reset_reads.restype = C.c_uint64
    hp.L.kxh_reset_reads.argtypes = [C.c_void_p]
    return hp.L.kxh_reset_reads(hp.h)
