"""Fake-sysfs helpers for the host plugin's IOMMU group viability (Plugin::groupViability): the gathers with a counting
readLink seam, the setting, the per-device verdicts and a rediscovery."""
import ctypes as C
import json

import numpy as np

from fake_sysfs import host_lib

NV_CLASS = "10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-xxxx"


def _lib():
    L = host_lib()
    L.kxh_gather_viab.restype = C.c_int
    L.kxh_gather_viab.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_uint, C.c_int, C.c_void_p,
                                  C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    L.kxh_set_viability.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    L.kxh_rediscover.restype = C.c_int
    L.kxh_rediscover.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_size_t]
    L.kxh_set_device_path.restype = C.c_int
    L.kxh_set_device_path.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    return L


def gather(base, dtype, on, drivers=None, classes=NV_CLASS, fast=False, threads=0, count=False, cap=4096):
    """(records, driver / iommu_group reads of entries whose vendor no class has) of the PCI gather with
    groupViability = on; drivers replaces viabilityDrivers (a list); count installs the counting readLink seam."""
    L = _lib()
    recs = np.zeros(cap, dtype=dtype)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_viab(base.encode(), classes.encode(), int(on), None if drivers is None else ",".join(drivers).encode(),
                           int(fast), threads, int(count), recs.ctypes.data, cap, C.byref(n), C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], reads.value


def set_viability(hp, on, drivers=None):
    _lib().kxh_set_viability(hp.h, int(on), None if drivers is None else ",".join(drivers).encode())


def devs(hp, plugin_index):
    """{id: (Health, blocker or None)} of one plugin's devices."""
    buf = C.create_string_buffer(1 << 16)
    assert hp.L.kxh_devs(hp.h, plugin_index, buf, len(buf)) >= 0
    out = {}
    for item in buf.value.decode().split(","):
        if not item:
            continue
        k, v = item.split("=", 1)
        health, _, blocker = v.partition("/")
        out[k] = (health, blocker or None)
    return out


def rediscover(hp):
    L = _lib()
    buf = C.create_string_buffer(1 << 20)
    rc = L.kxh_rediscover(hp.h, b"YAML", buf, len(buf))
    if rc < 0:
        raise RuntimeError(buf.value.decode())
    return json.loads(buf.value.decode())
