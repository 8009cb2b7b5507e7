"""Fake-sysfs helpers for the host plugin's NUMA topology (Plugin::topologyAware): numa_node files on fake_sysfs /
fake_mdev trees, the gathers with a counting readNumaNode seam, the options and GetPreferredAllocation."""
import ctypes as C
import json
import os

import numpy as np

from fake_sysfs import host_lib


def add_numa(root, numa):
    """numa: {PCI address: bytes}.  Writes <root>/devices/<address>/numa_node, the directory a fake_sysfs entry (or a
    fake_mdev parent) links to; an address that is not in the dict gets no file."""
    for addr, raw in numa.items():
        open(os.path.join(root, "devices", addr, "numa_node"), "wb").write(raw)


def _lib():
    L = host_lib()
    L.kxh_gather_topo.restype = C.c_int
    L.kxh_gather_topo.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_uint, C.c_int, C.c_void_p, C.c_size_t,
                                  C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    L.kxh_gather_mdev_topo.restype = C.c_int
    L.kxh_gather_mdev_topo.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                       C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    L.kxh_set_topology.argtypes = [C.c_void_p, C.c_int]
    L.kxh_options.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.kxh_preferred_allocation.restype = C.c_int
    L.kxh_preferred_allocation.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_size_t]
    L.kxh_devs_numa.restype = C.c_int
    L.kxh_devs_numa.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    return L


def gather(base, dtype, topo, fast=False, threads=0, count=True, cap=4096):
    """(records, numa_node reads) of the PCI gather with topologyAware = topo; count installs the counting seam."""
    L = _lib()
    recs = np.zeros(cap, dtype=dtype)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_topo(base.encode(), int(topo), int(fast), threads, int(count), recs.ctypes.data, cap, C.byref(n),
                           C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], reads.value


def gather_mdev(mdev_base, classes, dtype, topo, count=True, cap=4096):
    L = _lib()
    recs = np.zeros(cap, dtype=dtype)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    spec = ";".join(",".join(c) for c in classes).encode()
    rc = L.kxh_gather_mdev_topo(mdev_base.encode(), spec, int(topo), int(count), recs.ctypes.data, cap, C.byref(n),
                                C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], reads.value


def set_topology(hp, on):
    _lib().kxh_set_topology(hp.h, int(on))


def options(hp):
    a, b = C.c_int(-1), C.c_int(-1)
    _lib().kxh_options(hp.h, C.byref(a), C.byref(b))
    return dict(PreStartRequired=bool(a.value), GetPreferredAllocationAvailable=bool(b.value))


def preferred_allocation(hp, plugin_index, requests):
    """requests: [(available ids, must-include ids, size)] -> [[ids]] (raises RuntimeError with the plugin's error)."""
    spec = ";".join("%s|%s|%d" % (",".join(a), ",".join(m), s) for a, m, s in requests).encode()
    buf = C.create_string_buffer(1 << 20)
    rc = _lib().kxh_preferred_allocation(hp.h, plugin_index, spec, buf, len(buf))
    if rc < 0:
        raise RuntimeError(buf.value.decode())
    return json.loads(buf.value.decode())


def devs_numa(hp, plugin_index):
    buf = C.create_string_buffer(1 << 16)
    assert _lib().kxh_devs_numa(hp.h, plugin_index, buf, len(buf)) >= 0
    return {k: int(v) for k, v in (x.split("=") for x in buf.value.decode().split(",") if x)}
