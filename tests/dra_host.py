"""Fake-sysfs helpers for the host plugin's DRA ResourceSlices (XpuClass::draDriver, Plugin::ResourceSlices): the
settings, the configuration checks, the slices and generation, PrepareDraDevices, the counting read seams, and the
records a test builds from its own tree description."""
import ctypes as C
import json
import os

import numpy as np

from fake_sysfs import host_lib
from oracle.dra_oracle import DRADEV_DTYPE


def _lib():
    L = host_lib()
    L.kxh_set_classes.restype = C.c_int
    L.kxh_set_classes.argtypes = [C.c_void_p, C.c_char_p]
    L.kxh_set_dra.restype = C.c_int
    L.kxh_set_dra.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
    L.kxh_initiate.restype = C.c_int
    L.kxh_initiate.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    L.kxh_resource_slices.restype = C.c_int
    L.kxh_resource_slices.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p,
                                      C.c_size_t, C.POINTER(C.c_size_t)]
    L.kxh_dra_generation.restype = C.c_uint64
    L.kxh_dra_generation.argtypes = [C.c_void_p]
    L.kxh_prepare_dra.restype = C.c_int
    L.kxh_prepare_dra.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]
    L.kxh_count_reads.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.kxh_set_topology.argtypes = [C.c_void_p, C.c_int]
    L.kxh_set_pcie_topology.argtypes = [C.c_void_p, C.c_int]
    L.kxh_set_viability.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
    L.kxh_rediscover.restype = C.c_int
    L.kxh_rediscover.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_size_t]
    return L


def configure(hp, classes=None, dra=None, node="node-a", topo=False, pcie=False, viability=False):
    """classes: "vendor,driver,namespace,kind,stem;..." (None keeps the default); dra: the draDriver of every class
    (a list, "" = none; None sets nothing)."""
    L = _lib()
    if classes is not None:
        assert L.kxh_set_classes(hp.h, classes.encode()) == 0
    if dra is not None:
        assert L.kxh_set_dra(hp.h, ",".join(dra).encode(), node.encode()) == 0
    L.kxh_set_topology(hp.h, int(topo))
    L.kxh_set_pcie_topology(hp.h, int(pcie))
    if viability:
        L.kxh_set_viability(hp.h, 1, None)


class Counter:
    """numa_node and entry-link reads of a plugin's gathers"""

    def __init__(self, hp):
        self.numa, self.paths = C.c_uint64(0), C.c_uint64(0)
        _lib().kxh_count_reads(hp.h, C.byref(self.numa), C.byref(self.paths))

    def reads(self):
        return self.numa.value, self.paths.value


def initiate(hp):
    """InitiateDevicePlugin: None, or its error message"""
    err = C.create_string_buffer(1024)
    return None if _lib().kxh_initiate(hp.h, err, len(err)) == 0 else err.value.decode()


def slices(hp, cls):
    """(bytes, slice_off) of ResourceSlices(cls); RuntimeError with the message on failure"""
    L = _lib()
    ln, ns = C.c_size_t(0), C.c_size_t(0)
    out, offs = np.zeros(1 << 16, np.uint8), np.zeros(1024, np.uint64)
    rc = L.kxh_resource_slices(hp.h, cls, out.ctypes.data, out.size, C.byref(ln), offs.ctypes.data, offs.size, C.byref(ns))
    if rc == -1:
        raise RuntimeError(out.tobytes().split(b"\0", 1)[0].decode())
    assert rc == 0, rc
    return out[:ln.value].tobytes(), offs[:ns.value + 1]


def generation(hp):
    return _lib().kxh_dra_generation(hp.h)


def prepare(hp, driver, pool, names):
    buf = C.create_string_buffer(1 << 16)
    if _lib().kxh_prepare_dra(hp.h, driver.encode(), pool.encode(), ",".join(names).encode(), buf, len(buf)) < 0:
        raise RuntimeError(buf.value.decode())
    return json.loads(buf.value.decode())


def rediscover(hp):
    buf = C.create_string_buffer(1 << 20)
    if _lib().kxh_rediscover(hp.h, b"YAML", buf, len(buf)) < 0:
        raise RuntimeError(buf.value.decode())
    return json.loads(buf.value.decode())


def add_numa(root, devices):
    """numa_node files in the entries' directories (devices/<path>) of a pcie_host.make_nested_tree tree"""
    for d in devices:
        if d.get("numa") is not None:
            open(os.path.join(root, "devices", d["path"], "numa_node"), "wb").write(d["numa"])


def expected_records(state, devices, cls):
    """the kxpu_dradev records ResourceSlices(cls) publishes, built from the test's own tree description and the
    plugin's state (kxh_init's dump): one per iommuMap group of the class in walk order, from its first member, the
    product being the name of the plugin that serves the group; blocked: group ids left out"""
    by_bdf = {d["bdf"]: d for d in devices}
    product = {dev[0]: p["name"] for p in state["plugins"] if not p["vgpu"] for dev in p["devs"]}
    recs = []
    for (gid, members), c in zip(state["iommuMap"], state["iommuClass"]):
        if c != cls:
            continue
        d = by_bdf[members[0][0]]
        r = np.zeros(1, DRADEV_DTYPE)
        r["bdf"] = d["bdf"].encode()
        r["vendor"], r["device"] = d["vendor"][2:].strip(), d["device"][2:].strip()
        r["pcie_root"] = d["path"].split("/")[0].encode()
        numa = d.get("numa")
        r["numa_mask"] = 1 << int(numa) if numa is not None and numa.strip().isdigit() and int(numa) < 64 else 0
        r["iommu_group"] = int(gid)
        name = product[gid].encode()[:64]
        r["product"][0, :len(name)] = np.frombuffer(name, np.uint8)
        r["product_len"] = len(name)
        recs.append(r)
    return np.concatenate(recs) if recs else np.zeros(0, DRADEV_DTYPE)
