"""Fake-sysfs helpers for the host plugin's vGPUs on SR-IOV VFs (XpuClass::vfVgpu): nvidia/current_vgpu_type and
nvidia/creatable_vgpu_types in a fake tree, the gather with its side records, the setting, the read counter and the
learned type names."""
import ctypes as C
import json
import os

import numpy as np

from fake_sysfs import host_lib
from kxpu_b200.binding import VFVGPUREC_DTYPE

NV = "10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-xxxx"
VGPU = "10de,nvidia,nvidia.com,nvidia.com/vgpu,cdi-vgpu-vf"
CLASSES = NV + ";" + VGPU  # class 1 serves vGPUs on VFs
HEADER = b"ID    : vGPU Name\n"


def set_files(base, bdf, current=None, creatable=None):
    """<bdf>/nvidia/current_vgpu_type and creatable_vgpu_types (None: leave the file as it is)."""
    d = os.path.join(os.path.realpath(os.path.join(base, bdf)), "nvidia")
    os.makedirs(d, exist_ok=True)
    for name, data in (("current_vgpu_type", current), ("creatable_vgpu_types", creatable)):
        if data is not None:
            open(os.path.join(d, name), "wb").write(data)


def gather(base, dtype, classes, vf_mask, cap=1024):
    """(records, side records, nvidia/ files read) of the PCI gather with the classes of vf_mask serving vGPUs on VFs."""
    L = host_lib()
    L.kxh_gather_vf_vgpu.restype = C.c_int
    L.kxh_gather_vf_vgpu.argtypes = [C.c_char_p, C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_size_t,
                                     C.POINTER(C.c_size_t), C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    recs, vts = np.zeros(cap, dtype), np.zeros(cap, VFVGPUREC_DTYPE)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_vf_vgpu(base.encode(), classes.encode(), vf_mask, recs.ctypes.data, vts.ctypes.data, cap, C.byref(n),
                              C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], vts[:n.value], reads.value


def set_vf_vgpu(hp, cls, on=True, names=None, vgpu=False):
    """vfVgpu of passthrough class cls (vgpu: of vGPU class cls) with vgpuTypeNames {id: name}."""
    hp.L.kxh_set_vf_vgpu.restype = C.c_int
    hp.L.kxh_set_vf_vgpu.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p]
    spec = ";".join("%d=%s" % kv for kv in sorted((names or {}).items()))
    assert hp.L.kxh_set_vf_vgpu(hp.h, int(vgpu), cls, int(on), spec.encode()) == 0


def reads(hp):
    hp.L.kxh_vf_vgpu_reads.restype = C.c_uint64
    hp.L.kxh_vf_vgpu_reads.argtypes = [C.c_void_p]
    return hp.L.kxh_vf_vgpu_reads(hp.h)


def learned(hp):
    hp.L.kxh_vgpu_learned.restype = C.c_int
    hp.L.kxh_vgpu_learned.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(1 << 16)
    assert hp.L.kxh_vgpu_learned(hp.h, buf, len(buf)) >= 0
    return {int(k): v for k, v in json.loads(buf.value.decode()).items()}
