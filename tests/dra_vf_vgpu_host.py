"""Fake-sysfs helpers for the host plugin's DRA ResourceSlices of vGPUs on SR-IOV VFs (XpuClass::vgpuDraDriver,
Plugin::VfVgpuResourceSlices): the setting and the slices."""
import ctypes as C

import numpy as np

from fake_sysfs import host_lib


def _lib():
    L = host_lib()
    L.kxh_set_vf_vgpu_dra.restype = C.c_int
    L.kxh_set_vf_vgpu_dra.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p, C.c_char_p]
    L.kxh_vf_vgpu_slices.restype = C.c_int
    L.kxh_vf_vgpu_slices.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p,
                                     C.c_size_t, C.POINTER(C.c_size_t)]
    return L


def set_driver(hp, cls, driver, node="node-a", vgpu=False):
    """vgpuDraDriver of passthrough class cls (vgpu: of vGPU class cls), and the node name"""
    assert _lib().kxh_set_vf_vgpu_dra(hp.h, int(vgpu), cls, driver.encode(), node.encode()) == 0


def slices(hp, cls):
    """(bytes, slice_off) of VfVgpuResourceSlices(cls); RuntimeError with the message on failure"""
    L = _lib()
    ln, ns = C.c_size_t(0), C.c_size_t(0)
    out, offs = np.zeros(1 << 16, np.uint8), np.zeros(1024, np.uint64)
    rc = L.kxh_vf_vgpu_slices(hp.h, cls, out.ctypes.data, out.size, C.byref(ln), offs.ctypes.data, offs.size, C.byref(ns))
    if rc == -1:
        raise RuntimeError(out.tobytes().split(b"\0", 1)[0].decode())
    assert rc == 0, rc
    return out[:ln.value].tobytes(), offs[:ns.value + 1]
