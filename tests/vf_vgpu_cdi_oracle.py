"""The C statement of the typed VF-vGPU CDI layouts (kxpu_cdi_emit_vf_vgpu / _cdev), next to tests/pyref_vf_vgpu_cdi.py: a
ctypes binding of tests/vf_vgpu_cdi_oracle.c, compiled once per process into a temporary directory, so the tree stays
read-only.

TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from conftest import ROOT
from kxpu_b200.binding import VFVGPUCDI_DTYPE

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="kxv_"), "libkxv_vf_vgpu_cdi.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-Werror", "-fPIC", "-shared",
                               "-I", os.path.join(ROOT, "include"), "-o", out,
                               os.path.join(os.path.dirname(os.path.abspath(__file__)), "vf_vgpu_cdi_oracle.c")])
        L = C.CDLL(out)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxv_cdi_vf_vgpu.restype = C.c_int
        L.kxv_cdi_vf_vgpu.argtypes = [C.c_int, C.c_char_p, vp, sz, C.c_int, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(sz)]
        L.kxv_free.restype = None
        L.kxv_free.argtypes = [C.POINTER(C.c_uint8)]
        _LIB = L
    return _LIB


def emit(fmt, kind, recs, cdev=False):
    """The document of VFVGPUCDI_DTYPE records, or None when the kind or a record is outside the domain."""
    recs = np.ascontiguousarray(recs)
    assert recs.dtype == VFVGPUCDI_DTYPE
    kind = kind.encode() if isinstance(kind, str) else kind
    L = lib()
    p, n = C.POINTER(C.c_uint8)(), C.c_size_t(0)
    rc = L.kxv_cdi_vf_vgpu(fmt, kind, recs.ctypes.data if len(recs) else None, len(recs), int(cdev), C.byref(p), C.byref(n))
    if rc == -7:
        return None
    assert rc == 0, rc
    try:
        return C.string_at(p, n.value)
    finally:
        L.kxv_free(p)
