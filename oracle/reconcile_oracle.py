"""ctypes binding of the rediscovery CPU oracle (oracle/kxpu_reconcile_oracle.c): the checker of kxpu_reconcile.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kxpu_reconcile_oracle.c")
_SO = os.path.join(_HERE, "libkxpu_reconcile_oracle.so")
_LIB = None


def build():
    deps = [_SRC, os.path.join(_HERE, "..", "include", "kxpu.h")]
    if os.path.exists(_SO) and os.path.getmtime(_SO) >= max(os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-Wall", "-Wextra", "-fPIC", "-shared", "-o", _SO, _SRC])


def lib():
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(_SO)
        vp, sz = C.c_void_p, C.c_size_t
        L.kxo_reconcile.restype = C.c_int32
        L.kxo_reconcile.argtypes = [vp, sz, C.c_uint64, vp, sz, vp, vp, vp, vp]
        _LIB = L
    return _LIB


def reconcile(prev, cur, next_index):
    """kxo_reconcile: dict(index, cur_state, prev_state, counts) as Kxpu.reconcile returns it, or None when the input
    is invalid."""
    from kxpu_b200.binding import SNAPREC_DTYPE, reconcile_outputs, reconcile_result
    prev, cur = np.ascontiguousarray(prev), np.ascontiguousarray(cur)
    assert prev.dtype == SNAPREC_DTYPE and cur.dtype == SNAPREC_DTYPE
    out = reconcile_outputs(len(prev), len(cur))
    rc = lib().kxo_reconcile(prev.ctypes.data, len(prev), next_index, cur.ctypes.data, len(cur), out["index"].ctypes.data,
                             out["cur_state"].ctypes.data, out["prev_state"].ctypes.data, out["counts"].ctypes.data)
    if rc != 0:
        return None
    return reconcile_result(out)
