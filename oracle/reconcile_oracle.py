"""ctypes binding of the rediscovery CPU oracle (oracle/kxpu_reconcile_oracle.c): the checker of kxpu_reconcile.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import numpy as np

from . import oracle as O


def reconcile(prev, cur, next_index):
    """kxo_reconcile: dict(index, cur_state, prev_state, counts) as Kxpu.reconcile returns it, or None when the input
    is invalid."""
    from kxpu_b200.binding import SNAPREC_DTYPE, reconcile_outputs, reconcile_result
    prev, cur = np.ascontiguousarray(prev), np.ascontiguousarray(cur)
    assert prev.dtype == SNAPREC_DTYPE and cur.dtype == SNAPREC_DTYPE
    out = reconcile_outputs(len(prev), len(cur))
    rc = O.lib().kxo_reconcile(prev.ctypes.data, len(prev), next_index, cur.ctypes.data, len(cur),
                               out["index"].ctypes.data, out["cur_state"].ctypes.data, out["prev_state"].ctypes.data,
                               out["counts"].ctypes.data)
    if rc != 0:
        return None
    return reconcile_result(out)
