"""Independent Python restatement of kxpu_aer_ports and kxpu_aer_ports_mdev (include/kxpu.h, additions to ABI v14), the
second checker next to tests/aer_ports_oracle.c: each record's chain from pyref_pcie / pyref_pcie_mdev (the mdev chain
less its parent), its function keys reversed, and the port numbers from a dict in first-seen order.  It shares no code
with the kernels."""
import numpy as np

import pyref_pcie as PP
import pyref_pcie_mdev as PM

HOST_BRIDGE = 1 << 63


def record_ports(rec, path_row, mdev):
    """the port keys of one record, nearest first"""
    chain = PM.record_chain(rec, path_row)[:-1] if mdev else PP.record_chain(rec, path_row)
    return [k for k in reversed(chain) if not k & HOST_BRIDGE]


def aer_ports(recs, paths, mdev=False):
    """(port_off, port_of, port_key) as lists"""
    number = {}
    off, of = [0], []
    for r, p in zip(recs, paths):
        for k in record_ports(r, p, mdev):
            of.append(number.setdefault(k, len(number)))
        off.append(len(of))
    return off, of, list(number)


def as_arrays(res):
    off, of, key = res
    return np.array(off, np.uint32), np.array(of, np.uint32), np.array(key, np.uint64)
