"""ctypes binding of the IOMMU group viability CPU oracle (oracle/kxpu_viab_oracle.c): the checker of
kxpu_classify_viable.

TEST INFRASTRUCTURE ONLY, like oracle.py: imported by tests/, never by the product package.
"""
import numpy as np

from . import oracle as O
from . import xpu_oracle as XO

VIABLE = 0xFFFFFFFF


def classify_viable(rules, recs: np.ndarray, topo=False):
    """kxo_classify_viable: the classify dict plus dev_rule, group_blocker and (topo=True) group_numa.  A failing call
    returns its status instead: -1 for an invalid rule list, -7 for a blocker of group 0xFFFFFFFF."""
    ra = XO.rules_array(rules)
    assert recs.dtype.itemsize == 64
    rc, res = O.classify_call(O.lib().kxo_classify_viable, (ra.ctypes.data if len(ra) else None, len(ra)), recs,
                              dev=[("dev_rule", np.uint8)],
                              group=[("group_numa", np.uint64 if topo else None), ("group_blocker", np.uint32)])
    return rc if rc != 0 else res
