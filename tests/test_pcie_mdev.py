"""CPU tests of kxpu_pcie_tree_mdev's semantics (include/kxpu.h, addition to ABI v14): the C checker
(tests/pcie_mdev_oracle.c) against the Python restatement (tests/pyref_pcie_mdev.py) on every hand case and under
hypothesis, the chain lengths the grammar gives, and the link to kxpu_pcie_tree's grammar: a known mdev chain is the
parent function's own chain followed by the parent's key."""
import os
import re

import numpy as np
from hypothesis import given, settings

import pcie_mdev_cases as MC
import pcie_mdev_oracle as MO
import pyref_pcie as PP
import pyref_pcie_mdev as P
from conftest import ROOT


def _both(recs, paths, off, mem):
    want = MO.tree(recs, paths, off, mem)
    assert want == P.tree(recs, paths, off, mem)
    return want


def test_hand_cases_agree():
    for name, (recs, paths, off, mem) in MC.HAND.items():
        _both(recs, paths, off, mem)
        for i in range(len(recs)):
            assert MO.parse(recs[i], paths[i]) == P.record_chain(recs[i], paths[i]), (name, i)


def test_chain_lengths():
    for name, want in MC.CHAIN_LEN.items():
        recs, paths, _, _ = MC.HAND[name]
        assert len(MO.parse(recs[0], paths[0])) == want, name


def test_example_tree():
    recs, paths, off, mem = MC.HAND["two_vgpus_one_gpu"]
    t = _both(recs, paths, off, mem)
    # host bridge, root port, switch up port, switch down port, the GPU; both vGPUs hang off the GPU's node
    assert t["depth"] == [0, 1, 2, 3, 4] and t["parent"] == [MC.NO_NODE, 0, 1, 2, 3]
    assert t["key"][4] == 0x0000 << 16 | 0x03 << 8 | 0 << 3 | 0
    assert t["key"][0] == 1 << 63
    assert t["group_node"] == [4, 4]


def test_two_gpus_one_switch_share_the_switch():
    t = _both(*MC.HAND["two_gpus_one_switch"])
    a, b = t["group_node"]
    assert a != b and t["parent"][t["parent"][a]] == t["parent"][t["parent"][b]]  # the down ports' common up port


def test_mixed_and_unknown_groups():
    t = _both(*MC.HAND["group_mixed_parents"])
    # the group of the two parents ends at the switch's up port; the other group reaches its GPU below it
    g0, g1 = t["group_node"]
    assert t["depth"][g0] == 2 and t["depth"][g1] == 4
    t = _both(*MC.HAND["group_unknown_and_known"])
    assert t["depth"][t["group_node"][0]] == 4  # the unknown member does not cut the chain
    assert _both(*MC.HAND["group_all_unknown"]) == dict(group_node=[MC.NO_NODE], key=[], parent=[], depth=[])


def test_vf_parent_is_the_last_key():
    t = _both(*MC.HAND["mdev_on_a_vf"])
    a, b = t["group_node"]
    assert t["depth"][a] == t["depth"][b] == 4 and t["parent"][a] == t["parent"][b]


def test_empty_and_invalid():
    recs, paths, off, mem = MC.HAND["empty"]
    assert _both(recs, paths, off, mem) == dict(group_node=[], key=[], parent=[], depth=[])
    recs, paths, off, mem = MC.HAND["two_vgpus_one_gpu"]
    assert MO.tree(recs, paths, np.array([0, 2, 1], np.uint32), mem) is None
    assert P.tree(recs, paths, np.array([0, 2, 1], np.uint32), mem) is None
    assert MO.tree(recs, paths, off, np.array([0, 2], np.uint32)) is None
    assert P.tree(recs, paths, off, np.array([0, 2], np.uint32)) is None


@settings(max_examples=400, deadline=None, derandomize=True)
@given(MC.mdev_walks())
def test_fuzz(w):
    recs, paths, off, mem = w
    _both(recs, paths, off, mem)
    for i in range(len(recs)):
        c = P.record_chain(recs[i], paths[i])
        if not c:
            continue
        # the PCI grammar over the path without the UUID, the parent as the function itself
        text = bytes(paths[i]["path"])[:int(paths[i]["len"])].rsplit(b"/", 1)[0]
        parent = bytes(recs[i]["parent"]).split(b"\0", 1)[0]
        assert c == PP.chain(parent, text, len(text)) + [PP.component_key(parent.decode())[0]]


def test_header_declares_the_call():
    from kxpu_b200 import binding as B
    hdr = open(os.path.join(ROOT, "include", "kxpu.h")).read()
    assert re.search(r"int32_t kxpu_pcie_tree_mdev\(", hdr) and "kxpu_pcie_tree_mdev" in B.ABI_SYMBOLS
