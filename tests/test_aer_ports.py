"""CPU tests of the PCIe ports above every record (kxpu_aer_ports and kxpu_aer_ports_mdev, include/kxpu.h) on the C
checker (tests/aer_ports_oracle.c) and the Python restatement (tests/pyref_aer_ports.py): both on the hand cases, against
each other on seeded walks, the mdev rule against the parents' own PCI records, and the first-occurrence numbering."""
import numpy as np

import pytest
from hypothesis import given, settings, strategies as st

import aer_ports_cases as AC
import aer_ports_oracle as CO
import dra_pcie_cases as DC
import pyref_aer_ports as R
import vgpu_pcie_cases as VC


def _lists(res):
    return tuple([int(x) for x in a] for a in res)


@pytest.mark.parametrize("case", AC.PCI, ids=[c[0] for c in AC.PCI])
def test_pci_hand_cases(case):
    _, rows, want = case
    recs, paths = AC.pci_walk(rows)
    assert R.aer_ports(recs, paths) == AC.expected(want)
    assert _lists(CO.aer_ports(recs, paths)) == AC.expected(want)


@pytest.mark.parametrize("case", AC.MDEV, ids=[c[0] for c in AC.MDEV])
def test_mdev_hand_cases(case):
    _, rows, want = case
    recs, paths = AC.mdev_walk(rows)
    assert R.aer_ports(recs, paths, mdev=True) == AC.expected(want)
    assert _lists(CO.aer_ports(recs, paths)) == AC.expected(want)


def test_first_occurrence_numbering():
    _, rows, _ = next(c for c in AC.PCI if c[0] == "first_occurrence")
    off, of, key = R.aer_ports(*AC.pci_walk(rows))
    assert of == [0, 1, 2, 3, 4, 1, 3, 4]
    assert key == [DC.fkey(a) for a in ["0000:41:00.0", "0000:40:01.0", "0000:02:00.0", "0000:01:00.0", "0000:00:01.0"]]
    assert off == [0, 2, 5, 6, 8]


@settings(max_examples=60, deadline=None)
@given(st.integers(0, 120), st.integers(0, 2 ** 31), st.floats(0, 0.5))
def test_pci_restatements_agree(n_groups, seed, unknown):
    recs, paths, _, _ = DC.random_walk(n_groups, seed, unknown=unknown)
    assert _lists(CO.aer_ports(recs, paths)) == R.aer_ports(recs, paths)


@settings(max_examples=60, deadline=None)
@given(st.integers(0, 200), st.integers(0, 2 ** 31))
def test_mdev_restatements_agree(n, seed):
    (recs, paths, _, _), _ = VC.random_walk(n, seed)
    assert _lists(CO.aer_ports(recs, paths)) == R.aer_ports(recs, paths, mdev=True)


@settings(max_examples=40, deadline=None)
@given(st.integers(0, 200), st.integers(0, 2 ** 31))
def test_mdev_ports_are_the_parents(n, seed):
    (recs, paths, _, _), (precs, ppaths, _, _) = VC.random_walk(n, seed, unknown=0)
    assert R.aer_ports(recs, paths, mdev=True) == R.aer_ports(precs, ppaths)


def test_large_walk_agrees():
    import kxpu_b200  # noqa: F401
    from kxpu_b200 import workloads as W
    recs, paths = W.aer_port_walk(1 << 12, depth=3, fanout=4, seed=5)
    got = CO.aer_ports(recs, paths)
    want = R.as_arrays(R.aer_ports(recs, paths))
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
