"""CPU test of Plugin::sriovPfAware's start-up check: refused while sriovAware is off, before any walk."""
import dra_host as DH
import dra_pf_host as H
import fake_sysfs
import pytest
import sriov_host as SH


@pytest.fixture
def hp(tmp_path):
    base = H.make_tree(str(tmp_path))
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    assert p.L.kxh_set_classes(p.h, H.CLASSES.encode()) == 0
    try:
        yield p
    finally:
        p.close()


def test_refused_without_sriov_aware(hp):
    H.enable(hp, True)
    assert DH.initiate(hp) == "sriovPfAware is set but sriovAware is off"
    SH.set_sriov(hp, False)
    assert DH.initiate(hp) == "sriovPfAware is set but sriovAware is off"
