"""CPU test of Plugin::draVgpuPcie's start-up checks: the setting is refused, naming why, while draPcieDomain is empty
and while no vGPU class publishes DRA."""
import ctypes as C

import dra_host as DH
import dra_pcie_host as H
import fake_sysfs
import pytest


@pytest.fixture
def hp(tmp_path):
    base = H.make_tree(str(tmp_path))
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    DH.configure(p, classes=H.CLASSES, dra=H.DRIVERS)
    p.L.kxh_set_dra_vgpu_pcie.argtypes = [C.c_void_p, C.c_int]
    try:
        yield p
    finally:
        p.close()


def test_refuses_without_a_domain(hp):
    hp.L.kxh_set_dra_vgpu_pcie(hp.h, 1)
    assert DH.initiate(hp) == "draVgpuPcie is set but draPcieDomain is empty: it names the attributes"


def test_refuses_without_a_vgpu_dra_class(hp):
    H.set_domain(hp, H.DOMAIN)
    hp.L.kxh_set_dra_vgpu_pcie(hp.h, 1)
    assert DH.initiate(hp) == ("draVgpuPcie is set but no vGPU class publishes DRA (no vGPU class has a draDriver, "
                               "no class a vgpuDraDriver)")
