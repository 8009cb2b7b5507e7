"""CPU tests of the start-up checks of XpuClass::vgpuDraDriver (the DRA driver of a vfVgpu class's vGPUs): refused on a
class without vfVgpu and on a vGPU class, naming the class; a driver that another class already uses and an empty node
name are refused as for every DRA driver; draDriver on a vfVgpu class keeps its refusal."""
import ctypes as C

import pytest

import dra_host as DH
import dra_vf_vgpu_host as VH
import fake_sysfs
import vf_vgpu_host as H

DEVS = [dict(bdf="0000:03:00.0", group=30, vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia"),
        dict(bdf="0000:03:00.4", group=31, vendor=b"0x10de\n", device=b"0x2331\n", driver="nvidia")]


@pytest.fixture
def hp(tmp_path):
    base = fake_sysfs.make_tree(str(tmp_path), DEVS)
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    assert p.L.kxh_set_classes(p.h, H.CLASSES.encode()) == 0
    try:
        yield p
    finally:
        p.close()


def test_refused_without_vf_vgpu(hp):
    VH.set_driver(hp, 0, "vgpu-vf.nvidia.com")
    assert DH.initiate(hp) == ("class 10de/vfio-pci (nvidia.com/gpu): vgpuDraDriver vgpu-vf.nvidia.com needs vfVgpu on "
                               "the class")


def test_refused_on_a_vgpu_class(hp):
    hp.L.kxh_set_vgpu_classes.argtypes = [C.c_void_p, C.c_char_p]
    assert hp.L.kxh_set_vgpu_classes(hp.h, b"10de,nvidia-vgpu-vfio,nvidia.com,nvidia.com/mdev,cdi-mdev") == 0
    H.set_vf_vgpu(hp, 1)
    VH.set_driver(hp, 0, "vgpu-vf.nvidia.com", vgpu=True)
    assert DH.initiate(hp) == ("vGPU class 10de/nvidia-vgpu-vfio (nvidia.com/mdev): vgpuDraDriver vgpu-vf.nvidia.com "
                               "applies to vfVgpu classes only")


@pytest.mark.parametrize("other", ["passthrough", "vgpu"])
def test_refused_when_another_class_uses_the_driver(hp, other):
    H.set_vf_vgpu(hp, 1)
    if other == "passthrough":
        DH.configure(hp, dra=["vfio.nvidia.com", ""])
        VH.set_driver(hp, 1, "vfio.nvidia.com")
        assert DH.initiate(hp) == "DRA driver vfio.nvidia.com is set on two classes (0 and 1 vGPUs)"
    else:
        hp.L.kxh_set_vgpu_classes.argtypes = [C.c_void_p, C.c_char_p]
        assert hp.L.kxh_set_vgpu_classes(hp.h, b"10de,nvidia-vgpu-vfio,nvidia.com,nvidia.com/mdev,cdi-mdev") == 0
        hp.L.kxh_set_vgpu_dra.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        assert hp.L.kxh_set_vgpu_dra(hp.h, b"vgpu.nvidia.com", b"node-a") == 0
        VH.set_driver(hp, 1, "vgpu.nvidia.com")
        assert DH.initiate(hp) == "DRA driver vgpu.nvidia.com is set on two classes (vGPU 0 and 1 vGPUs)"


def test_refused_without_a_node_name(hp):
    H.set_vf_vgpu(hp, 1)
    VH.set_driver(hp, 1, "vgpu-vf.nvidia.com", node="")
    assert DH.initiate(hp) == "DRA driver vgpu-vf.nvidia.com is set but the node name is empty (NODE_NAME)"


def test_dra_driver_on_a_vf_vgpu_class_is_still_refused(hp):
    H.set_vf_vgpu(hp, 1)
    VH.set_driver(hp, 1, "vgpu-vf.nvidia.com")
    DH.configure(hp, dra=["", "vgpu.nvidia.com"])
    assert DH.initiate(hp) == ("class 10de/nvidia (nvidia.com/vgpu): vfVgpu cannot be published as DRA ResourceSlices "
                               "(draDriver vgpu.nvidia.com)")


def test_slices_need_the_driver(hp):
    with pytest.raises(RuntimeError, match="VfVgpuResourceSlices: class 1 has no vGPU DRA driver"):
        VH.slices(hp, 1)
