"""CPU tests of Plugin::vfVgpuHealth's start-up check and of its refresh with the setting off: refused without a vfVgpu
class, and refreshVfVgpuTypes reads nothing and reports nothing when the setting is off."""
import ctypes as C

import dra_host as DH
import fake_sysfs
import pytest
import vf_vgpu_host as H

DEVS = [dict(bdf="0000:03:00.0", group=30, vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia"),
        dict(bdf="0000:03:00.4", group=31, vendor=b"0x10de\n", device=b"0x2331\n", driver="nvidia")]


@pytest.fixture
def hp(tmp_path):
    base = fake_sysfs.make_tree(str(tmp_path), DEVS)
    H.set_files(base, DEVS[1]["bdf"], b"557\n", H.HEADER)
    p = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, str(tmp_path / "pci.ids"), str(tmp_path) + "/")
    assert p.L.kxh_set_classes(p.h, H.CLASSES.encode()) == 0
    p.L.kxh_set_vf_vgpu_health.argtypes = [C.c_void_p, C.c_int]
    try:
        yield p
    finally:
        p.close()


def test_refused_without_a_vf_vgpu_class(hp):
    hp.L.kxh_set_vf_vgpu_health(hp.h, 1)
    assert DH.initiate(hp) == "vfVgpuHealth is set but no class has vfVgpu"


def test_off_refresh_reads_nothing(hp):
    L = hp.L
    L.kxh_refresh_vf_vgpu_types.restype = C.c_int
    L.kxh_refresh_vf_vgpu_types.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                            C.POINTER(C.c_int), C.c_char_p, C.c_size_t]
    H.set_vf_vgpu(hp, 1)
    changed, n, moved, err = (C.c_size_t * 8)(), C.c_size_t(7), C.c_int(-1), C.create_string_buffer(256)
    assert L.kxh_refresh_vf_vgpu_types(hp.h, changed, 8, C.byref(n), C.byref(moved), err, len(err)) == 0, err.value
    assert n.value == 0 and moved.value == 0 and H.reads(hp) == 0
