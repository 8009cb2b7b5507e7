"""CPU tests of the host plugin's reads for vGPUs on SR-IOV VFs (XpuClass::vfVgpu) on fake sysfs trees: which functions
the gather reads (only the class's VFs, never the PF), what it stores, nothing read and byte-identical records without
the setting, and the two configuration refusals."""
import ctypes as C

import pytest

import dra_host as DH
import fake_sysfs
import sriov_host as SH
import vf_vgpu_host as H
import xpu_host
from oracle import xpu_oracle as XO

NVD = dict(vendor=b"0x10de\n", device=b"0x2331\n", driver="nvidia")
DEVS = [dict(bdf="0000:03:00.0", group=30, vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia"),  # the PF
        dict(bdf="0000:03:00.4", group=31, **NVD), dict(bdf="0000:03:00.5", group=32, **NVD),
        dict(bdf="0000:03:00.6", group=33, **NVD),
        dict(bdf="0000:05:00.0", group=50, vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci"),  # passthrough
        dict(bdf="0000:05:00.4", group=51, vendor=b"0x10de\n", device=b"0x2331\n", driver="vfio-pci")]  # its VF

H_READ, H_CUR_ERR = 1, 2  # KXPU_VT_READ, KXPU_VT_CUR_ERR


@pytest.fixture
def tree(tmp_path):
    base = fake_sysfs.make_tree(str(tmp_path), DEVS)
    SH.link_vfs(base, "0000:03:00.0", ["0000:03:00.4", "0000:03:00.5", "0000:03:00.6"], b"3\n")
    SH.link_vfs(base, "0000:05:00.0", ["0000:05:00.4"], b"1\n")
    H.set_files(base, "0000:03:00.0", b"0\n", H.HEADER + b"557 : A\n")  # a PF never has these; never read anyway
    H.set_files(base, "0000:03:00.4", b"557\n", H.HEADER)
    H.set_files(base, "0000:03:00.5", b"0\n", H.HEADER + b"557 : NVIDIA H100-4C\n")
    H.set_files(base, "0000:05:00.4", b"557\n", H.HEADER)  # not a vfVgpu class: never read
    return str(tmp_path), base


def _by_bdf(recs, vts):
    return {bytes(r["bdf"]).rstrip(b"\0").decode(): v for r, v in zip(recs, vts)}


def test_off_reads_nothing(tree):
    _, base = tree
    recs, vts, reads = H.gather(base, XO.DEVREC_DTYPE, H.CLASSES, 0)
    assert reads == 0 and vts.tobytes() == bytes(32 * len(vts))
    want = xpu_host.gather_classes(base, XO.DEVREC_DTYPE, [c.split(",") for c in H.CLASSES.split(";")])
    assert recs.tobytes() == want.tobytes()


def test_reads_the_class_vfs_only(tree):
    _, base = tree
    recs, vts, reads = H.gather(base, XO.DEVREC_DTYPE, H.CLASSES, 0b10)
    assert reads == 6  # two files for each of the three VFs of the vfVgpu class
    v = _by_bdf(recs, vts)
    for bdf in ("0000:03:00.0", "0000:05:00.0", "0000:05:00.4"):  # the PF, and the other class's functions
        assert v[bdf].tobytes() == bytes(32)
    assert bytes(v["0000:03:00.4"]["cur_txt"][:4]) == b"557\n" and v["0000:03:00.4"]["cur_len"] == 4
    assert v["0000:03:00.4"]["flags"] == H_READ
    assert v["0000:03:00.6"]["flags"] == H_READ | H_CUR_ERR  # no nvidia/ directory: a failed read
    off, _, _ = H.gather(base, XO.DEVREC_DTYPE, H.CLASSES, 0)
    assert off.tobytes() == recs.tobytes()


def test_long_current_type_is_marked(tree):
    _, base = tree
    H.set_files(base, "0000:03:00.4", b"1" * 40)
    recs, vts, _ = H.gather(base, XO.DEVREC_DTYPE, H.CLASSES, 0b10)
    v = _by_bdf(recs, vts)["0000:03:00.4"]
    assert v["cur_len"] == 17 and bytes(v["cur_txt"]) == b"1" * 16



def _plugin(tree, classes=H.CLASSES):
    root, base = tree
    hp = fake_sysfs.HostPlugin(type("NoGpu", (), {"ctx": None})(), base, root + "/pci.ids", root + "/")
    assert hp.L.kxh_set_classes(hp.h, classes.encode()) == 0
    return hp


def test_refused_with_a_dra_driver(tree):
    hp = _plugin(tree)
    try:
        H.set_vf_vgpu(hp, 1)
        DH.configure(hp, dra=["", "vgpu.nvidia.com"])
        assert DH.initiate(hp) == ("class 10de/nvidia (nvidia.com/vgpu): vfVgpu cannot be published as DRA ResourceSlices "
                                   "(draDriver vgpu.nvidia.com)")
    finally:
        hp.close()


def test_refused_on_a_vgpu_class(tree):
    hp = _plugin(tree, H.NV)
    try:
        hp.L.kxh_set_vgpu_classes.argtypes = [C.c_void_p, C.c_char_p]
        assert hp.L.kxh_set_vgpu_classes(hp.h, b"10de,nvidia-vgpu-vfio,nvidia.com,nvidia.com/mdev,cdi-mdev") == 0
        H.set_vf_vgpu(hp, 0, vgpu=True)
        assert DH.initiate(hp) == "vGPU class 10de/nvidia-vgpu-vfio (nvidia.com/mdev): vfVgpu applies to passthrough classes only"
    finally:
        hp.close()
