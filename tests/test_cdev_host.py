"""CPU checks of the host walk for classes served through VFIO cdevs (XpuClass::vfioCdev) on fake sysfs trees: canonical
vfio-dev/ entries are read, every malformed case means "no cdev", the plain and fast gathers agree, nothing under
vfio-dev/ is opened without a cdev class, and a vGPU class cannot set vfioCdev."""
import numpy as np
import pytest

import cdev_host as H
import fake_sysfs
from kxpu_b200.binding import DEVREC_DTYPE

GPU = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
CASES = [  # (vfio-dev entries or None, expected cdev)
    (["vfio0"], 0), (["vfio9"], 9), (["vfio10"], 10), (["vfio4294967295"], (1 << 32) - 1),
    (None, -1), ([], -1), (["vfio1", "vfio2"], -1), (["vfio01"], -1), (["vfio"], -1), (["vfio4294967296"], -1),
    (["vfio99999999999"], -1), (["vfio1x"], -1), (["cdev1"], -1), (["vfio-1"], -1), (["vfio+1"], -1), (["VFIO1"], -1)]


def _tree(tmp_path):
    devs = [dict(bdf="0000:%02x:00.0" % (k + 1), group=30 + k, **GPU) for k in range(len(CASES))]
    devs.append(dict(bdf="0000:80:00.0", group=90, vendor=b"0x8086\n", device=b"0x1533\n", driver="vfio-pci"))  # no class
    base = fake_sysfs.make_tree(str(tmp_path), devs)
    for k, (entries, _) in enumerate(CASES):
        H.set_vfio_dev(base, "0000:%02x:00.0" % (k + 1), entries)
    H.set_vfio_dev(base, "0000:80:00.0", ["vfio7"])  # read only for a function of a cdev class
    return base


@pytest.mark.parametrize("fast,threads", [(False, 0), (True, 1), (True, 4)])
def test_gather_reads_cdevs(tmp_path, fast, threads):
    base = _tree(tmp_path)
    recs, cdevs, reads = H.gather(base, DEVREC_DTYPE, [H.NV_CDEV], fast, threads)
    assert [r.decode() for r in recs["bdf"]][:len(CASES)] == ["0000:%02x:00.0" % (k + 1) for k in range(len(CASES))]
    assert list(cdevs) == [want for _, want in CASES] + [-1]
    assert reads == len(CASES)


def test_plain_and_fast_gathers_agree(tmp_path):
    base = _tree(tmp_path)
    a = H.gather(base, DEVREC_DTYPE, [H.NV, ("8086", "vfio-pci", "intel.com", "intel.com/nic", "nic", "cdev")])
    b = H.gather(base, DEVREC_DTYPE, [H.NV, ("8086", "vfio-pci", "intel.com", "intel.com/nic", "nic", "cdev")], True, 3)
    assert a[0].tobytes() == b[0].tobytes() and list(a[1]) == list(b[1]) and a[2] == b[2] == 1
    assert list(a[1]) == [-1] * len(CASES) + [7]  # only the cdev class's function is read


@pytest.mark.parametrize("fast", [False, True])
def test_no_cdev_class_reads_nothing(tmp_path, fast):
    base = _tree(tmp_path)
    recs, cdevs, reads = H.gather(base, DEVREC_DTYPE, [H.NV], fast, 2)
    assert reads == 0 and (cdevs == -1).all()
    plain = fake_sysfs.gather(base, DEVREC_DTYPE)
    assert recs.tobytes() == plain.tobytes()  # the records themselves do not change


def test_vgpu_class_cannot_be_cdev():
    vgpu = ("10de", "nvidia", "nvidia.com", "nvidia.com/vgpu", "cdi-vgpu")
    assert H.check_vgpu_classes([H.NV], [vgpu]) is None
    err = H.check_vgpu_classes([H.NV], [vgpu + ("cdev",)])
    assert err is not None and "nvidia.com/vgpu" in err and "vfioCdev" in err
