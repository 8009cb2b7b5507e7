"""CPU tests of the host plugin's SR-IOV reads (Plugin::sriovAware) on fake sysfs trees with physfn / virtfnN links and
sriov_numvfs files: what each gather stores, which functions it reads, the read-error flags, and no read with the setting
off."""
import ctypes as C
import os

import numpy as np
import pytest

import fake_sysfs
import sriov_host as H
from oracle import xpu_oracle as XO

NVD = dict(vendor=b"0x10de\n", device=b"0x2330\n")
DEVS = [dict(bdf="0000:03:00.0", group=30, driver="nvidia", **NVD),      # PF on a host driver: no candidate
        dict(bdf="0000:03:00.4", group=31, driver="vfio-pci", **NVD),
        dict(bdf="0000:03:00.5", group=32, driver="vfio-pci", **NVD),
        dict(bdf="0000:05:00.0", group=50, driver="vfio-pci", **NVD),    # PF on vfio-pci
        dict(bdf="0000:05:00.4", group=51, driver="vfio-pci", **NVD),
        dict(bdf="0000:06:00.0", group=60, driver="nvme", vendor=b"0x144d\n", device=b"0xa80a\n")]


@pytest.fixture
def tree(tmp_path):
    base = fake_sysfs.make_tree(str(tmp_path), DEVS)
    H.link_vfs(base, "0000:03:00.0", ["0000:03:00.4", "0000:03:00.5"], b"2\n")
    H.link_vfs(base, "0000:05:00.0", ["0000:05:00.4"], b"1\n")
    open(os.path.join(base, "0000:06:00.0", "sriov_numvfs"), "wb").write(b"4\n")  # not a candidate: never read
    return str(tmp_path), base


def _by_bdf(recs, srs):
    return {bytes(r["bdf"]).rstrip(b"\0").decode(): s for r, s in zip(recs, srs)}


@pytest.mark.parametrize("fast", [False, True])
def test_reads_of_the_candidates(tree, fast):
    _, base = tree
    recs, srs, reads = H.gather(base, XO.DEVREC_DTYPE, True, fast=fast)
    assert reads == 4  # the four vfio-pci functions of the NVIDIA class
    s = _by_bdf(recs, srs)
    assert bytes(s["0000:03:00.4"]["physfn"]) == b"0000:03:00.0" and bytes(s["0000:05:00.4"]["physfn"]) == b"0000:05:00.0"
    assert bytes(s["0000:05:00.0"]["physfn"]) == b"" and s["0000:05:00.0"]["numvfs_len"] == 2
    assert bytes(s["0000:05:00.0"]["numvfs_txt"][:2]) == b"1\n"
    for bdf in ("0000:03:00.0", "0000:06:00.0"):  # no candidates: zero-filled
        assert s[bdf].tobytes() == bytes(32)
    assert all(int(x["flags"]) == 0 for x in srs)
    # the records themselves are the gather's without the setting
    recs_off, srs_off, reads_off = H.gather(base, XO.DEVREC_DTYPE, False, fast=fast)
    assert recs_off.tobytes() == recs.tobytes()
    assert reads_off == 0 and srs_off.tobytes() == bytes(32 * len(srs_off))


def test_read_errors(tree):
    _, base = tree
    vf = os.path.realpath(os.path.join(base, "0000:05:00.4"))
    os.remove(os.path.join(vf, "physfn"))
    open(os.path.join(vf, "physfn"), "w").write("x")  # not a link: readlink fails with EINVAL
    pf = os.path.realpath(os.path.join(base, "0000:05:00.0"))
    os.remove(os.path.join(pf, "sriov_numvfs"))
    os.mkdir(os.path.join(pf, "sriov_numvfs"))  # a directory: the read fails
    long_vf = os.path.realpath(os.path.join(base, "0000:03:00.5"))
    os.remove(os.path.join(long_vf, "physfn"))
    os.symlink("../0000:03:00.0-and-more", os.path.join(long_vf, "physfn"))  # longer than an address can be
    open(os.path.join(base, "0000:03:00.4", "sriov_numvfs"), "wb").write(b"123456789\n")
    recs, srs, _ = H.gather(base, XO.DEVREC_DTYPE, True)
    s = _by_bdf(recs, srs)
    assert s["0000:05:00.4"]["flags"] == 1 and bytes(s["0000:05:00.4"]["physfn"]) == b""
    assert s["0000:05:00.0"]["flags"] == 2
    assert s["0000:03:00.5"]["flags"] == 1
    assert s["0000:03:00.4"]["numvfs_len"] == 9 and bytes(s["0000:03:00.4"]["numvfs_txt"]) == b"12345678"
    assert s["0000:03:00.4"]["flags"] == 0



def test_vf_uevents_end_the_snapshot():
    """Enabling VFs adds PCI functions, disabling removes them, and rebinding a PF unbinds and binds it: each moves the
    bind generation that snapshot validation compares, so a changed SR-IOV verdict never answers from the snapshot."""
    L = fake_sysfs.host_lib()
    L.kxh_uevent_feed.restype = C.c_uint64
    L.kxh_uevent_feed.argtypes = [C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.kxh_uevent_free.argtypes = [C.c_void_p]
    w = C.c_void_p(None)

    def feed(*fields):
        m = b"\0".join(fields) + b"\0"
        return L.kxh_uevent_feed(C.byref(w), m, len(m))

    vf = b"/devices/pci0000:00/0000:00:01.0/0000:03:00.4"
    pf = b"/devices/pci0000:00/0000:00:01.0/0000:03:00.0"
    assert feed(b"add@" + vf, b"ACTION=add", b"DEVPATH=" + vf, b"SUBSYSTEM=pci") == 1  # echo 1 > sriov_numvfs
    assert feed(b"unbind@" + pf, b"ACTION=unbind", b"DEVPATH=" + pf, b"SUBSYSTEM=pci") == 2
    assert feed(b"bind@" + pf, b"ACTION=bind", b"DEVPATH=" + pf, b"SUBSYSTEM=pci", b"DRIVER=vfio-pci") == 3
    assert feed(b"remove@" + vf, b"ACTION=remove", b"DEVPATH=" + vf, b"SUBSYSTEM=pci") == 4  # echo 0 > sriov_numvfs
    L.kxh_uevent_free(w)
