"""CPU tests of the mdev walk's VFIO cdev reads (XpuClass::mdevCdev) on a fake /sys/bus/mdev/devices tree: the cdev side
array for canonical and malformed <uuid>/vfio-dev/ entries, reads only for mdevCdev classes, and the class checks in
both directions."""
import ctypes as C

import numpy as np

import cdev_host
import fake_mdev
import fake_sysfs
from fake_sysfs import host_lib
from oracle import mdev_oracle as mo

NVV = ("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")
NVV_CDEV = NVV + ("mdev-cdev",)
INTEL = ("8086", "vfio_mdev", "intel.com", "intel.com/gvt", "cdi-mdev-intel")
PARENTS = [dict(bdf="0000:3b:00.0", vendor=b"0x10de\n", device=b"0x1eb8\n", driver="nvidia", group=40),
           dict(bdf="0000:00:02.0", vendor=b"0x8086\n", device=b"0x3e92\n", driver="i915", group=1)]
U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(16)]
MDEVS = [dict(uuid=U[k], parent="0000:3b:00.0", group=300 + k) for k in range(1, 10)] + \
        [dict(uuid=U[10], parent="0000:00:02.0", group=310),
         dict(uuid=U[11], parent="0000:3b:00.0", group=311, driver=None),  # unbound: never read
         dict(uuid=U[12], kind="dir")]                                      # a directory entry: never read
# uuid -> vfio-dev/ entries (None: no vfio-dev/) and the N the walk must report (-1: no cdev)
VFIO_DEV = {U[1]: (["vfio0"], 0), U[2]: (["vfio4294967295"], (1 << 32) - 1), U[3]: (["vfio17"], 17),
            U[4]: (None, -1), U[5]: ([], -1), U[6]: (["vfio1", "vfio2"], -1), U[7]: (["vfio01"], -1),
            U[8]: (["vfio"], -1), U[9]: (["vfio4294967296"], -1), U[10]: (["vfio3"], 3), U[11]: (["vfio4"], 4)}


def make(tmp_path):
    fake_sysfs.make_tree(str(tmp_path), PARENTS)
    base = fake_mdev.make_tree(str(tmp_path), MDEVS)
    for u, (entries, _) in VFIO_DEV.items():
        cdev_host.set_vfio_dev(base, u, entries)
    return base


def gather(base, classes, cap=256):
    """(records, cdevs, vfio-dev reads) of the mdev gather under a vGPU class list."""
    L = host_lib()
    L.kxh_gather_mdev_cdev.restype = C.c_int
    L.kxh_gather_mdev_cdev.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                       C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    recs = np.zeros(cap, mo.MDEVREC_DTYPE)
    cdevs = np.zeros(cap, np.int64)
    n, reads = C.c_size_t(0), C.c_uint64(0)
    err = C.create_string_buffer(512)
    rc = L.kxh_gather_mdev_cdev(base.encode(), cdev_host.spec(classes), recs.ctypes.data, cdevs.ctypes.data, cap, C.byref(n),
                                C.byref(reads), err, 512)
    if rc != 0:
        raise RuntimeError(err.value.decode())
    return recs[:n.value], cdevs[:n.value], reads.value


def by_uuid(recs, cdevs):
    return {r["uuid"].decode(): int(c) for r, c in zip(recs, cdevs) if r["uuid"]}


def test_cdev_entries(tmp_path):
    base = make(tmp_path)
    recs, cdevs, reads = gather(base, [NVV_CDEV, INTEL])
    got = by_uuid(recs, cdevs)
    for u in U[1:10]:
        assert got[u] == VFIO_DEV[u][1], u
    assert got[U[10]] == -1  # the Intel class does not set mdevCdev
    assert got[U[11]] == -1 and got[U[12]] == -1  # an unbound entry and a directory are not read
    assert reads == 9
    # the records are the walk's, with or without the setting
    assert recs.tobytes() == fake_mdev.gather(base, [NVV, INTEL]).tobytes()


def test_reads_only_for_mdev_cdev_classes(tmp_path):
    base = make(tmp_path)
    recs, cdevs, reads = gather(base, [NVV, INTEL])
    assert reads == 0 and (cdevs == -1).all()
    recs, cdevs, reads = gather(base, [NVV, INTEL + ("mdev-cdev",)])
    assert reads == 1 and by_uuid(recs, cdevs)[U[10]] == 3
    assert sum(c >= 0 for c in cdevs) == 1


def test_class_checks_both_directions():
    err = cdev_host.check_vgpu_classes([cdev_host.NV], [NVV + ("cdev",)])
    assert err and "vGPU class" in err and "vfioCdev" in err and "mdevCdev" in err
    err = cdev_host.check_vgpu_classes([cdev_host.NV + ("mdev-cdev",)], [NVV])
    assert err and "passthrough class" in err and "10de/vfio-pci" in err and "mdevCdev" in err
    assert cdev_host.check_vgpu_classes([cdev_host.NV], [NVV_CDEV]) is None
    assert cdev_host.check_vgpu_classes([cdev_host.NV_CDEV], [NVV_CDEV, INTEL]) is None
