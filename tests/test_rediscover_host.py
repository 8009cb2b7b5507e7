"""CPU tests of the host side of rediscovery: BindWatcher's separate mdev counter, fed by raw uevent messages."""
import ctypes as C

import fake_sysfs


def test_bind_watcher_counts_mdev_events_apart_from_pci():
    """mdev add / remove / bind / unbind move the mdev counter and never the PCI generation; pci events never move the
    mdev counter."""
    L = fake_sysfs.host_lib()
    L.kxh_uevent_feed.restype = C.c_uint64
    L.kxh_uevent_feed.argtypes = [C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.kxh_uevent_mdev_generation.restype = C.c_uint64
    L.kxh_uevent_mdev_generation.argtypes = [C.c_void_p]
    L.kxh_uevent_free.argtypes = [C.c_void_p]
    w = C.c_void_p()

    def feed(*fields):
        m = b"\0".join(fields) + b"\0"
        return L.kxh_uevent_feed(C.byref(w), m, len(m)), L.kxh_uevent_mdev_generation(w)

    uuid = b"8a6d5b2e-6f7a-4b2c-9d1e-0123456789ab"
    assert feed(b"add@/devices/pci0000:00/0000:00:02.0/" + uuid, b"ACTION=add",
                b"DEVPATH=/devices/pci0000:00/0000:00:02.0/" + uuid, b"SUBSYSTEM=mdev", b"MDEV_TYPE=nvidia-63") == (0, 1)
    assert feed(b"bind@/devices/x/" + uuid, b"ACTION=bind", b"SUBSYSTEM=mdev", b"DRIVER=vfio_mdev") == (0, 2)
    assert feed(b"change@/devices/x/" + uuid, b"ACTION=change", b"SUBSYSTEM=mdev") == (0, 2)
    assert feed(b"bind@/devices/pci0000:00/0000:00:1f.0", b"ACTION=bind", b"SUBSYSTEM=pci") == (1, 2)
    assert feed(b"unbind@/devices/x/" + uuid, b"ACTION=unbind", b"SUBSYSTEM=mdev") == (1, 3)
    assert feed(b"remove@/devices/x/" + uuid, b"SUBSYSTEM=mdev", b"ACTION=remove") == (1, 4)
    assert feed(b"add@/devices/x", b"ACTION=add", b"SUBSYSTEM=mdev_bus") == (1, 4)  # the parent registering: not an mdev
    L.kxh_uevent_free(w)


def test_atomic_spec_writer(tmp_path):
    """The rediscovery writer: rewrites only changed bytes, goes through .<name>.tmp + rename (no .tmp left behind), and
    a reader that opened the old file keeps reading the old bytes."""
    L = fake_sysfs.host_lib()
    L.kxh_write_spec_atomic.restype = C.c_int
    L.kxh_write_spec_atomic.argtypes = [C.c_char_p, C.c_char_p, C.c_size_t]
    path = tmp_path / "cdi-vfio-xxxx.yaml"
    old = b"kind: nvidia.com/gpu\ndevices: []\n"
    assert L.kxh_write_spec_atomic(str(path).encode(), old, len(old)) == 1
    assert path.read_bytes() == old
    ino = path.stat().st_ino
    assert L.kxh_write_spec_atomic(str(path).encode(), old, len(old)) == 0  # same bytes: not rewritten
    assert path.stat().st_ino == ino
    reader = open(path, "rb")
    new = b"kind: nvidia.com/gpu\ndevices:\n- name: \"0\"\n"
    assert L.kxh_write_spec_atomic(str(path).encode(), new, len(new)) == 1
    assert reader.read() == old  # the old inode, whole
    reader.close()
    assert path.read_bytes() == new and path.stat().st_ino != ino
    assert sorted(p.name for p in tmp_path.iterdir()) == ["cdi-vfio-xxxx.yaml"]
    assert L.kxh_write_spec_atomic(str(tmp_path / "missing" / "x.yaml").encode(), new, len(new)) == -1
    assert sorted(p.name for p in tmp_path.iterdir()) == ["cdi-vfio-xxxx.yaml"]
