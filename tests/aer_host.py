"""AER files for the host tests of Plugin::aerHealth (ABI v12): aer_dev_fatal / aer_dev_nonfatal written into the
existing fake sysfs trees, and the C test surface of the AER settings."""
import ctypes as C
import os

import fake_sysfs
from kxpu_b200.workloads import aer_file


def lib():
    L = fake_sysfs.host_lib()
    L.kxh_set_aer_health.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_uint64]
    L.kxh_aer_reads.restype = C.c_uint64
    L.kxh_aer_reads.argtypes = [C.c_void_p]
    L.kxh_refresh_aer_health.restype = C.c_int
    L.kxh_refresh_aer_health.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int),
                                         C.c_char_p, C.c_size_t]
    L.kxh_devs_aer.restype = C.c_int
    L.kxh_devs_aer.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    L.kxh_devs.restype = C.c_int
    L.kxh_devs.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t]
    return L


def write(entry_dir, fatal=0, nonfatal=0):
    """the two files of one function in the kernel's format, the count on the first error kind"""
    for name, total, c in (("aer_dev_fatal", "TOTAL_ERR_FATAL", fatal), ("aer_dev_nonfatal", "TOTAL_ERR_NONFATAL", nonfatal)):
        with open(os.path.join(entry_dir, name), "wb") as f:
            f.write(aer_file(total, [c] + [0] * 17))


def write_raw(entry_dir, fatal_bytes, nonfatal_bytes):
    for name, b in (("aer_dev_fatal", fatal_bytes), ("aer_dev_nonfatal", nonfatal_bytes)):
        with open(os.path.join(entry_dir, name), "wb") as f:
            f.write(b)


def enable(hp, on=True, fatal_limit=0, nonfatal_limit=0):
    lib().kxh_set_aer_health(hp.h, int(on), fatal_limit, nonfatal_limit)


def reads(hp):
    return lib().kxh_aer_reads(hp.h)


def refresh(hp):
    """refreshAerHealth: (changed plugins, passthrough pools moved, vGPU pools moved)"""
    changed, n, moved, err = (C.c_size_t * 64)(), C.c_size_t(0), C.c_int(-1), C.create_string_buffer(512)
    assert lib().kxh_refresh_aer_health(hp.h, changed, 64, C.byref(n), C.byref(moved), err, len(err)) == 0, err.value
    return list(changed[:n.value]), bool(moved.value & 1), bool(moved.value & 2)


def reasons(hp, idx):
    """{device id: AER reason} of plugin idx"""
    buf = C.create_string_buffer(1 << 16)
    assert lib().kxh_devs_aer(hp.h, idx, buf, len(buf)) >= 0
    return dict(kv.split("=", 1) for kv in buf.value.decode().split(",") if kv)


def health(hp, idx):
    """{device id: health} of plugin idx's ListAndWatch bytes (repeated Device{ID = 1, health = 2})"""
    b, out, i = hp.list_and_watch(idx), {}, 0
    while i < len(b):
        assert b[i] == 0x0A
        end = i + 2 + b[i + 1]
        j, fields = i + 2, {}
        while j < end:
            tag, ln = b[j], b[j + 1]
            fields[tag] = b[j + 2:j + 2 + ln].decode()
            j += 2 + ln
        out[fields[0x0A]] = fields.get(0x12, "")
        i = end
    return out
