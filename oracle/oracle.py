"""ctypes binding of the CPU oracle (oracle/kxpu_oracle.c).

TEST INFRASTRUCTURE ONLY -- imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py.  Never imported by the product
package.  PARITY UNPINNED (see kxpu_oracle.c header).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

u8p = C.POINTER(C.c_uint8)


class DevRec(C.Structure):
    _fields_ = [("bdf", C.c_char * 16), ("vendor_txt", C.c_uint8 * 8), ("device_txt", C.c_uint8 * 8),
                ("driver", C.c_char * 16), ("iommu_group", C.c_uint32), ("vendor_len", C.c_uint8),
                ("device_len", C.c_uint8), ("flags", C.c_uint8), ("reserved0", C.c_uint8),
                ("reserved1", C.c_uint32 * 2)]


DEVREC_DTYPE = np.dtype([("bdf", "S16"), ("vendor_txt", "u1", (8,)), ("device_txt", "u1", (8,)),
                         ("driver", "S16"), ("iommu_group", "<u4"), ("vendor_len", "u1"),
                         ("device_len", "u1"), ("flags", "u1"), ("reserved0", "u1"),
                         ("reserved1", "<u4", (2,))])
CDIDEV_DTYPE = np.dtype([("bdf", "S16"), ("iommu_group", "<u4"), ("reserved", "<u4"), ("index", "<u8")])
ROW_DTYPE = np.dtype([("key", "<u4"), ("pad", "<u4"), ("line_off", "<u8"), ("anchor_off", "<u8")])
assert DEVREC_DTYPE.itemsize == 64 and CDIDEV_DTYPE.itemsize == 32 and ROW_DTYPE.itemsize == 24


class ClassifyOut(C.Structure):
    _fields_ = [("accept_index", C.c_void_p), ("group_ids", C.c_void_p), ("group_off", C.c_void_p),
                ("group_members", C.c_void_p), ("dev_ids", C.c_void_p), ("dev_off", C.c_void_p),
                ("dev_groups", C.c_void_p), ("n_accepted", C.c_uint32), ("n_groups", C.c_uint32),
                ("n_devids", C.c_uint32)]


def build():
    subprocess.check_call(["make", "-s", "-C", _HERE])


def lib():
    """libkxpu_oracle.so, every oracle file in one library; make rebuilds it first if a source is newer."""
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(os.path.join(_HERE, "libkxpu_oracle.so"))
        vp, sz, s = C.c_void_p, C.c_size_t, C.c_char_p
        sig = {
            # kxpu_oracle.c
            "kxo_scan_lookup": (C.c_int64, [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t,
                                            C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]),
            "kxo_sanitise": (C.c_size_t, [C.c_char_p, C.c_size_t, C.c_void_p]),
            "kxo_device_name": (C.c_int64, [C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_size_t,
                                            C.POINTER(C.c_int64), C.POINTER(C.c_uint64)]),
            "kxo_table_build": (C.c_size_t, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
            "kxo_line_rest": (C.c_size_t, [C.c_void_p, C.c_size_t, C.c_uint64, C.POINTER(C.c_size_t)]),
            "kxo_names_bulk": (C.c_size_t, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                            C.c_void_p]),
            "kxo_classify": (C.c_int32, [C.c_void_p, C.c_size_t, C.POINTER(ClassifyOut)]),
            "kxo_is_base60": (C.c_int, [C.c_char_p, C.c_size_t]),
            "kxo_cdi_emit": (C.c_size_t, [C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
            "kxo_alloc_names": (C.c_size_t, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
            "kxo_lw_encode": (C.c_size_t, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
            "kxo_bench_scan": (C.c_double, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p,
                                            C.POINTER(C.c_uint64)]),
            "kxo_bench_parse_once": (C.c_double, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                                  C.POINTER(C.c_double)]),
            "kxo_table_build_mt": (C.c_size_t, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t]),
            "kxo_bench_parse_mt": (C.c_double, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                                C.POINTER(C.c_double)]),
            "kxo_full_build": (C.c_size_t, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t]),
            # kxpu_xpu_oracle.c
            "kxo_classify_rules": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(ClassifyOut),
                                               C.c_void_p]),
            "kxo_kind_ok": (C.c_int, [C.c_char_p]),
            "kxo_cdi_emit_kind": (C.c_size_t, [C.c_int32, C.c_char_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
            "kxo_alloc_names_kind": (C.c_size_t, [C.c_char_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                  C.c_void_p]),
            # kxpu_mdev_oracle.c
            "kxo_mdev_classify": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(ClassifyOut),
                                              C.c_void_p]),
            "kxo_type_key": (C.c_size_t, [C.c_char_p, C.c_size_t, C.c_void_p]),
            "kxo_uuid_ok": (C.c_int, [C.c_char_p]),
            "kxo_mdev_names": (C.c_size_t, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
            "kxo_cdi_emit_mdev": (C.c_size_t, [C.c_int32, C.c_char_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
            # kxpu_topo_oracle.c
            "kxo_classify_topo": (C.c_int32, [vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp]),
            "kxo_classify_mdev_topo": (C.c_int32, [vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp]),
            "kxo_lw_encode_topo": (sz, [vp, vp, vp, sz, vp, sz]),
            "kxo_preferred_allocation": (C.c_int32, [vp, sz, vp, vp, vp, vp, vp, sz, vp, vp]),
            # kxpu_viab_oracle.c
            "kxo_classify_viable": (C.c_int32, [vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp, vp]),
            # kxpu_reconcile_oracle.c
            "kxo_reconcile": (C.c_int32, [vp, sz, C.c_uint64, vp, sz, vp, vp, vp, vp]),
            # kxpu_pcie_oracle.c
            "kxo_pcie_parse": (C.c_int32, [vp, vp, vp]),
            "kxo_pcie_tree": (C.c_int32, [vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, vp]),
            "kxo_preferred_allocation_pcie": (C.c_int32, [vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, vp, sz, vp, vp]),
            # kxpu_aer_oracle.c and the DRA oracles it includes
            "kxo_dra_slices": (C.c_int32, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint64, vp, sz, vp, sz,
                                           C.POINTER(sz), vp, C.POINTER(sz), C.POINTER(C.c_int32)]),
            "kxo_dra_slices_mdev": (C.c_int32, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_uint64, vp, sz, vp, sz,
                                                C.POINTER(sz), vp, C.POINTER(sz), C.POINTER(C.c_int32)]),
            "kxo_dra_slices_taint": (C.c_int32, [s, s, s, C.c_uint64, vp, sz, s, s, s, vp, vp, sz, C.POINTER(sz), vp,
                                                 C.POINTER(sz), C.POINTER(C.c_int32)]),
            "kxo_dra_slices_mdev_taint": (C.c_int32, [s, s, s, C.c_uint64, vp, sz, s, s, s, vp, vp, sz, C.POINTER(sz),
                                                      vp, C.POINTER(sz), C.POINTER(C.c_int32)]),
            "kxo_aer_health": (C.c_int32, [vp, sz, vp, vp, sz, C.c_uint64, C.c_uint64, vp, vp, sz, vp, vp]),
            "kxo_dra_slices_taints": (C.c_int32, [s, s, s, C.c_uint64, vp, sz, vp, sz, vp, vp, sz, C.POINTER(sz), vp,
                                                  C.POINTER(sz), C.POINTER(C.c_int32)]),
            "kxo_dra_slices_mdev_taints": (C.c_int32, [s, s, s, C.c_uint64, vp, sz, vp, sz, vp, vp, sz, C.POINTER(sz),
                                                       vp, C.POINTER(sz), C.POINTER(C.c_int32)]),
        }
        for name, (res, args) in sig.items():
            f = getattr(L, name)
            f.restype, f.argtypes = res, args
        _LIB = L
    return _LIB


def _buf(b):
    """bytes / numpy -> (pointer, length, keepalive)."""
    a = np.frombuffer(b, dtype=np.uint8) if not isinstance(b, np.ndarray) else b
    return a.ctypes.data, a.size, a


def sanitise(rest: bytes) -> bytes:
    out = C.create_string_buffer(len(rest) + 1)
    m = lib().kxo_sanitise(rest, len(rest), out)
    return out.raw[:m]


def scan_lookup(text, vendor: bytes, device: bytes):
    """Literal getDeviceName: returns (line_off or -1, rest bytes or None, bytes scanned)."""
    p, n, keep = _buf(text)
    ro, rl, sc = C.c_size_t(0), C.c_size_t(0), C.c_uint64(0)
    off = lib().kxo_scan_lookup(p, n, vendor, len(vendor), device, len(device), C.byref(ro), C.byref(rl), C.byref(sc))
    if off < 0:
        return -1, None, sc.value
    return off, bytes(keep[ro.value:ro.value + rl.value]), sc.value


def device_name(text, key: int):
    """(line_off, name bytes) with name=None on a miss."""
    p, n, keep = _buf(text)
    out = C.create_string_buffer(65536)
    off = C.c_int64(0)
    l = lib().kxo_device_name(p, n, key, out, 65536, C.byref(off), None)
    return (off.value, None) if l < 0 else (off.value, out.raw[:l])


def lookup_many(text, keys):
    """Literal scan per key -> (line_off int64[n], names list[bytes|None])."""
    offs = np.empty(len(keys), dtype=np.int64)
    names = []
    for i, k in enumerate(keys):
        o, nm = device_name(text, int(k))
        offs[i] = o
        names.append(nm)
    return offs, names


def table_build(text):
    """Single-pass table: structured array (key, line_off, anchor_off) in file order."""
    p, n, keep = _buf(text)
    cap = 1 << 16
    rows = np.zeros(cap, dtype=ROW_DTYPE)
    nr = lib().kxo_table_build(p, n, rows.ctypes.data, cap)
    if nr > cap:
        rows = np.zeros(nr, dtype=ROW_DTYPE)
        nr = lib().kxo_table_build(p, n, rows.ctypes.data, nr)
    return rows[:nr]


def row_name(text, line_off: int) -> bytes:
    p, n, keep = _buf(text)
    ro = C.c_size_t(0)
    rl = lib().kxo_line_rest(p, n, line_off, C.byref(ro))
    return sanitise(bytes(keep[ro.value:ro.value + rl]))


def names_bulk(text, line_offs):
    """row_name of every line in line_offs, in one call: (blob bytes, offs uint32[count+1]) with
    name i = blob[offs[i]:offs[i+1]] -- the layout kxpu_names returns."""
    p, n, keep = _buf(text)
    lo = np.ascontiguousarray(line_offs, dtype=np.uint64)
    offs = np.empty(len(lo) + 1, np.uint32)
    # a sanitised name is never longer than its line, so the text length bounds the names of distinct lines
    cap = n
    blob = np.empty(max(cap, 1), np.uint8)
    need = lib().kxo_names_bulk(p, n, lo.ctypes.data, lo.size, blob.ctypes.data, cap, offs.ctypes.data)
    if need > cap:
        blob = np.empty(need, np.uint8)
        lib().kxo_names_bulk(p, n, lo.ctypes.data, lo.size, blob.ctypes.data, need, offs.ctypes.data)
    assert need < (1 << 32), "names of more than 4 GiB do not fit uint32 offsets"
    return blob[:need].tobytes(), offs


def classify_call(fn, head, recs, dev=(), group=()):
    """fn(*head, recs, n, &out, *dev outputs, *group outputs), the shape of every kxo_*classify* call: allocates the
    seven CSR arrays of kxpu_classify_out and the extra outputs, runs the call and returns (status, result).
    dev / group: (name, dtype) of the extra outputs with one entry per device id / per group, dtype None for a NULL
    argument.  result is classify's dict plus the extra outputs trimmed to the counts the call wrote, or None when the
    status is not 0."""
    n = len(recs)
    recs = np.ascontiguousarray(recs)
    arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                dev_groups=np.empty(n, np.uint32))
    out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
    extra = [(name, None if dt is None else np.empty(max(n, 1), dt), per)
             for per, outs in (("dev", dev), ("group", group)) for name, dt in outs]
    rc = fn(*head, recs.ctypes.data, n, C.byref(out), *[None if e is None else e.ctypes.data for _, e, _ in extra])
    if rc != 0:
        return rc, None
    g, d, a = out.n_groups, out.n_devids, out.n_accepted
    res = dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
               group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
               group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
               dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g])
    res.update((name, arr[:d if per == "dev" else g]) for name, arr, per in extra if arr is not None)
    return rc, res


def classify(recs: np.ndarray):
    rc, res = classify_call(lib().kxo_classify, (), recs)
    assert rc == 0
    return res


def cdi_emit(fmt: int, devs: np.ndarray) -> bytes:
    devs = np.ascontiguousarray(devs)
    need = lib().kxo_cdi_emit(fmt, devs.ctypes.data, len(devs), None, 0)
    out = np.empty(need, np.uint8)
    got = lib().kxo_cdi_emit(fmt, devs.ctypes.data, len(devs), out.ctypes.data, need)
    assert got == need
    return out.tobytes()


def alloc_names(idx: np.ndarray):
    idx = np.ascontiguousarray(idx, dtype=np.uint64)
    offs = np.empty(len(idx) + 1, np.uint32)
    cap = 36 * len(idx) + 1
    out = np.empty(cap, np.uint8)
    need = lib().kxo_alloc_names(idx.ctypes.data, len(idx), out.ctypes.data, cap, offs.ctypes.data)
    return out[:need].tobytes(), offs


def lw_encode(groups: np.ndarray, healthy=None) -> bytes:
    groups = np.ascontiguousarray(groups, dtype=np.uint32)
    hp = None
    if healthy is not None:
        healthy = np.ascontiguousarray(healthy, dtype=np.uint8)
        hp = healthy.ctypes.data
    need = lib().kxo_lw_encode(groups.ctypes.data, hp, len(groups), None, 0)
    out = np.empty(need, np.uint8)
    lib().kxo_lw_encode(groups.ctypes.data, hp, len(groups), out.ctypes.data, need)
    return out.tobytes()


def is_base60(s: bytes) -> bool:
    return bool(lib().kxo_is_base60(s, len(s)))


def bench_scan(text, keys, threads):
    """Reference algorithm timed: returns (seconds, bytes_scanned, line_off[])."""
    p, n, keep = _buf(text)
    keys = np.ascontiguousarray(keys, dtype=np.uint32)
    offs = np.empty(len(keys), np.int64)
    sc = C.c_uint64(0)
    dt = lib().kxo_bench_scan(p, n, keys.ctypes.data, len(keys), threads, offs.ctypes.data, C.byref(sc))
    return dt, sc.value, offs


def bench_parse_once(text, keys):
    p, n, keep = _buf(text)
    keys = np.ascontiguousarray(keys, dtype=np.uint32)
    offs = np.empty(len(keys), np.int64)
    ps = C.c_double(0)
    dt = lib().kxo_bench_parse_once(p, n, keys.ctypes.data, len(keys), offs.ctypes.data, C.byref(ps))
    return dt, ps.value, offs


def table_build_mt(text, threads):
    """kxo_table_build on `threads` host threads (shards cut at vendor lines, first anchors merged)."""
    p, n, keep = _buf(text)
    cap = 1 << 16
    rows = np.zeros(cap, dtype=ROW_DTYPE)
    nr = lib().kxo_table_build_mt(p, n, threads, rows.ctypes.data, cap)
    if nr > cap:
        rows = np.zeros(nr, dtype=ROW_DTYPE)
        nr = lib().kxo_table_build_mt(p, n, threads, rows.ctypes.data, nr)
    return rows[:nr]


def bench_parse_mt(text, keys, threads):
    """(total seconds, parse seconds, line_off[]) of the all-threads single-pass CPU path."""
    p, n, keep = _buf(text)
    keys = np.ascontiguousarray(keys, dtype=np.uint32)
    offs = np.empty(len(keys), np.int64)
    ps = C.c_double(0)
    dt = lib().kxo_bench_parse_mt(p, n, threads, keys.ctypes.data, len(keys), offs.ctypes.data, C.byref(ps))
    return dt, ps.value, offs


ROW64_DTYPE = np.dtype([("key", "<u8"), ("line_off", "<u8")])


def full_build(text, kind):
    """SURVEY 8(f) row 4: vendor (0) / subsystem (1) / class-section (2) rows (key, line_off) in file order."""
    L = lib()
    p, n, keep = _buf(text)
    cap = 1 << 15
    rows = np.zeros(cap, dtype=ROW64_DTYPE)
    nr = L.kxo_full_build(p, n, kind, rows.ctypes.data, cap)
    if nr > cap:
        rows = np.zeros(nr, dtype=ROW64_DTYPE)
        nr = L.kxo_full_build(p, n, kind, rows.ctypes.data, nr)
    return rows[:nr]
