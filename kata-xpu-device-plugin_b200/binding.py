"""ctypes binding of libkxpu.so (C ABI declared in include/kxpu.h).

Mirrors one-to-one what the cgo shim in INTEGRATION.md binds.  No torch, no numpy
compute: numpy arrays are only used as typed host buffers.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

KXPU_OK = 0
E_INVALID, E_CUDA, E_NOGPU, E_NOSPACE, E_CAPACITY, E_NCCL, E_UNSUPPORTED, E_NOMEM = -1, -2, -3, -4, -5, -6, -7, -8
ROW_MISS = -1
REJECTED = 0xFFFFFFFF
FMT_YAML, FMT_JSON = 0, 1
T_PARSE, T_FINALIZE, T_LOOKUP, T_NAMES, T_CLASSIFY, T_EMIT, T_MERGE, T_RESOLVE, T_COUNT = 0, 1, 2, 3, 4, 5, 6, 7, 8
COMM_ID_BYTES = 128

REC_VENDOR_ERR, REC_DRIVER_ERR, REC_IOMMU_ERR, REC_DEVICE_ERR, REC_IS_DIR = 1, 2, 4, 8, 16

DEVREC_DTYPE = np.dtype([("bdf", "S16"), ("vendor_txt", "u1", (8,)), ("device_txt", "u1", (8,)),
                         ("driver", "S16"), ("iommu_group", "<u4"), ("vendor_len", "u1"),
                         ("device_len", "u1"), ("flags", "u1"), ("reserved0", "u1"),
                         ("reserved1", "<u4", (2,))])
CDIDEV_DTYPE = np.dtype([("bdf", "S16"), ("iommu_group", "<u4"), ("reserved", "<u4"), ("index", "<u8")])
assert DEVREC_DTYPE.itemsize == 64 and CDIDEV_DTYPE.itemsize == 32

# every symbol include/kxpu.h declares (tests check that the library exports all of them)
ABI_SYMBOLS = [
    "kxpu_ctx_create", "kxpu_ctx_destroy", "kxpu_strerror", "kxpu_last_error", "kxpu_launch_count",
    "kxpu_last_timings", "kxpu_set_stage_timing", "kxpu_timer_begin", "kxpu_timer_end", "kxpu_dev_alloc", "kxpu_dev_free", "kxpu_dev_upload", "kxpu_dev_download",
    "kxpu_dev_replicate", "kxpu_pinned_alloc", "kxpu_pinned_free", "kxpu_sync", "kxpu_pciids_load",
    "kxpu_pciids_load_device", "kxpu_table_free", "kxpu_table_rows", "kxpu_table_export", "kxpu_lookup",
    "kxpu_lookup_device", "kxpu_pciids_join_device", "kxpu_pciids_join", "kxpu_names", "kxpu_comm_unique_id", "kxpu_comm_init", "kxpu_comm_destroy",
    "kxpu_pciids_load_sharded", "kxpu_pciids_join_sharded", "kxpu_plan_shards", "kxpu_ctx_create_multi", "kxpu_multi_destroy",
    "kxpu_multi_size", "kxpu_multi_ctx", "kxpu_multi_pciids_join", "kxpu_classify", "kxpu_cdi_emit", "kxpu_alloc_names",
    "kxpu_lw_encode", "kxpu_pciids_full_load_device", "kxpu_full_free", "kxpu_full_export", "kxpu_full_lookup",
]


class ClassifyOut(C.Structure):
    _fields_ = [("accept_index", C.c_void_p), ("group_ids", C.c_void_p), ("group_off", C.c_void_p),
                ("group_members", C.c_void_p), ("dev_ids", C.c_void_p), ("dev_off", C.c_void_p),
                ("dev_groups", C.c_void_p), ("n_accepted", C.c_uint32), ("n_groups", C.c_uint32),
                ("n_devids", C.c_uint32)]


class Shard(C.Structure):
    _fields_ = [("d_text", C.c_void_p), ("n", C.c_size_t), ("global_base", C.c_uint64), ("d_keys", C.c_void_p),
                ("nq", C.c_size_t), ("key_offset", C.c_size_t), ("d_rows_all", C.c_void_p)]


class KxpuError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("kxpu status %d: %s" % (status, msg))
        self.status = status


def lib_path():
    return os.path.join(_HERE, "lib", "libkxpu.so")


_LIB = None


def load_library():
    """dlopen lib/libkxpu.so.  Fails loudly when the CUDA library has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    p = lib_path()
    if not os.path.exists(p):
        raise KxpuError(E_NOGPU, "libkxpu.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'`" % p)
    L = C.CDLL(p)
    vp, sz, i32, u64 = C.c_void_p, C.c_size_t, C.c_int32, C.c_uint64
    sig = {
        "kxpu_ctx_create": (i32, [i32, C.POINTER(vp)]),
        "kxpu_ctx_destroy": (i32, [vp]),
        "kxpu_strerror": (C.c_char_p, [i32]),
        "kxpu_last_error": (C.c_char_p, [vp]),
        "kxpu_launch_count": (u64, [vp]),
        "kxpu_last_timings": (i32, [vp, C.POINTER(C.c_float)]),
        "kxpu_timer_begin": (i32, [vp]),
        "kxpu_timer_end": (i32, [vp, C.POINTER(C.c_float)]),
        "kxpu_dev_alloc": (i32, [vp, sz, C.POINTER(vp)]),
        "kxpu_dev_free": (i32, [vp, vp]),
        "kxpu_dev_upload": (i32, [vp, vp, vp, sz]),
        "kxpu_dev_download": (i32, [vp, vp, vp, sz]),
        "kxpu_dev_replicate": (i32, [vp, vp, vp, sz, sz]),
        "kxpu_pinned_alloc": (i32, [vp, sz, C.POINTER(vp)]),
        "kxpu_pinned_free": (i32, [vp, vp]),
        "kxpu_set_stage_timing": (i32, [vp, i32]),
        "kxpu_sync": (i32, [vp]),
        "kxpu_pciids_load": (i32, [vp, vp, sz, C.POINTER(vp)]),
        "kxpu_pciids_load_device": (i32, [vp, vp, sz, C.POINTER(vp)]),
        "kxpu_table_free": (i32, [vp, vp]),
        "kxpu_table_rows": (i32, [vp, vp, C.POINTER(C.c_uint32)]),
        "kxpu_table_export": (i32, [vp, vp, vp, vp, vp, sz, C.POINTER(C.c_uint32)]),
        "kxpu_lookup": (i32, [vp, vp, vp, sz, vp]),
        "kxpu_lookup_device": (i32, [vp, vp, vp, sz, vp]),
        "kxpu_pciids_join_device": (i32, [vp, vp, sz, vp, sz, vp, C.POINTER(vp)]),
        "kxpu_pciids_join": (i32, [vp, vp, sz, vp, sz, vp, C.POINTER(vp)]),
        "kxpu_names": (i32, [vp, vp, vp, sz, vp, sz, vp, C.POINTER(sz)]),
        "kxpu_comm_unique_id": (i32, [vp]),
        "kxpu_comm_init": (i32, [vp, i32, i32, vp]),
        "kxpu_comm_destroy": (i32, [vp]),
        "kxpu_pciids_load_sharded": (i32, [vp, vp, sz, u64, C.POINTER(vp)]),
        "kxpu_pciids_join_sharded": (i32, [vp, vp, sz, u64, vp, sz, sz, sz, vp, C.POINTER(vp)]),
        "kxpu_plan_shards": (i32, [vp, sz, i32, vp]),
        "kxpu_ctx_create_multi": (i32, [vp, i32, C.POINTER(vp)]),
        "kxpu_multi_destroy": (i32, [vp]),
        "kxpu_multi_size": (i32, [vp]),
        "kxpu_multi_ctx": (vp, [vp, i32]),
        "kxpu_multi_pciids_join": (i32, [vp, C.POINTER(Shard), sz, C.POINTER(vp)]),
        "kxpu_classify": (i32, [vp, vp, sz, C.POINTER(ClassifyOut)]),
        "kxpu_cdi_emit": (i32, [vp, i32, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_alloc_names": (i32, [vp, vp, sz, vp, sz, vp, C.POINTER(sz)]),
        "kxpu_lw_encode": (i32, [vp, vp, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_pciids_full_load_device": (i32, [vp, vp, sz, vp, C.POINTER(vp)]),
        "kxpu_full_free": (i32, [vp, vp]),
        "kxpu_full_export": (i32, [vp, vp, i32, vp, vp, sz, C.POINTER(C.c_uint32)]),
        "kxpu_full_lookup": (i32, [vp, vp, i32, vp, sz, vp]),
    }
    for name, (res, args) in sig.items():
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    _LIB = L
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data


class Table:
    def __init__(self, kx, handle):
        self.kx, self.handle = kx, handle

    @property
    def rows(self):
        n = C.c_uint32(0)
        self.kx._chk(self.kx.L.kxpu_table_rows(self.kx.ctx, self.handle, C.byref(n)))
        return n.value

    def free(self):
        if self.handle:
            self.kx._chk(self.kx.L.kxpu_table_free(self.kx.ctx, self.handle))
            self.handle = None


class Kxpu:
    """One context bound to one GPU (== one kxpu_ctx)."""

    def __init__(self, ordinal=0, _borrowed=None):
        self.L = load_library()
        self.borrowed = _borrowed is not None
        if self.borrowed:  # a context of a KxpuMulti group: destroyed with the group
            self.ctx = C.c_void_p(_borrowed)
            return
        ctx = C.c_void_p()
        rc = self.L.kxpu_ctx_create(ordinal, C.byref(ctx))
        if rc != KXPU_OK:
            raise KxpuError(rc, self.L.kxpu_strerror(rc).decode() + " (no CPU fallback exists)")
        self.ctx = ctx

    def close(self):
        if self.ctx and not self.borrowed:
            self.L.kxpu_ctx_destroy(self.ctx)
        self.ctx = None

    def _chk(self, rc):
        if rc != KXPU_OK:
            raise KxpuError(rc, "%s: %s" % (self.L.kxpu_strerror(rc).decode(), self.L.kxpu_last_error(self.ctx).decode()))

    # -- bookkeeping
    def launch_count(self):
        return int(self.L.kxpu_launch_count(self.ctx))

    def timings(self):
        t = (C.c_float * T_COUNT)()
        self._chk(self.L.kxpu_last_timings(self.ctx, t))
        return list(t)

    def sync(self):
        self._chk(self.L.kxpu_sync(self.ctx))

    def timer_begin(self):
        self._chk(self.L.kxpu_timer_begin(self.ctx))

    def timer_end(self):
        ms = C.c_float(0)
        self._chk(self.L.kxpu_timer_end(self.ctx, C.byref(ms)))
        return ms.value

    # -- memory
    def set_stage_timing(self, on):
        self._chk(self.L.kxpu_set_stage_timing(self.ctx, 1 if on else 0))

    def dev_alloc(self, nbytes):
        p = C.c_void_p()
        self._chk(self.L.kxpu_dev_alloc(self.ctx, nbytes, C.byref(p)))
        return p.value

    def dev_free(self, p):
        self._chk(self.L.kxpu_dev_free(self.ctx, p))

    def upload(self, d_dst, arr):
        arr = np.ascontiguousarray(arr)
        self._chk(self.L.kxpu_dev_upload(self.ctx, d_dst, arr.ctypes.data, arr.nbytes))

    def download(self, d_src, nbytes, dtype=np.uint8):
        out = np.empty(nbytes // np.dtype(dtype).itemsize, dtype=dtype)
        self._chk(self.L.kxpu_dev_download(self.ctx, out.ctypes.data, d_src, nbytes))
        return out

    def replicate(self, d_dst, d_src, n, copies):
        self._chk(self.L.kxpu_dev_replicate(self.ctx, d_dst, d_src, n, copies))

    def pinned(self, nbytes, dtype=np.uint8):
        """numpy view over cudaMallocHost memory (kept alive by the returned array's base)."""
        p = C.c_void_p()
        self._chk(self.L.kxpu_pinned_alloc(self.ctx, nbytes, C.byref(p)))
        buf = (C.c_uint8 * nbytes).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype)
        return arr, p.value

    def pinned_free(self, p):
        self._chk(self.L.kxpu_pinned_free(self.ctx, p))

    # -- pci.ids
    def pciids_load(self, text):
        a = np.frombuffer(text, dtype=np.uint8) if not isinstance(text, np.ndarray) else text
        h = C.c_void_p()
        self._chk(self.L.kxpu_pciids_load(self.ctx, a.ctypes.data if a.size else None, a.size, C.byref(h)))
        return Table(self, h)

    def pciids_load_device(self, d_text, n):
        h = C.c_void_p()
        self._chk(self.L.kxpu_pciids_load_device(self.ctx, d_text, n, C.byref(h)))
        return Table(self, h)

    def pciids_join_device(self, d_text, n, d_keys, nq, d_rows):
        h = C.c_void_p()
        self._chk(self.L.kxpu_pciids_join_device(self.ctx, d_text, n, d_keys, nq, d_rows, C.byref(h)))
        return Table(self, h)

    def pciids_join(self, text, keys, rows_out=None):
        """Host text + host keys -> (table, row handles): one call, one host round trip."""
        a = np.frombuffer(text, dtype=np.uint8) if not isinstance(text, np.ndarray) else text
        keys = np.ascontiguousarray(keys, dtype=np.uint32)
        rows = rows_out if rows_out is not None else np.empty(len(keys), np.int32)
        h = C.c_void_p()
        self._chk(self.L.kxpu_pciids_join(self.ctx, a.ctypes.data if a.size else None, a.size, _ptr(keys), len(keys), _ptr(rows),
                                          C.byref(h)))
        return Table(self, h), rows

    def pciids_join_call(self, text, keys, rows_out):
        """The bare kxpu_pciids_join C call with its arguments prepared once (numpy arrays that stay alive): returns
        a function that runs the call and hands back the table handle -- what a C / cgo host executes, without the
        ~7 us of numpy / ctypes argument marshalling per call."""
        fn, ctx = self.L.kxpu_pciids_join, self.ctx
        p_text, n_text = C.c_void_p(text.ctypes.data), C.c_size_t(text.size)
        p_keys, n_keys, p_rows = _ptr(keys), C.c_size_t(len(keys)), _ptr(rows_out)

        def call():
            h = C.c_void_p()
            rc = fn(ctx, p_text, n_text, p_keys, n_keys, p_rows, C.byref(h))
            if rc != 0:
                self._chk(rc)
            return h
        return call

    def table_free_handle(self, h):
        self._chk(self.L.kxpu_table_free(self.ctx, h))

    def pciids_load_sharded(self, d_text, n, global_base):
        h = C.c_void_p()
        self._chk(self.L.kxpu_pciids_load_sharded(self.ctx, d_text, n, global_base, C.byref(h)))
        return Table(self, h)

    def pciids_join_sharded(self, d_text, n, global_base, d_keys, nq, key_offset, nq_total, d_rows_all):
        h = C.c_void_p()
        self._chk(self.L.kxpu_pciids_join_sharded(self.ctx, d_text, n, global_base, d_keys, nq, key_offset, nq_total,
                                                  d_rows_all, C.byref(h)))
        return Table(self, h)

    def table_export(self, table):
        n = table.rows
        keys, offs, rows = np.empty(n, np.uint32), np.empty(n, np.uint64), np.empty(n, np.int32)
        got = C.c_uint32(0)
        self._chk(self.L.kxpu_table_export(self.ctx, table.handle, _ptr(keys), _ptr(offs), _ptr(rows), n, C.byref(got)))
        return keys, offs, rows

    def lookup(self, table, keys):
        keys = np.ascontiguousarray(keys, dtype=np.uint32)
        rows = np.empty(len(keys), np.int32)
        self._chk(self.L.kxpu_lookup(self.ctx, table.handle, _ptr(keys), len(keys), _ptr(rows)))
        return rows

    def lookup_device(self, table, d_keys, n, d_rows):
        self._chk(self.L.kxpu_lookup_device(self.ctx, table.handle, d_keys, n, d_rows))

    def names_blob(self, table, rows):
        """kxpu_names as it comes: (blob bytes, offs uint32[n+1]), name i = blob[offs[i]:offs[i+1]]."""
        rows = np.ascontiguousarray(rows, dtype=np.int32)
        offs = np.empty(len(rows) + 1, np.uint32)
        need = C.c_size_t(0)
        rc = self.L.kxpu_names(self.ctx, table.handle, _ptr(rows), len(rows), None, 0, _ptr(offs), C.byref(need))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        out = np.empty(max(need.value, 1), np.uint8)
        self._chk(self.L.kxpu_names(self.ctx, table.handle, _ptr(rows), len(rows), _ptr(out), need.value, _ptr(offs),
                                    C.byref(need)))
        return out[:need.value].tobytes(), offs

    def names(self, table, rows):
        blob, offs = self.names_blob(table, rows)
        return [blob[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)], blob, offs

    # -- the rest of the pci.ids model
    def full_load_device(self, d_text, n, table):
        h = C.c_void_p()
        self._chk(self.L.kxpu_pciids_full_load_device(self.ctx, d_text, n, table.handle, C.byref(h)))
        return h

    def full_free(self, full):
        self._chk(self.L.kxpu_full_free(self.ctx, full))

    def full_export(self, full, kind):
        n = C.c_uint32(0)
        rc = self.L.kxpu_full_export(self.ctx, full, kind, None, None, 0, C.byref(n))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        keys, offs = np.empty(n.value, np.uint64), np.empty(n.value, np.uint64)
        self._chk(self.L.kxpu_full_export(self.ctx, full, kind, _ptr(keys), _ptr(offs), n.value, C.byref(n)))
        return keys, offs

    def full_lookup(self, full, kind, keys):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.empty(len(keys), np.int64)
        self._chk(self.L.kxpu_full_lookup(self.ctx, full, kind, _ptr(keys), len(keys), _ptr(out)))
        return out

    # -- multi GPU
    def comm_unique_id(self):
        b = np.zeros(COMM_ID_BYTES, np.uint8)
        self._chk(self.L.kxpu_comm_unique_id(_ptr(b)))
        return b

    def comm_init(self, nranks, rank, uid):
        uid = np.ascontiguousarray(uid, dtype=np.uint8)
        self._chk(self.L.kxpu_comm_init(self.ctx, nranks, rank, _ptr(uid)))

    def comm_destroy(self):
        self._chk(self.L.kxpu_comm_destroy(self.ctx))

    # -- discovery
    def classify(self, recs):
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == DEVREC_DTYPE
        n = len(recs)
        arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                    group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                    dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                    dev_groups=np.empty(n, np.uint32))
        out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
        self._chk(self.L.kxpu_classify(self.ctx, _ptr(recs) if n else None, n, C.byref(out)))
        g, d, a = out.n_groups, out.n_devids, out.n_accepted
        return dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                    group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                    group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                    dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g])

    def cdi_emit(self, fmt, devs):
        devs = np.ascontiguousarray(devs)
        assert devs.dtype == CDIDEV_DTYPE
        # one call with a buffer no document can outgrow (<= 384 B per device); the two-call sizing
        # protocol (out = NULL -> *len) remains available and is exercised by the tests
        cap = 400 * len(devs) + 1024
        out = np.empty(cap, np.uint8)
        got = C.c_size_t(0)
        self._chk(self.L.kxpu_cdi_emit(self.ctx, fmt, _ptr(devs) if len(devs) else None, len(devs), _ptr(out), cap,
                                       C.byref(got)))
        return out[:got.value].tobytes()

    def cdi_emit_len(self, fmt, devs):
        """Sizing call of the two-call protocol: out = NULL, returns the required length."""
        devs = np.ascontiguousarray(devs)
        need = C.c_size_t(0)
        rc = self.L.kxpu_cdi_emit(self.ctx, fmt, _ptr(devs) if len(devs) else None, len(devs), None, 0, C.byref(need))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        return need.value

    def alloc_names(self, idx):
        idx = np.ascontiguousarray(idx, dtype=np.uint64)
        offs = np.empty(len(idx) + 1, np.uint32)
        need = C.c_size_t(0)
        cap = 36 * len(idx) + 16
        out = np.empty(cap, np.uint8)
        self._chk(self.L.kxpu_alloc_names(self.ctx, _ptr(idx), len(idx), _ptr(out), cap, _ptr(offs), C.byref(need)))
        return out[:need.value].tobytes(), offs

    def lw_encode(self, groups, healthy=None):
        groups = np.ascontiguousarray(groups, dtype=np.uint32)
        if healthy is not None:
            healthy = np.ascontiguousarray(healthy, dtype=np.uint8)
        need = C.c_size_t(0)
        rc = self.L.kxpu_lw_encode(self.ctx, _ptr(groups), _ptr(healthy), len(groups), None, 0, C.byref(need))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        out = np.empty(max(need.value, 1), np.uint8)
        got = C.c_size_t(0)
        self._chk(self.L.kxpu_lw_encode(self.ctx, _ptr(groups), _ptr(healthy), len(groups), _ptr(out), need.value,
                                        C.byref(got)))
        return out[:got.value].tobytes()


def plan_shards(text, nranks):
    """kxpu_plan_shards: [(start, end)] * nranks, cuts at top-level (vendor) line starts."""
    L = load_library()
    a = np.frombuffer(text, dtype=np.uint8) if not isinstance(text, np.ndarray) else text
    cuts = np.zeros(nranks + 1, np.uint64)
    rc = L.kxpu_plan_shards(a.ctypes.data if a.size else None, a.size, nranks, cuts.ctypes.data)
    if rc != KXPU_OK:
        raise KxpuError(rc, L.kxpu_strerror(rc).decode())
    return [(int(cuts[i]), int(cuts[i + 1])) for i in range(nranks)]


class KxpuMulti:
    """kxpu_ctx_create_multi: N contexts of ONE process (what a single Go host binds)."""

    def __init__(self, ordinals):
        self.L = load_library()
        arr = (C.c_int32 * len(ordinals))(*ordinals)
        h = C.c_void_p()
        rc = self.L.kxpu_ctx_create_multi(arr, len(ordinals), C.byref(h))
        if rc != KXPU_OK:
            raise KxpuError(rc, self.L.kxpu_strerror(rc).decode() + " (no CPU fallback exists)")
        self.handle = h
        self.ctxs = [Kxpu(_borrowed=self.L.kxpu_multi_ctx(h, i)) for i in range(len(ordinals))]

    def __len__(self):
        return int(self.L.kxpu_multi_size(self.handle))

    def pciids_join(self, shards, nq_total=0):
        """shards: one dict per rank with d_text, n, global_base and optionally d_keys, nq, key_offset, d_rows_all."""
        n = len(self.ctxs)
        arr = (Shard * n)()
        for i, s in enumerate(shards):
            arr[i] = Shard(s["d_text"], s["n"], s["global_base"], s.get("d_keys"), s.get("nq", 0), s.get("key_offset", 0),
                           s.get("d_rows_all"))
        tabs = (C.c_void_p * n)()
        rc = self.L.kxpu_multi_pciids_join(self.handle, arr, nq_total, tabs)
        if rc != KXPU_OK:
            msgs = "; ".join(self.L.kxpu_last_error(k.ctx).decode() for k in self.ctxs)
            raise KxpuError(rc, "%s: %s" % (self.L.kxpu_strerror(rc).decode(), msgs))
        return [Table(self.ctxs[i], C.c_void_p(tabs[i])) for i in range(n)]

    def close(self):
        if self.handle:
            for k in self.ctxs:
                k.ctx = None
            self.L.kxpu_multi_destroy(self.handle)
            self.handle = None
