"""ctypes binding of libkxpu.so (C ABI declared in include/kxpu.h).

Mirrors one-to-one what the cgo shim in INTEGRATION.md binds.  No torch, no numpy
compute: numpy arrays are only used as typed host buffers.
"""
import ctypes as C
import os
import re

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

KXPU_OK = 0
E_INVALID, E_CUDA, E_NOGPU, E_NOSPACE, E_CAPACITY, E_NCCL, E_UNSUPPORTED, E_NOMEM = -1, -2, -3, -4, -5, -6, -7, -8
ROW_MISS = -1
REJECTED = 0xFFFFFFFF
FMT_YAML, FMT_JSON = 0, 1
T_PARSE, T_FINALIZE, T_LOOKUP, T_NAMES, T_CLASSIFY, T_EMIT, T_MERGE, T_RESOLVE, T_COUNT = 0, 1, 2, 3, 4, 5, 6, 7, 8
COMM_ID_BYTES = 128

REC_VENDOR_ERR, REC_DRIVER_ERR, REC_IOMMU_ERR, REC_DEVICE_ERR, REC_IS_DIR, REC_NAME_ERR = 1, 2, 4, 8, 16, 32
REC_NUMA = 64  # the record's numa_node byte is valid (ABI v5)
MAX_NUMA_NODES = 64
REC_BLOCKS = 0x80  # bound to a driver outside the viability list; iommu_group holds its group (ABI v8)
VIABLE = 0xFFFFFFFF  # kxpu_classify_viable: the group has no blocker
# The numa_node byte of kxpu_devrec / kxpu_mdevrec (ABI v5) keeps its pre-v5 numpy field name "reserved0": the
# dtypes below must stay equal to the checkers' (oracle/*.py), which compare dtypes field name by field name.
NUMA_FIELD = "reserved0"

DEVREC_DTYPE = np.dtype([("bdf", "S16"), ("vendor_txt", "u1", (8,)), ("device_txt", "u1", (8,)),
                         ("driver", "S16"), ("iommu_group", "<u4"), ("vendor_len", "u1"),
                         ("device_len", "u1"), ("flags", "u1"), ("reserved0", "u1"),
                         ("reserved1", "<u4", (2,))])
CDIDEV_DTYPE = np.dtype([("bdf", "S16"), ("iommu_group", "<u4"), ("reserved", "<u4"), ("index", "<u8")])
# kxpu_cdidev.vfio_cdev (ABI v14: N of /dev/vfio/devices/vfio<N>) keeps its pre-v14 numpy field name, as NUMA_FIELD does
CDEV_FIELD = "reserved"
RULE_DTYPE = np.dtype([("vendor", "S8"), ("driver", "S16"), ("reserved", "<u4", (2,))])  # kxpu_xpu_rule
assert DEVREC_DTYPE.itemsize == 64 and CDIDEV_DTYPE.itemsize == 32 and RULE_DTYPE.itemsize == 32
MAX_RULES = 16
# kxpu_mdevrec / kxpu_mdevcdi (vGPUs on the mdev bus)
MDEVREC_DTYPE = np.dtype([("uuid", "S36"), ("parent", "S16"), ("parent_vendor_txt", "u1", (8,)), ("driver", "S16"),
                          ("type_name", "u1", (40,)), ("iommu_group", "<u4"), ("vendor_len", "u1"), ("name_len", "u1"),
                          ("flags", "u1"), ("reserved0", "u1"), ("reserved1", "<u4")])
MDEVCDI_DTYPE = np.dtype([("uuid", "S36"), ("iommu_group", "<u4"), ("parent", "S16"), ("index", "<u8")])
assert MDEVREC_DTYPE.itemsize == 128 and MDEVCDI_DTYPE.itemsize == 64
# kxpu_mdevcdev: a vGPU of a class served through VFIO cdevs (an addition to ABI v14)
MDEVCDEV_DTYPE = np.dtype([("dev", MDEVCDI_DTYPE), ("vfio_cdev", "<u4"), ("reserved", "<u4", (3,))])
assert MDEVCDEV_DTYPE.itemsize == 80 and MDEVCDEV_DTYPE.fields["vfio_cdev"][1] == 64
# kxpu_vfvgpucdi: a served VF of a class that serves vGPUs on SR-IOV VFs, with its type (an addition to ABI v14)
VFVGPUCDI_DTYPE = np.dtype([("dev", CDIDEV_DTYPE), ("type_id", "<u4"), ("key_len", "u1"), ("reserved", "u1", (3,)),
                            ("key", "S40")])
assert VFVGPUCDI_DTYPE.itemsize == 80 and VFVGPUCDI_DTYPE.fields["key"][1] == 40
# kxpu_snaprec / kxpu_reconcile_counts (runtime rediscovery, ABI v6)
SNAPREC_DTYPE = np.dtype([("key", "S40"), ("iommu_group", "<u4"), ("klass", "<u4"), ("tag", "<u8"), ("index", "<u8")])
RC_COUNTS_DTYPE = np.dtype([("n_kept", "<u8"), ("n_new", "<u8"), ("n_changed", "<u8"), ("n_retired", "<u8"),
                            ("next_index_out", "<u8")])
assert SNAPREC_DTYPE.itemsize == 64 and RC_COUNTS_DTYPE.itemsize == 40
RC_KEPT, RC_NEW, RC_CHANGED, RC_RETIRED = 0, 1, 2, 3
# kxpu_pcipath (PCIe topology, ABI v7): one per kxpu_devrec, at the same index
PCIPATH_DTYPE = np.dtype([("path", "S120"), ("len", "u1"), ("reserved", "u1", (7,))])
assert PCIPATH_DTYPE.itemsize == 128
PCIE_MAX_DEPTH = 8
PCIE_NO_NODE = 0xFFFFFFFF
# kxpu_dradev (DRA ResourceSlices, ABI v9): one published device
DRADEV_DTYPE = np.dtype([("product", "u1", (64,)), ("bdf", "S16"), ("pcie_root", "S16"), ("vendor", "S8"), ("device", "S8"),
                         ("numa_mask", "<u8"), ("iommu_group", "<u4"), ("product_len", "u1"), ("reserved", "u1", (3,))])
assert DRADEV_DTYPE.itemsize == 128
# kxpu_dramdev (DRA ResourceSlices of vGPUs, ABI v10): one published vGPU
DRAMDEV_DTYPE = np.dtype([("product", "u1", (64,)), ("mdev_type", "S40"), ("uuid", "S36"), ("iommu_group", "<u4"),
                          ("parent", "S16"), ("pcie_root", "S16"), ("vendor", "S8"), ("device", "S8"), ("numa_mask", "<u8"),
                          ("product_len", "u1"), ("reserved", "u1", (7,))])
assert DRAMDEV_DTYPE.itemsize == 208
# kxpu_dravfvgpu (DRA ResourceSlices of vGPUs on SR-IOV VFs, an addition to ABI v14): one published vGPU
DRAVFVGPU_DTYPE = np.dtype([("product", "u1", (64,)), ("type_key", "S40"), ("bdf", "S16"), ("parent", "S16"),
                            ("pcie_root", "S16"), ("vendor", "S8"), ("device", "S8"), ("numa_mask", "<u8"),
                            ("iommu_group", "<u4"), ("type_id", "<u4"), ("product_len", "u1"), ("reserved", "u1", (7,))])
assert DRAVFVGPU_DTYPE.itemsize == 192
# kxpu_dramdevpf (DRA ResourceSlices of mdev vGPUs with their parent's PF, an addition to ABI v14): one published vGPU
DRAMDEVPF_DTYPE = np.dtype([("dev", DRAMDEV_DTYPE), ("physfn", "S16"), ("physfn_device", "S8"), ("reserved", "u1", (8,))])
assert DRAMDEVPF_DTYPE.itemsize == 240
# kxpu_dradevpf (DRA ResourceSlices of passthrough devices with their PF, an addition to ABI v14): one published device
DRADEVPF_DTYPE = np.dtype([("dev", DRADEV_DTYPE), ("physfn", "S16"), ("physfn_device", "S8"), ("reserved", "u1", (8,))])
assert DRADEVPF_DTYPE.itemsize == 160
# kxpu_dradevpcie (DRA ResourceSlices with PCIe root ports and switches, an addition to ABI v14): one published device
DRADEVPCIE_DTYPE = np.dtype([("pf", DRADEVPF_DTYPE), ("root_port", "u8"), ("pcie_switch", "u8")])
assert DRADEVPCIE_DTYPE.itemsize == 176
PCIE_NO_KEY = 0xFFFFFFFFFFFFFFFF
# kxpu_dramdevpcie / kxpu_dravfvgpupcie (vGPU DRA ResourceSlices with PCIe root ports and switches, additions to ABI v14)
DRAMDEVPCIE_DTYPE = np.dtype([("pf", DRAMDEVPF_DTYPE), ("root_port", "u8"), ("pcie_switch", "u8")])
assert DRAMDEVPCIE_DTYPE.itemsize == 256
DRAVFVGPUPCIE_DTYPE = np.dtype([("dev", DRAVFVGPU_DTYPE), ("root_port", "u8"), ("pcie_switch", "u8")])
assert DRAVFVGPUPCIE_DTYPE.itemsize == 208
DRA_SLICE_DEVICES = 128
DRA_MAX_DEVICES = 1 << 24
DRA_TAINT_SLICE_DEVICES = 64  # devices per slice of the _taint calls (ABI v11) when taint_since is given
DRA_TAINT_SINCE_MAX = 253402300799  # 9999-12-31T23:59:59Z
DRA_MAX_TAINTS = 4  # entries of the _taints calls' table (ABI v12)
AER_FATAL, AER_NONFATAL, AER_UNKNOWN = 1, 2, 4  # kxpu_aer_health's group bits
AER_FILE_MAX = 4096
AER_UNKNOWN_COUNT = (1 << 64) - 1  # totals of an unknown count
# kxpu_sriovrec (SR-IOV virtual functions, an addition to ABI v14): one per kxpu_devrec, at the same index
SRIOVREC_DTYPE = np.dtype([("physfn", "S16"), ("numvfs_txt", "u1", (8,)), ("numvfs_len", "u1"), ("flags", "u1"),
                           ("reserved", "u1", (6,))])
assert SRIOVREC_DTYPE.itemsize == 32
SR_PHYSFN_ERR, SR_NUMVFS_ERR = 1, 2
NO_PF = 0xFFFFFFFF
# vGPUs on SR-IOV VFs (additions to ABI v14): kxpu_vfvgpurec, one per kxpu_devrec at the same index, and the 48-byte key
# rows of kxpu_vf_vgpu_types / kxpu_classify_vf_vgpu
VFVGPUREC_DTYPE = np.dtype([("cur_txt", "u1", (16,)), ("cur_len", "u1"), ("flags", "u1"), ("reserved", "u1", (14,))])
assert VFVGPUREC_DTYPE.itemsize == 32
VGPUKEY_DTYPE = np.dtype([("key", "u1", (40,)), ("zero", "u1", (7,)), ("len", "u1")])
assert VGPUKEY_DTYPE.itemsize == 48
# kxpu_name_entry: one entry of kxpu_classify_named's name table
NAME_DTYPE = np.dtype([("rule", "<u4"), ("slot", "<u4"), ("device", "S8")])
assert NAME_DTYPE.itemsize == 16
MAX_NAMES = 64
NO_SLOT = 0xFFFFFFFF
VT_READ, VT_CUR_ERR = 1, 2
VT_NONE, VT_NAMED, VT_UNNAMED, VT_BAD = 0, 1, 2, 3
VD_SAME, VD_CLEARED, VD_CHANGED, VD_BAD = 0, 1, 2, 3  # kxpu_vf_vgpu_drift's per-record status
VD_STEADY = 0xFFFFFFFF  # kxpu_vf_vgpu_drift's group_first of a group with no drifted member
# kxpu_resetrec (resets between tenants, an addition to ABI v14): one per kxpu_devrec, at the same index
RESET_FILE_MAX = 64
RESETREC_DTYPE = np.dtype([("txt", "u1", (RESET_FILE_MAX,)), ("len", "u1"), ("flags", "u1"), ("reserved", "u1", (14,))])
assert RESETREC_DTYPE.itemsize == 80
RS_ABSENT, RS_READ_ERR, RS_LEGACY = 1, 2, 4
# method bits, in the order of RESET_METHODS
RESET_METHODS = ("flr", "af_flr", "pm", "bus", "cxl_bus", "device_specific", "acpi")
RM_ALL, RM_UNNAMED = 0x7F, 0x80
RESET_SET_OK, RESET_NO_PATH, RESET_ROOT_BUS = 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD
# kxpu_metricdev / kxpu_metricreason (Prometheus metrics, an addition to ABI v14)
METRICDEV_DTYPE = np.dtype([("resource_off", "<u8"), ("address_off", "<u8"), ("resource_len", "<u4"), ("address_len", "<u4"),
                            ("group", "<u4"), ("healthy", "<u4"), ("aer_fatal", "<u8"), ("aer_nonfatal", "<u8"),
                            ("reason_off", "<u8"), ("reason_count", "<u4"), ("reserved", "<u4")])
assert METRICDEV_DTYPE.itemsize == 64
METRICREASON_DTYPE = np.dtype([("kind", "<u4"), ("detail_len", "<u4"), ("detail_off", "<u8")])
assert METRICREASON_DTYPE.itemsize == 16
METRICS_NO_VALUE = 0xFFFFFFFFFFFFFFFF
METRICS_STRING_MAX = 4096


def _header_macros():
    """The string macros of include/kxpu.h the metrics document is made of: {name: bytes}, adjacent literals joined."""
    text = open(os.path.join(os.path.dirname(_HERE), "include", "kxpu.h")).read().replace("\\\n", " ")
    out = {}
    for m in re.finditer(r'^#define (KXPU_METRICS_\w+)\s+((?:"(?:[^"\\]|\\.)*"\s*)+)$', text, re.M):
        lits = re.findall(r'"((?:[^"\\]|\\.)*)"', m.group(2))
        out[m.group(1)] = "".join(lits).encode().decode("unicode_escape").encode()
    return out


_MACROS = _header_macros()
METRICS_REASONS = tuple(_MACROS["KXPU_METRICS_REASONS"].decode().split(","))  # kind k = METRICS_REASONS[k]
METRICS_HEADS = tuple(_MACROS["KXPU_METRICS_%s_HEAD" % f] for f in ("HEALTHY", "REASON", "AER", "READS", "VALIDATIONS"))
CDI_FRAG_MIN = 166  # the shortest device fragment of a CDI spec: len // CDI_FRAG_MIN records hold any document (ABI v13)


class DraTaint(C.Structure):
    """kxpu_dra_taint: one entry of the _taints calls' table"""
    _fields_ = [("key", C.c_char_p), ("value", C.c_char_p), ("effect", C.c_char_p)]

# every symbol include/kxpu.h declares (tests check that the library exports all of them)
ABI_SYMBOLS = [
    "kxpu_ctx_create", "kxpu_ctx_destroy", "kxpu_strerror", "kxpu_last_error", "kxpu_launch_count",
    "kxpu_last_timings", "kxpu_set_stage_timing", "kxpu_timer_begin", "kxpu_timer_end", "kxpu_dev_alloc", "kxpu_dev_free", "kxpu_dev_upload", "kxpu_dev_download",
    "kxpu_dev_replicate", "kxpu_pinned_alloc", "kxpu_pinned_free", "kxpu_sync", "kxpu_pciids_load",
    "kxpu_pciids_load_device", "kxpu_table_free", "kxpu_table_rows", "kxpu_table_export", "kxpu_lookup",
    "kxpu_lookup_device", "kxpu_pciids_join_device", "kxpu_pciids_join", "kxpu_names", "kxpu_comm_unique_id", "kxpu_comm_init", "kxpu_comm_destroy",
    "kxpu_pciids_load_sharded", "kxpu_pciids_join_sharded", "kxpu_plan_shards", "kxpu_ctx_create_multi", "kxpu_multi_destroy",
    "kxpu_multi_size", "kxpu_multi_ctx", "kxpu_multi_pciids_join", "kxpu_classify", "kxpu_cdi_emit", "kxpu_alloc_names",
    "kxpu_lw_encode", "kxpu_classify_rules", "kxpu_cdi_emit_kind", "kxpu_alloc_names_kind",
    "kxpu_classify_mdev", "kxpu_mdev_names", "kxpu_cdi_emit_mdev",
    "kxpu_pciids_full_load_device", "kxpu_full_free", "kxpu_full_export", "kxpu_full_lookup",
    "kxpu_classify_topo", "kxpu_classify_mdev_topo", "kxpu_lw_encode_topo", "kxpu_preferred_allocation",
    "kxpu_reconcile", "kxpu_pcie_tree", "kxpu_preferred_allocation_pcie", "kxpu_classify_viable",
    "kxpu_dra_slices", "kxpu_dra_slices_mdev", "kxpu_dra_slices_taint", "kxpu_dra_slices_mdev_taint",
    "kxpu_aer_health", "kxpu_dra_slices_taints", "kxpu_dra_slices_mdev_taints", "kxpu_cdi_parse", "kxpu_cdi_parse_mdev",
    "kxpu_cdi_emit_cdev", "kxpu_cdi_parse_cdev", "kxpu_cdi_emit_mdev_cdev", "kxpu_cdi_parse_mdev_cdev",
    "kxpu_sriov", "kxpu_pcie_tree_sriov", "kxpu_vf_vgpu_types", "kxpu_classify_vf_vgpu", "kxpu_pcie_tree_mdev",
    "kxpu_cdi_emit_vf_vgpu", "kxpu_cdi_emit_vf_vgpu_cdev", "kxpu_cdi_parse_vf_vgpu", "kxpu_cdi_parse_vf_vgpu_cdev",
    "kxpu_dra_slices_vf_vgpu", "kxpu_vf_vgpu_drift", "kxpu_reset_check", "kxpu_metrics_devices",
    "kxpu_mdev_pf", "kxpu_dra_slices_mdev_pf", "kxpu_classify_named", "kxpu_dra_slices_pf",
    "kxpu_pcie_ports", "kxpu_dra_slices_pcie",
    "kxpu_pcie_ports_mdev", "kxpu_dra_slices_mdev_pcie", "kxpu_dra_slices_vf_vgpu_pcie",
    "kxpu_aer_ports", "kxpu_aer_ports_mdev",
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
        "kxpu_classify_rules": (i32, [vp, vp, sz, vp, sz, C.POINTER(ClassifyOut), vp]),
        "kxpu_cdi_emit_kind": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_alloc_names_kind": (i32, [vp, C.c_char_p, vp, sz, vp, sz, vp, C.POINTER(sz)]),
        "kxpu_lw_encode": (i32, [vp, vp, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_classify_mdev": (i32, [vp, vp, sz, vp, sz, C.POINTER(ClassifyOut), vp]),
        "kxpu_mdev_names": (i32, [vp, vp, sz, vp, sz, vp, sz, vp, C.POINTER(sz)]),
        "kxpu_cdi_emit_mdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_pciids_full_load_device": (i32, [vp, vp, sz, vp, C.POINTER(vp)]),
        "kxpu_full_free": (i32, [vp, vp]),
        "kxpu_full_export": (i32, [vp, vp, i32, vp, vp, sz, C.POINTER(C.c_uint32)]),
        "kxpu_full_lookup": (i32, [vp, vp, i32, vp, sz, vp]),
        "kxpu_classify_topo": (i32, [vp, vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp]),
        "kxpu_classify_mdev_topo": (i32, [vp, vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp]),
        "kxpu_lw_encode_topo": (i32, [vp, vp, vp, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_preferred_allocation": (i32, [vp, vp, sz, vp, vp, vp, vp, vp, sz, vp, vp]),
        "kxpu_reconcile": (i32, [vp, vp, sz, u64, vp, sz, vp, vp, vp, vp]),
        "kxpu_pcie_tree": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, C.POINTER(C.c_uint32)]),
        "kxpu_preferred_allocation_pcie": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, vp, sz, vp, vp]),
        "kxpu_classify_viable": (i32, [vp, vp, sz, vp, sz, C.POINTER(ClassifyOut), vp, vp, vp]),
        "kxpu_dra_slices": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, vp, sz, C.POINTER(sz), vp,
                                  C.POINTER(sz)]),
        "kxpu_dra_slices_mdev": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, vp, sz, C.POINTER(sz), vp,
                                       C.POINTER(sz)]),
        "kxpu_dra_slices_taint": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, C.c_char_p, C.c_char_p,
                                        C.c_char_p, vp, vp, sz, C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_dra_slices_mdev_taint": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, C.c_char_p, C.c_char_p,
                                             C.c_char_p, vp, vp, sz, C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_aer_health": (i32, [vp, vp, sz, vp, vp, sz, u64, u64, vp, vp, sz, vp, vp]),
        "kxpu_cdi_parse": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_parse_mdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_emit_cdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_parse_cdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_emit_mdev_cdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_parse_mdev_cdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_emit_vf_vgpu": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_emit_vf_vgpu_cdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_parse_vf_vgpu": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_cdi_parse_vf_vgpu_cdev": (i32, [vp, i32, C.c_char_p, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_sriov": (i32, [vp, vp, sz, vp, vp, sz, vp, vp, vp, sz, vp, vp, vp]),
        "kxpu_vf_vgpu_types": (i32, [vp, vp, sz, vp, vp, sz, vp, vp, vp]),
        "kxpu_vf_vgpu_drift": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp, vp]),
        "kxpu_reset_check": (i32, [vp, vp, sz, vp, vp, vp, sz, C.c_uint32, vp, vp, sz, vp, vp, vp]),
        "kxpu_metrics_devices": (i32, [vp, vp, sz, vp, sz, vp, sz, vp, sz, C.POINTER(sz)]),
        "kxpu_classify_vf_vgpu": (i32, [vp, vp, sz, C.c_uint32, vp, sz, vp, C.POINTER(ClassifyOut), vp, vp, vp]),
        "kxpu_classify_named": (i32, [vp, vp, sz, C.c_uint32, vp, sz, vp, vp, sz, C.POINTER(ClassifyOut), vp, vp, vp, vp]),
        "kxpu_pcie_tree_sriov": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, C.POINTER(C.c_uint32), vp]),
        "kxpu_pcie_tree_mdev": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp, vp, vp, C.POINTER(C.c_uint32)]),
        "kxpu_dra_slices_taints": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, vp, sz, vp, vp, sz,
                                         C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_dra_slices_mdev_taints": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, vp, sz, vp, vp, sz,
                                              C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_dra_slices_vf_vgpu": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, vp, sz, vp, vp, sz,
                                          C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_mdev_pf": (i32, [vp, vp, sz, vp, vp, sz, vp]),
        "kxpu_dra_slices_pf": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, vp, sz, vp, vp, sz,
                                     C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_pcie_ports": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp]),
        "kxpu_dra_slices_pcie": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, C.c_char_p, vp, sz, vp, sz, vp, vp,
                                       sz, C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_pcie_ports_mdev": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp]),
        "kxpu_aer_ports": (i32, [vp, vp, vp, sz, vp, vp, vp, C.POINTER(C.c_uint32)]),
        "kxpu_aer_ports_mdev": (i32, [vp, vp, vp, sz, vp, vp, vp, C.POINTER(C.c_uint32)]),
        "kxpu_dra_slices_mdev_pcie": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, C.c_char_p, vp, sz, vp, sz, vp,
                                            vp, sz, C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_dra_slices_vf_vgpu_pcie": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, C.c_char_p, vp, sz, vp, sz,
                                               vp, vp, sz, C.POINTER(sz), vp, C.POINTER(sz)]),
        "kxpu_dra_slices_mdev_pf": (i32, [vp, C.c_char_p, C.c_char_p, C.c_char_p, u64, vp, sz, vp, sz, vp, vp, sz,
                                          C.POINTER(sz), vp, C.POINTER(sz)]),
    }
    for name, (res, args) in sig.items():
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    _LIB = L
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data


def _kind(kind):
    return kind.encode() if isinstance(kind, str) else kind


def vgpu_tables(tables):
    """(blob uint8, table_off uint64) of kxpu_vf_vgpu_types from a list of table texts, or a (blob, table_off) pair
    passed through."""
    if isinstance(tables, tuple):
        blob, toff = tables
        return np.frombuffer(bytes(blob), np.uint8), np.ascontiguousarray(toff, dtype=np.uint64)
    toff = np.zeros(len(tables) + 1, np.uint64)
    toff[1:] = np.cumsum([len(t) for t in tables]) if tables else []
    return np.frombuffer(b"".join(tables), np.uint8), toff


def rules_array(rules):
    """[(vendor, driver)] (bytes or str) -> RULE_DTYPE array for kxpu_classify_rules; an array passes through."""
    if isinstance(rules, np.ndarray):
        assert rules.dtype == RULE_DTYPE
        return np.ascontiguousarray(rules)
    a = np.zeros(len(rules), RULE_DTYPE)
    for i, (v, d) in enumerate(rules):
        a[i]["vendor"], a[i]["driver"] = _kind(v), _kind(d)
    return a


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

    def classify_rules(self, rules, recs):
        """kxpu_classify_rules: rules is a RULE_DTYPE array or [(vendor bytes, driver bytes)]; classify's dict plus
        dev_rule (rule index of every device-map entry)."""
        ra = rules_array(rules)
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == DEVREC_DTYPE
        n = len(recs)
        arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                    group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                    dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                    dev_groups=np.empty(n, np.uint32))
        dev_rule = np.empty(max(n, 1), np.uint8)
        out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
        self._chk(self.L.kxpu_classify_rules(self.ctx, _ptr(ra) if len(ra) else None, len(ra), _ptr(recs) if n else None, n,
                                             C.byref(out), _ptr(dev_rule)))
        g, d, a = out.n_groups, out.n_devids, out.n_accepted
        return dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                    group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                    group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                    dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d])

    def classify_mdev(self, rules, recs):
        """kxpu_classify_mdev over MDEVREC_DTYPE records: classify_rules' dict, except that dev_ids[d] is the index
        of the first candidate record carrying entry d's type key."""
        ra = rules_array(rules)
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == MDEVREC_DTYPE
        n = len(recs)
        arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                    group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                    dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                    dev_groups=np.empty(n, np.uint32))
        dev_rule = np.empty(max(n, 1), np.uint8)
        out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
        self._chk(self.L.kxpu_classify_mdev(self.ctx, _ptr(ra) if len(ra) else None, len(ra), _ptr(recs) if n else None, n,
                                            C.byref(out), _ptr(dev_rule)))
        g, d, a = out.n_groups, out.n_devids, out.n_accepted
        return dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                    group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                    group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                    dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d])

    def classify_topo(self, rules, recs, mdev=False):
        """kxpu_classify_topo (DEVREC_DTYPE records) or kxpu_classify_mdev_topo (mdev=True, MDEVREC_DTYPE): the dict of
        classify_rules / classify_mdev plus group_numa, the NUMA mask of every group ordinal."""
        ra = rules_array(rules)
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == (MDEVREC_DTYPE if mdev else DEVREC_DTYPE)
        n = len(recs)
        arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                    group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                    dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                    dev_groups=np.empty(n, np.uint32))
        dev_rule = np.empty(max(n, 1), np.uint8)
        gnuma = np.empty(max(n, 1), np.uint64)
        out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
        fn = self.L.kxpu_classify_mdev_topo if mdev else self.L.kxpu_classify_topo
        self._chk(fn(self.ctx, _ptr(ra) if len(ra) else None, len(ra), _ptr(recs) if n else None, n, C.byref(out),
                     _ptr(dev_rule), _ptr(gnuma)))
        g, d, a = out.n_groups, out.n_devids, out.n_accepted
        return dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                    group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                    group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                    dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d],
                    group_numa=gnuma[:g])

    def classify_viable(self, rules, recs, topo=False):
        """kxpu_classify_viable (DEVREC_DTYPE records): the dict of classify_rules (topo=False) or classify_topo
        (topo=True) plus group_blocker, the first blocking record of every group ordinal or VIABLE."""
        ra = rules_array(rules)
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == DEVREC_DTYPE
        n = len(recs)
        arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                    group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                    dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                    dev_groups=np.empty(n, np.uint32))
        dev_rule = np.empty(max(n, 1), np.uint8)
        gnuma = np.empty(max(n, 1), np.uint64) if topo else None
        gblk = np.empty(max(n, 1), np.uint32)
        out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
        self._chk(self.L.kxpu_classify_viable(self.ctx, _ptr(ra) if len(ra) else None, len(ra), _ptr(recs) if n else None,
                                              n, C.byref(out), _ptr(dev_rule), _ptr(gnuma), _ptr(gblk)))
        g, d, a = out.n_groups, out.n_devids, out.n_accepted
        res = dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                   group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                   group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                   dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d],
                   group_blocker=gblk[:g])
        if topo:
            res["group_numa"] = gnuma[:g]
        return res

    def lw_encode_topo(self, groups, healthy=None, masks=None):
        """kxpu_lw_encode_topo: ListAndWatchResponse bytes with Device.topology from the NUMA masks."""
        groups = np.ascontiguousarray(groups, dtype=np.uint32)
        if healthy is not None:
            healthy = np.ascontiguousarray(healthy, dtype=np.uint8)
        if masks is not None:
            masks = np.ascontiguousarray(masks, dtype=np.uint64)
        need = C.c_size_t(0)
        rc = self.L.kxpu_lw_encode_topo(self.ctx, _ptr(groups), _ptr(healthy), _ptr(masks), len(groups), None, 0, C.byref(need))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        out = np.empty(max(need.value, 1), np.uint8)
        got = C.c_size_t(0)
        self._chk(self.L.kxpu_lw_encode_topo(self.ctx, _ptr(groups), _ptr(healthy), _ptr(masks), len(groups), _ptr(out),
                                             need.value, C.byref(got)))
        return out[:got.value].tobytes()

    def preferred_allocation(self, dev_numa, requests):
        """kxpu_preferred_allocation.  requests: [(available positions, must-include positions, size)]; returns one
        position list per request."""
        a = pref_requests(requests)
        out = np.empty(max(int(a["size"].sum()), 1), np.uint32)
        out_off = np.empty(len(requests) + 1, np.uint32)
        self.preferred_allocation_raw(dev_numa, a, out, out_off)
        return [out[out_off[q]:out_off[q + 1]].tolist() for q in range(len(requests))]

    def preferred_allocation_raw(self, dev_numa, a, out, out_off):
        """The bare call on a pref_requests() dict and caller buffers (timing loops)."""
        dev_numa = np.ascontiguousarray(dev_numa, dtype=np.uint64)
        self._chk(self.L.kxpu_preferred_allocation(self.ctx, _ptr(dev_numa) if len(dev_numa) else None, len(dev_numa),
                                                   _ptr(a["avail_off"]), _ptr(a["avail"]), _ptr(a["must_off"]),
                                                   _ptr(a["must"]), _ptr(a["size"]), len(a["size"]), _ptr(out),
                                                   _ptr(out_off)))

    def vf_vgpu_types(self, recs_vt, tables):
        """kxpu_vf_vgpu_types: recs_vt (VFVGPUREC_DTYPE) and the name tables in priority order (a list of bytes, or a
        (blob, table_off) pair).  Returns dict(keys (VGPUKEY_DTYPE), type_id, status)."""
        recs_vt = np.ascontiguousarray(recs_vt)
        assert recs_vt.dtype == VFVGPUREC_DTYPE
        blob, toff = vgpu_tables(tables)
        n = len(recs_vt)
        keys, tid, st = np.zeros(max(n, 1), VGPUKEY_DTYPE), np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint8)
        self._chk(self.L.kxpu_vf_vgpu_types(self.ctx, _ptr(recs_vt) if n else None, n, _ptr(blob) if len(blob) else None,
                                            _ptr(toff), len(toff) - 1, _ptr(keys), _ptr(tid), _ptr(st)))
        return dict(keys=keys[:n], type_id=tid[:n], status=st[:n])

    def vf_vgpu_drift(self, recs_vt, type_was, group_off, group_members):
        """kxpu_vf_vgpu_drift: recs_vt (VFVGPUREC_DTYPE) re-read, type_was the walk's type IDs, group_off [G+1] /
        group_members the groups.  Returns dict(type_now, status_now (VD_*), group_first (VD_STEADY: none drifted))."""
        recs_vt = np.ascontiguousarray(recs_vt)
        assert recs_vt.dtype == VFVGPUREC_DTYPE
        was = np.ascontiguousarray(type_was, dtype=np.uint32)
        goff = np.ascontiguousarray(group_off, dtype=np.uint32)
        gmem = np.ascontiguousarray(group_members, dtype=np.uint32)
        n, G = len(recs_vt), len(goff) - 1
        assert len(was) == n
        now, st, first = np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint8), np.zeros(max(G, 1), np.uint32)
        self._chk(self.L.kxpu_vf_vgpu_drift(self.ctx, _ptr(recs_vt) if n else None, _ptr(was) if n else None, n, _ptr(goff),
                                            _ptr(gmem) if len(gmem) else None, G, _ptr(now), _ptr(st), _ptr(first)))
        return dict(type_now=now[:n], status_now=st[:n], group_first=first[:G])

    def reset_check(self, rules, recs, paths, rrs, allow, group_off, group_members):
        """kxpu_reset_check: recs (DEVREC_DTYPE), paths (PCIPATH_DTYPE) and rrs (RESETREC_DTYPE) at the same indices, the
        rules and group CSR of a classify call, allow a mask of method bits.  Returns dict(methods, set_verdict,
        group_reset (VIABLE: every member can be reset))."""
        ra = rules_array(rules)
        recs, paths, rrs = np.ascontiguousarray(recs), np.ascontiguousarray(paths), np.ascontiguousarray(rrs)
        assert recs.dtype == DEVREC_DTYPE and paths.dtype == PCIPATH_DTYPE and rrs.dtype == RESETREC_DTYPE
        assert len(recs) == len(paths) == len(rrs)
        goff = np.ascontiguousarray(group_off, dtype=np.uint32)
        gmem = np.ascontiguousarray(group_members, dtype=np.uint32)
        n, G = len(recs), len(goff) - 1
        meth, sv, gr = np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.uint32), np.zeros(max(G, 1), np.uint32)
        self._chk(self.L.kxpu_reset_check(self.ctx, _ptr(ra) if len(ra) else None, len(ra), _ptr(recs) if n else None,
                                          _ptr(paths) if n else None, _ptr(rrs) if n else None, n, allow, _ptr(goff),
                                          _ptr(gmem) if len(gmem) else None, G, _ptr(meth), _ptr(sv), _ptr(gr)))
        return dict(methods=meth[:n], set_verdict=sv[:n], group_reset=gr[:G])

    def metrics_devices_raw(self, devs, strings, reasons, out, cap):
        """The bare kxpu_metrics_devices call: (status, *len).  out: a uint8 array or None."""
        devs, reasons = np.ascontiguousarray(devs), np.ascontiguousarray(reasons)
        assert devs.dtype == METRICDEV_DTYPE and reasons.dtype == METRICREASON_DTYPE
        sb = np.frombuffer(bytes(strings), np.uint8)
        n = C.c_size_t(0)
        rc = self.L.kxpu_metrics_devices(self.ctx, _ptr(devs) if len(devs) else None, len(devs), _ptr(sb) if len(sb) else None,
                                         len(sb), _ptr(reasons) if len(reasons) else None, len(reasons), _ptr(out), cap,
                                         C.byref(n))
        return rc, n.value

    def metrics_devices(self, devs, strings, reasons):
        """kxpu_metrics_devices: families 1 to 3 of the Prometheus text of devs (METRICDEV_DTYPE) and reasons
        (METRICREASON_DTYPE), their strings in `strings` (bytes).  Sizes with a first call, writes with a second."""
        rc, need = self.metrics_devices_raw(devs, strings, reasons, None, 0)
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        out = np.empty(max(need, 1), np.uint8)
        rc, got = self.metrics_devices_raw(devs, strings, reasons, out, need)
        self._chk(rc)
        return out[:got].tobytes()

    def classify_vf_vgpu(self, rules, vgpu_rules, recs, keys, topo=False, viable=False):
        """kxpu_classify_vf_vgpu: the dict of classify_rules, plus group_numa (topo) and group_blocker (viable).  keys:
        VGPUKEY_DTYPE rows, one per record (None: NULL)."""
        ra = rules_array(rules)
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == DEVREC_DTYPE
        if keys is not None:
            keys = np.ascontiguousarray(keys)
            assert keys.dtype == VGPUKEY_DTYPE and len(keys) == len(recs)
        n = len(recs)
        arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                    group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                    dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                    dev_groups=np.empty(n, np.uint32))
        dev_rule = np.empty(max(n, 1), np.uint8)
        gnuma = np.empty(max(n, 1), np.uint64) if topo else None
        gblk = np.empty(max(n, 1), np.uint32) if viable else None
        out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
        self._chk(self.L.kxpu_classify_vf_vgpu(self.ctx, _ptr(ra) if len(ra) else None, len(ra), vgpu_rules,
                                               _ptr(recs) if n else None, n,
                                               None if keys is None else _ptr(keys if n else np.zeros(1, VGPUKEY_DTYPE)),
                                               C.byref(out),
                                               _ptr(dev_rule), _ptr(gnuma), _ptr(gblk)))
        g, d, a = out.n_groups, out.n_devids, out.n_accepted
        res = dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                   group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                   group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                   dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d])
        if topo:
            res["group_numa"] = gnuma[:g]
        if viable:
            res["group_blocker"] = gblk[:g]
        return res

    def classify_named(self, rules, vgpu_rules, recs, keys, names, topo=False, viable=False):
        """kxpu_classify_named: classify_vf_vgpu's dict plus dev_slot.  names: a NAME_DTYPE array or
        [(rule, device bytes, slot)]; an empty table passes NULL and leaves dev_slot absent from the dict."""
        if not isinstance(names, np.ndarray):
            names = np.array([(r, s, d) for r, d, s in names], NAME_DTYPE)
        names = np.ascontiguousarray(names)
        assert names.dtype == NAME_DTYPE
        ra = rules_array(rules)
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == DEVREC_DTYPE
        if keys is not None:
            keys = np.ascontiguousarray(keys)
            assert keys.dtype == VGPUKEY_DTYPE and len(keys) == len(recs)
        n = len(recs)
        arrs = dict(accept_index=np.empty(n, np.uint32), group_ids=np.empty(n, np.uint32),
                    group_off=np.empty(n + 1, np.uint32), group_members=np.empty(n, np.uint32),
                    dev_ids=np.empty(n, np.uint64), dev_off=np.empty(n + 1, np.uint32),
                    dev_groups=np.empty(n, np.uint32))
        dev_rule = np.empty(max(n, 1), np.uint8)
        dev_slot = np.empty(max(n, 1), np.uint32)
        gnuma = np.empty(max(n, 1), np.uint64) if topo else None
        gblk = np.empty(max(n, 1), np.uint32) if viable else None
        out = ClassifyOut(**{k: v.ctypes.data for k, v in arrs.items()})
        self._chk(self.L.kxpu_classify_named(self.ctx, _ptr(ra) if len(ra) else None, len(ra), vgpu_rules,
                                             _ptr(recs) if n else None, n,
                                             None if keys is None else _ptr(keys if n else np.zeros(1, VGPUKEY_DTYPE)),
                                             _ptr(names) if len(names) else None, len(names), C.byref(out),
                                             _ptr(dev_rule), _ptr(dev_slot) if len(names) else None, _ptr(gnuma), _ptr(gblk)))
        g, d, a = out.n_groups, out.n_devids, out.n_accepted
        res = dict(accept_index=arrs["accept_index"], n_accepted=a, n_groups=g, n_devids=d,
                   group_ids=arrs["group_ids"][:g], group_off=arrs["group_off"][:g + 1],
                   group_members=arrs["group_members"][:a], dev_ids=arrs["dev_ids"][:d],
                   dev_off=arrs["dev_off"][:d + 1], dev_groups=arrs["dev_groups"][:g], dev_rule=dev_rule[:d])
        if len(names):
            res["dev_slot"] = dev_slot[:d]
        if topo:
            res["group_numa"] = gnuma[:g]
        if viable:
            res["group_blocker"] = gblk[:g]
        return res

    def sriov(self, rules, recs, srs, group_ids, group_off, group_members):
        """kxpu_sriov: recs (DEVREC_DTYPE) and srs (SRIOVREC_DTYPE) at the same indices, the rules and group CSR of a
        classify call.  Returns dict(pf_of, numvfs, group_sriov)."""
        ra = rules_array(rules)
        recs, srs = np.ascontiguousarray(recs), np.ascontiguousarray(srs)
        assert recs.dtype == DEVREC_DTYPE and srs.dtype == SRIOVREC_DTYPE and len(recs) == len(srs)
        group_ids = np.ascontiguousarray(group_ids, dtype=np.uint32)
        group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
        group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
        n, G = len(recs), len(group_off) - 1
        pf_of, numvfs = np.empty(max(n, 1), np.uint32), np.empty(max(n, 1), np.uint32)
        gs = np.empty(max(G, 1), np.uint32)
        self._chk(self.L.kxpu_sriov(self.ctx, _ptr(ra) if len(ra) else None, len(ra), _ptr(recs) if n else None,
                                    _ptr(srs) if n else None, n, _ptr(group_ids) if len(group_ids) else None, _ptr(group_off),
                                    _ptr(group_members) if len(group_members) else None, G, _ptr(pf_of), _ptr(numvfs),
                                    _ptr(gs)))
        return dict(pf_of=pf_of[:n], numvfs=numvfs[:n], group_sriov=gs[:G])

    def mdev_pf(self, recs, mrecs, msrs):
        """kxpu_mdev_pf: recs (DEVREC_DTYPE) of a PCI walk, mrecs (MDEVREC_DTYPE) and msrs (SRIOVREC_DTYPE, physfn only)
        of an mdev walk at the same indices.  Returns pf_of, one PCI-record index or NO_PF per mdev."""
        recs, mrecs, msrs = np.ascontiguousarray(recs), np.ascontiguousarray(mrecs), np.ascontiguousarray(msrs)
        assert recs.dtype == DEVREC_DTYPE and mrecs.dtype == MDEVREC_DTYPE and msrs.dtype == SRIOVREC_DTYPE
        assert len(mrecs) == len(msrs)
        m = len(mrecs)
        pf_of = np.empty(max(m, 1), np.uint32)
        self.mdev_pf_raw(recs, mrecs, msrs, pf_of)
        return pf_of[:m]

    def mdev_pf_raw(self, recs, mrecs, msrs, pf_of):
        """The bare call into a caller buffer (timing loops, untouched-output checks)."""
        n, m = len(recs), len(mrecs)
        self._chk(self.L.kxpu_mdev_pf(self.ctx, _ptr(recs) if n else None, n, _ptr(mrecs) if m else None,
                                      _ptr(msrs) if m else None, m, _ptr(pf_of) if m else None))

    def pcie_tree(self, recs, paths, group_off, group_members, pf_of=None):
        """kxpu_pcie_tree: recs (DEVREC_DTYPE) and paths (PCIPATH_DTYPE) at the same indices, the group CSR of a classify
        call.  Returns dict(group_node, key, parent, depth), the forest trimmed to its node count.  With pf_of (kxpu_sriov's,
        one per record): kxpu_pcie_tree_sriov."""
        recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths)
        assert recs.dtype == DEVREC_DTYPE and paths.dtype == PCIPATH_DTYPE and len(recs) == len(paths)
        group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
        group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
        G = len(group_off) - 1
        cap = max(PCIE_MAX_DEPTH * G, 1)
        gnode = np.empty(max(G, 1), np.uint32)
        key, parent, depth = np.empty(cap, np.uint64), np.empty(cap, np.uint32), np.empty(cap, np.uint8)
        nn = C.c_uint32(0)
        n = len(recs)
        args = (self.ctx, _ptr(recs) if n else None, _ptr(paths) if n else None, n, _ptr(group_off),
                _ptr(group_members) if len(group_members) else None, G, _ptr(gnode), _ptr(key), _ptr(parent), _ptr(depth),
                C.byref(nn))
        if pf_of is None:
            self._chk(self.L.kxpu_pcie_tree(*args))
        else:
            pf_of = np.ascontiguousarray(pf_of, dtype=np.uint32)
            assert len(pf_of) == n
            self._chk(self.L.kxpu_pcie_tree_sriov(*args, _ptr(pf_of) if n else None))
        m = nn.value
        return dict(group_node=gnode[:G], key=key[:m], parent=parent[:m], depth=depth[:m])

    def pcie_ports(self, recs, paths, group_off, group_members):
        """kxpu_pcie_ports: pcie_tree's inputs; returns (root_port, pcie_switch), one function key per group or
        PCIE_NO_KEY."""
        recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths)
        assert recs.dtype == DEVREC_DTYPE and paths.dtype == PCIPATH_DTYPE and len(recs) == len(paths)
        group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
        group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
        G = len(group_off) - 1
        rp, sw = np.empty(max(G, 1), np.uint64), np.empty(max(G, 1), np.uint64)
        self.pcie_ports_raw(recs, paths, group_off, group_members, rp, sw)
        return rp[:G], sw[:G]

    def pcie_ports_raw(self, recs, paths, group_off, group_members, root_port, pcie_switch):
        """The bare call into caller buffers (timing loops, untouched-output checks); group_off is taken as given."""
        n = len(recs)
        self._chk(self.L.kxpu_pcie_ports(self.ctx, _ptr(recs) if n else None, _ptr(paths) if n else None, n,
                                         _ptr(group_off), _ptr(group_members) if len(group_members) else None,
                                         len(group_off) - 1, _ptr(root_port), _ptr(pcie_switch)))

    def pcie_ports_mdev(self, recs, paths, group_off, group_members):
        """kxpu_pcie_ports_mdev: pcie_tree_mdev's inputs; returns (root_port, pcie_switch), one function key per group
        or PCIE_NO_KEY."""
        recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths)
        assert recs.dtype == MDEVREC_DTYPE and paths.dtype == PCIPATH_DTYPE and len(recs) == len(paths)
        group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
        group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
        G = len(group_off) - 1
        rp, sw = np.empty(max(G, 1), np.uint64), np.empty(max(G, 1), np.uint64)
        self.pcie_ports_mdev_raw(recs, paths, group_off, group_members, rp, sw)
        return rp[:G], sw[:G]

    def pcie_ports_mdev_raw(self, recs, paths, group_off, group_members, root_port, pcie_switch):
        """The bare call into caller buffers (timing loops, untouched-output checks); group_off is taken as given."""
        n = len(recs)
        self._chk(self.L.kxpu_pcie_ports_mdev(self.ctx, _ptr(recs) if n else None, _ptr(paths) if n else None, n,
                                              _ptr(group_off), _ptr(group_members) if len(group_members) else None,
                                              len(group_off) - 1, _ptr(root_port), _ptr(pcie_switch)))

    def aer_ports(self, recs, paths):
        """kxpu_aer_ports (recs DEVREC_DTYPE) or kxpu_aer_ports_mdev (recs MDEVREC_DTYPE), paths PCIPATH_DTYPE at the same
        indices.  Returns (port_off, port_of, port_key): the ports of record i are port_of[port_off[i]:port_off[i+1]],
        nearest first, and port_key[p] is the function key of port p."""
        recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths)
        assert recs.dtype in (DEVREC_DTYPE, MDEVREC_DTYPE) and paths.dtype == PCIPATH_DTYPE and len(recs) == len(paths)
        n = len(recs)
        cap = max(PCIE_MAX_DEPTH * n, 1)
        off, of, key = np.empty(n + 1, np.uint32), np.empty(cap, np.uint32), np.empty(cap, np.uint64)
        nk = C.c_uint32(0)
        self.aer_ports_raw(recs, paths, off, of, key, C.byref(nk))
        return off, of[:off[n]], key[:nk.value]

    def aer_ports_raw(self, recs, paths, port_off, port_of, port_key, n_ports, n=None, mdev=None):
        """The bare call into caller buffers (timing loops, untouched-output checks); n defaults to len(recs), mdev to
        whether recs are MDEVREC_DTYPE, and a None array is passed as NULL."""
        n = len(recs) if n is None else n
        mdev = recs is not None and recs.dtype == MDEVREC_DTYPE if mdev is None else mdev
        f = self.L.kxpu_aer_ports_mdev if mdev else self.L.kxpu_aer_ports
        self._chk(f(self.ctx, _ptr(recs), _ptr(paths), n, _ptr(port_off), _ptr(port_of), _ptr(port_key), n_ports))

    def pcie_tree_mdev(self, recs, paths, group_off, group_members):
        """kxpu_pcie_tree_mdev: recs (MDEVREC_DTYPE) and paths (PCIPATH_DTYPE, the entries' links) at the same indices,
        the group CSR of an mdev classify call.  Returns pcie_tree's dict."""
        recs, paths = np.ascontiguousarray(recs), np.ascontiguousarray(paths)
        assert recs.dtype == MDEVREC_DTYPE and paths.dtype == PCIPATH_DTYPE and len(recs) == len(paths)
        group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
        group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
        G = len(group_off) - 1
        cap = max(PCIE_MAX_DEPTH * G, 1)
        gnode = np.empty(max(G, 1), np.uint32)
        key, parent, depth = np.empty(cap, np.uint64), np.empty(cap, np.uint32), np.empty(cap, np.uint8)
        nn = C.c_uint32(0)
        n = len(recs)
        self._chk(self.L.kxpu_pcie_tree_mdev(self.ctx, _ptr(recs) if n else None, _ptr(paths) if n else None, n,
                                             _ptr(group_off), _ptr(group_members) if len(group_members) else None, G,
                                             _ptr(gnode), _ptr(key), _ptr(parent), _ptr(depth), C.byref(nn)))
        m = nn.value
        return dict(group_node=gnode[:G], key=key[:m], parent=parent[:m], depth=depth[:m])

    def preferred_allocation_pcie(self, dev_numa, dev_node, parent, depth, requests):
        """kxpu_preferred_allocation_pcie: kxpu_preferred_allocation's requests and answers, with each device's PCIe
        node (dev_node, None: no PCIe information) and the forest (parent, depth)."""
        a = pref_requests(requests)
        out = np.empty(max(int(a["size"].sum()), 1), np.uint32)
        out_off = np.empty(len(requests) + 1, np.uint32)
        self.preferred_allocation_pcie_raw(dev_numa, dev_node, parent, depth, a, out, out_off)
        return [out[out_off[q]:out_off[q + 1]].tolist() for q in range(len(requests))]

    def preferred_allocation_pcie_raw(self, dev_numa, dev_node, parent, depth, a, out, out_off):
        """The bare call on a pref_requests() dict and caller buffers (timing loops, untouched-output checks)."""
        dev_numa = np.ascontiguousarray(dev_numa, dtype=np.uint64)
        if dev_node is not None:
            dev_node = np.ascontiguousarray(dev_node, dtype=np.uint32)
            assert len(dev_node) == len(dev_numa)
        parent = np.ascontiguousarray(parent, dtype=np.uint32)
        depth = np.ascontiguousarray(depth, dtype=np.uint8)
        n = len(dev_numa)
        self._chk(self.L.kxpu_preferred_allocation_pcie(
            self.ctx, _ptr(dev_numa) if n else None, _ptr(dev_node) if dev_node is not None and n else None, n,
            _ptr(parent) if len(parent) else None, _ptr(depth) if len(depth) else None, len(parent),
            _ptr(a["avail_off"]), _ptr(a["avail"]), _ptr(a["must_off"]), _ptr(a["must"]), _ptr(a["size"]),
            len(a["size"]), _ptr(out), _ptr(out_off)))

    def reconcile(self, prev, cur, next_index):
        """kxpu_reconcile: prev / cur are SNAPREC_DTYPE arrays.  Returns dict(index, cur_state, prev_state, counts),
        counts a dict of the five kxpu_reconcile_counts fields."""
        prev, cur = np.ascontiguousarray(prev), np.ascontiguousarray(cur)
        assert prev.dtype == SNAPREC_DTYPE and cur.dtype == SNAPREC_DTYPE
        out = reconcile_outputs(len(prev), len(cur))
        self.reconcile_raw(prev, cur, next_index, out)
        return reconcile_result(out)

    def reconcile_raw(self, prev, cur, next_index, out):
        """The bare call into the buffers of reconcile_outputs() (timing loops, untouched-output checks)."""
        self._chk(self.L.kxpu_reconcile(self.ctx, _ptr(prev) if len(prev) else None, len(prev), next_index,
                                        _ptr(cur) if len(cur) else None, len(cur), _ptr(out["index"]),
                                        _ptr(out["cur_state"]), _ptr(out["prev_state"]), _ptr(out["counts"])))

    def mdev_names(self, recs, idx):
        """kxpu_mdev_names: (blob, offsets) of the type keys of recs[idx], with the two-call sizing."""
        recs = np.ascontiguousarray(recs)
        assert recs.dtype == MDEVREC_DTYPE
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        offs = np.empty(len(idx) + 1, np.uint32)
        need = C.c_size_t(0)
        rp = _ptr(recs) if len(recs) else None
        rc = self.L.kxpu_mdev_names(self.ctx, rp, len(recs), _ptr(idx), len(idx), None, 0, _ptr(offs), C.byref(need))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        out = np.empty(max(need.value, 1), np.uint8)
        self._chk(self.L.kxpu_mdev_names(self.ctx, rp, len(recs), _ptr(idx), len(idx), _ptr(out), need.value, _ptr(offs),
                                         C.byref(need)))
        return out[:need.value].tobytes(), offs

    def cdi_emit_mdev(self, fmt, devs, kind):
        """kxpu_cdi_emit_mdev: the CDI spec of a vGPU class (MDEVCDI_DTYPE devices, kind bytes or str)."""
        return self._emit_sized(self.L.kxpu_cdi_emit_mdev, MDEVCDI_DTYPE, fmt, devs, kind)

    def cdi_emit_cdev(self, fmt, devs, kind):
        """kxpu_cdi_emit_cdev: the CDI spec of a passthrough class whose functions are reached through their VFIO cdevs
        (CDIDEV_DTYPE devices, N of /dev/vfio/devices/vfio<N> in the CDEV_FIELD field; kind bytes or str)."""
        return self._emit_sized(self.L.kxpu_cdi_emit_cdev, CDIDEV_DTYPE, fmt, devs, kind)

    def cdi_emit_mdev_cdev(self, fmt, devs, kind):
        """kxpu_cdi_emit_mdev_cdev: the CDI spec of a vGPU class whose mdevs are reached through their VFIO cdevs
        (MDEVCDEV_DTYPE devices; kind bytes or str)."""
        return self._emit_sized(self.L.kxpu_cdi_emit_mdev_cdev, MDEVCDEV_DTYPE, fmt, devs, kind)

    def cdi_emit_vf_vgpu(self, fmt, devs, kind, cdev=False):
        """kxpu_cdi_emit_vf_vgpu (cdev: kxpu_cdi_emit_vf_vgpu_cdev): the CDI spec of a class that serves vGPUs on SR-IOV
        VFs, with each VF's type ID and key (VFVGPUCDI_DTYPE devices; kind bytes or str)."""
        fn = self.L.kxpu_cdi_emit_vf_vgpu_cdev if cdev else self.L.kxpu_cdi_emit_vf_vgpu
        return self._emit_sized(fn, VFVGPUCDI_DTYPE, fmt, devs, kind)

    def _emit_sized(self, fn, dtype, fmt, devs, kind):
        """the two-call sizing protocol: out = NULL gives the length, the second call writes the document"""
        devs = np.ascontiguousarray(devs)
        assert devs.dtype == dtype
        kb = _kind(kind)
        need = C.c_size_t(0)
        dp = _ptr(devs) if len(devs) else None
        rc = fn(self.ctx, fmt, kb, dp, len(devs), None, 0, C.byref(need))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        out = np.empty(max(need.value, 1), np.uint8)
        got = C.c_size_t(0)
        self._chk(fn(self.ctx, fmt, kb, dp, len(devs), _ptr(out), need.value, C.byref(got)))
        return out[:got.value].tobytes()

    def dra_slices(self, driver, pool, node, generation, devs):
        """kxpu_dra_slices: (bytes, slice_off) of the ResourceSlices of one pool (DRADEV_DTYPE devices), with the two-call
        sizing.  Slice s is the JSON object bytes[slice_off[s]:slice_off[s + 1] - 1], each followed by '\\n'."""
        return self._slices(self.L.kxpu_dra_slices, DRADEV_DTYPE, driver, pool, node, generation, devs)

    def dra_slices_mdev(self, driver, pool, node, generation, devs):
        """kxpu_dra_slices_mdev: the same for a pool of vGPUs (DRAMDEV_DTYPE devices)."""
        return self._slices(self.L.kxpu_dra_slices_mdev, DRAMDEV_DTYPE, driver, pool, node, generation, devs)

    def dra_slices_taint(self, driver, pool, node, generation, devs, key, value, effect, since):
        """kxpu_dra_slices_taint: dra_slices with at most one taint per device.  since: None (the untainted call's bytes)
        or one int64 per device, the taint's unix time (< 0: untainted); 64 devices per slice when given."""
        return self._slices(self.L.kxpu_dra_slices_taint, DRADEV_DTYPE, driver, pool, node, generation, devs,
                            (key, value, effect, since))

    def dra_slices_mdev_taint(self, driver, pool, node, generation, devs, key, value, effect, since):
        """kxpu_dra_slices_mdev_taint: the same for a pool of vGPUs (DRAMDEV_DTYPE devices)."""
        return self._slices(self.L.kxpu_dra_slices_mdev_taint, DRAMDEV_DTYPE, driver, pool, node, generation, devs,
                            (key, value, effect, since))

    def dra_slices_taints(self, driver, pool, node, generation, devs, taints, since):
        """kxpu_dra_slices_taints: dra_slices with a table of taints.  taints: a list of (key, value, effect); since: None
        (the untainted call's bytes) or an int64 [n, len(taints)] array, since[i, t] < 0 when device i does not carry
        taint t; 64 devices per slice when given."""
        return self._slices(self.L.kxpu_dra_slices_taints, DRADEV_DTYPE, driver, pool, node, generation, devs,
                            taints=(taints, since))

    def dra_slices_mdev_taints(self, driver, pool, node, generation, devs, taints, since):
        """kxpu_dra_slices_mdev_taints: the same for a pool of vGPUs (DRAMDEV_DTYPE devices)."""
        return self._slices(self.L.kxpu_dra_slices_mdev_taints, DRAMDEV_DTYPE, driver, pool, node, generation, devs,
                            taints=(taints, since))

    def dra_slices_vf_vgpu(self, driver, pool, node, generation, devs, taints, since):
        """kxpu_dra_slices_vf_vgpu: the same for a pool of vGPUs on SR-IOV VFs (DRAVFVGPU_DTYPE devices); since None gives
        the untainted bytes."""
        return self._slices(self.L.kxpu_dra_slices_vf_vgpu, DRAVFVGPU_DTYPE, driver, pool, node, generation, devs,
                            taints=(taints, since))

    def dra_slices_mdev_pf(self, driver, pool, node, generation, devs, taints, since):
        """kxpu_dra_slices_mdev_pf: the same for a pool of vGPUs with their parent's PF (DRAMDEVPF_DTYPE devices); since
        None gives the untainted bytes."""
        return self._slices(self.L.kxpu_dra_slices_mdev_pf, DRAMDEVPF_DTYPE, driver, pool, node, generation, devs,
                            taints=(taints, since))

    def dra_slices_pf(self, driver, pool, node, generation, devs, taints, since):
        """kxpu_dra_slices_pf: the same for a pool of passthrough devices with their PF (DRADEVPF_DTYPE devices); since
        None gives the untainted bytes."""
        return self._slices(self.L.kxpu_dra_slices_pf, DRADEVPF_DTYPE, driver, pool, node, generation, devs,
                            taints=(taints, since))

    def dra_slices_pcie(self, driver, pool, node, generation, attr_domain, devs, taints, since):
        """kxpu_dra_slices_pcie: the same for a pool of passthrough devices with their PF and PCIe ports
        (DRADEVPCIE_DTYPE devices), the two port attributes qualified by attr_domain; since None gives the untainted
        bytes."""
        dom = _kind(attr_domain)

        def fn(ctx, d, p, nd, g, *rest):
            return self.L.kxpu_dra_slices_pcie(ctx, d, p, nd, g, dom, *rest)
        return self._slices(fn, DRADEVPCIE_DTYPE, driver, pool, node, generation, devs, taints=(taints, since))

    def dra_slices_mdev_pcie(self, driver, pool, node, generation, attr_domain, devs, taints, since):
        """kxpu_dra_slices_mdev_pcie: the same for a pool of mdev vGPUs with their parent's PF and PCIe ports
        (DRAMDEVPCIE_DTYPE devices), the two port attributes qualified by attr_domain; since None gives the untainted
        bytes."""
        return self._slices(self._ports_fn(self.L.kxpu_dra_slices_mdev_pcie, attr_domain), DRAMDEVPCIE_DTYPE, driver,
                            pool, node, generation, devs, taints=(taints, since))

    def dra_slices_vf_vgpu_pcie(self, driver, pool, node, generation, attr_domain, devs, taints, since):
        """kxpu_dra_slices_vf_vgpu_pcie: the same for a pool of vGPUs on VFs with their PCIe ports
        (DRAVFVGPUPCIE_DTYPE devices)."""
        return self._slices(self._ports_fn(self.L.kxpu_dra_slices_vf_vgpu_pcie, attr_domain), DRAVFVGPUPCIE_DTYPE, driver,
                            pool, node, generation, devs, taints=(taints, since))

    def dra_slices_mdev_pcie_raw(self, driver, pool, node, generation, attr_domain, devs, taints, since, out, length,
                                 slice_off):
        """The bare kxpu_dra_slices_mdev_pcie call into caller buffers (refusal checks): returns the status code, no
        exception; length is a ctypes size_t, out / slice_off numpy arrays or None."""
        return self._slices_raw(self.L.kxpu_dra_slices_mdev_pcie, DRAMDEVPCIE_DTYPE, driver, pool, node, generation,
                                attr_domain, devs, taints, since, out, length, slice_off)

    def dra_slices_vf_vgpu_pcie_raw(self, driver, pool, node, generation, attr_domain, devs, taints, since, out, length,
                                    slice_off):
        """The bare kxpu_dra_slices_vf_vgpu_pcie call, as dra_slices_mdev_pcie_raw."""
        return self._slices_raw(self.L.kxpu_dra_slices_vf_vgpu_pcie, DRAVFVGPUPCIE_DTYPE, driver, pool, node, generation,
                                attr_domain, devs, taints, since, out, length, slice_off)

    @staticmethod
    def _ports_fn(call, attr_domain):
        """a slice call of the PCIe layouts with its attr_domain bound, in _slices' argument order"""
        dom = _kind(attr_domain)

        def fn(ctx, d, p, nd, g, *rest):
            return call(ctx, d, p, nd, g, dom, *rest)
        return fn

    def _slices_raw(self, call, dtype, driver, pool, node, generation, attr_domain, devs, taints, since, out, length,
                    slice_off):
        devs = np.ascontiguousarray(devs)
        assert devs.dtype == dtype
        tab = (DraTaint * max(len(taints), 1))(*[DraTaint(_kind(k), _kind(v), _kind(e)) for k, v, e in taints])
        if since is not None:
            since = np.ascontiguousarray(since, dtype=np.int64)
        ns = C.c_size_t(0)
        return call(self.ctx, _kind(driver), _kind(pool), _kind(node), generation, _kind(attr_domain),
                    _ptr(devs) if len(devs) else None, len(devs), C.cast(tab, C.c_void_p), len(taints),
                    None if since is None else _ptr(since), None if out is None else _ptr(out),
                    0 if out is None else len(out), C.byref(length), None if slice_off is None else _ptr(slice_off),
                    C.byref(ns))

    def aer_health(self, text, file_off, file_len, fatal_limit, nonfatal_limit, group_off, group_members):
        """kxpu_aer_health: (totals, group_aer).  text: bytes; file_off / file_len: 2n entries, the fatal file of record i
        at 2i and its non-fatal file at 2i+1; group_off [G+1] / group_members: the groups.  totals[2i + k] is a count or
        AER_UNKNOWN_COUNT; group_aer[o] holds AER_* bits."""
        t = np.frombuffer(bytes(text), np.uint8)
        file_off = np.ascontiguousarray(file_off, dtype=np.uint64)
        file_len = np.ascontiguousarray(file_len, dtype=np.uint32)
        assert len(file_off) == len(file_len) and len(file_off) % 2 == 0
        group_off = np.ascontiguousarray(group_off, dtype=np.uint32)
        group_members = np.ascontiguousarray(group_members, dtype=np.uint32)
        n, G = len(file_off) // 2, len(group_off) - 1
        totals = np.empty(max(2 * n, 1), np.uint64)
        group_aer = np.empty(max(G, 1), np.uint8)
        self._chk(self.L.kxpu_aer_health(
            self.ctx, _ptr(t) if len(t) else None, len(t), _ptr(file_off) if n else None, _ptr(file_len) if n else None, n,
            fatal_limit, nonfatal_limit, _ptr(group_off), _ptr(group_members) if len(group_members) else None, G,
            _ptr(totals), _ptr(group_aer)))
        return totals[:2 * n], group_aer[:G]

    def _slices(self, fn, dtype, driver, pool, node, generation, devs, taint=None, taints=None):
        devs = np.ascontiguousarray(devs)
        assert devs.dtype == dtype
        args = (self.ctx, _kind(driver), _kind(pool), _kind(node), generation, _ptr(devs) if len(devs) else None, len(devs))
        if taints is not None:
            table, since = taints
            tab = (DraTaint * max(len(table), 1))(*[DraTaint(_kind(k), _kind(v), _kind(e)) for k, v, e in table])
            if since is not None:
                since = np.ascontiguousarray(since, dtype=np.int64)
                assert since.size == len(devs) * len(table)
            args += (C.cast(tab, C.c_void_p), len(table), _ptr(since))
        if taint is not None:
            key, value, effect, since = taint
            if since is not None:
                since = np.ascontiguousarray(since, dtype=np.int64)
                assert since.shape == (len(devs),)
            args += (_kind(key), _kind(value), _kind(effect), None if since is None else _ptr(since))
        need, ns = C.c_size_t(0), C.c_size_t(0)
        rc = fn(*args, None, 0, C.byref(need), None, C.byref(ns))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        out = np.empty(max(need.value, 1), np.uint8)
        offs = np.empty(ns.value + 1, np.uint64)
        self._chk(fn(*args, _ptr(out), need.value, C.byref(need), _ptr(offs), C.byref(ns)))
        return out[:need.value].tobytes(), offs

    def cdi_emit(self, fmt, devs, kind=None):
        """kind=None: kxpu_cdi_emit (kind nvidia.com/gpu); else kxpu_cdi_emit_kind with that CDI kind (bytes or str)."""
        devs = np.ascontiguousarray(devs)
        assert devs.dtype == CDIDEV_DTYPE
        # one call with a buffer no document can outgrow (<= 384 B per device, plus the kind's bytes beyond 14); the
        # two-call sizing protocol (out = NULL -> *len) remains available and is exercised by the tests
        kb = _kind(kind)
        cap = (400 + (len(kb) if kb else 0)) * len(devs) + 1024
        out = np.empty(cap, np.uint8)
        got = C.c_size_t(0)
        dp = _ptr(devs) if len(devs) else None
        if kb is None:
            self._chk(self.L.kxpu_cdi_emit(self.ctx, fmt, dp, len(devs), _ptr(out), cap, C.byref(got)))
        else:
            self._chk(self.L.kxpu_cdi_emit_kind(self.ctx, fmt, kb, dp, len(devs), _ptr(out), cap, C.byref(got)))
        return out[:got.value].tobytes()

    def cdi_parse(self, fmt, doc, kind):
        """kxpu_cdi_parse: the CDIDEV_DTYPE records of a CDI spec kxpu_cdi_emit_kind wrote (doc bytes, kind bytes or
        str), in document order; KxpuError(E_INVALID) for any other document."""
        return self._parse(self.L.kxpu_cdi_parse, CDIDEV_DTYPE, fmt, doc, kind)

    def cdi_parse_mdev(self, fmt, doc, kind):
        """kxpu_cdi_parse_mdev: the MDEVCDI_DTYPE records of a vGPU class's CDI spec."""
        return self._parse(self.L.kxpu_cdi_parse_mdev, MDEVCDI_DTYPE, fmt, doc, kind)

    def cdi_parse_cdev(self, fmt, doc, kind):
        """kxpu_cdi_parse_cdev: the CDIDEV_DTYPE records (N in CDEV_FIELD) of a spec kxpu_cdi_emit_cdev wrote."""
        return self._parse(self.L.kxpu_cdi_parse_cdev, CDIDEV_DTYPE, fmt, doc, kind)

    def cdi_parse_mdev_cdev(self, fmt, doc, kind):
        """kxpu_cdi_parse_mdev_cdev: the MDEVCDEV_DTYPE records of a spec kxpu_cdi_emit_mdev_cdev wrote."""
        return self._parse(self.L.kxpu_cdi_parse_mdev_cdev, MDEVCDEV_DTYPE, fmt, doc, kind)

    def cdi_parse_vf_vgpu(self, fmt, doc, kind, cdev=False):
        """kxpu_cdi_parse_vf_vgpu (cdev: kxpu_cdi_parse_vf_vgpu_cdev): the VFVGPUCDI_DTYPE records of a spec the matching
        emit call wrote."""
        fn = self.L.kxpu_cdi_parse_vf_vgpu_cdev if cdev else self.L.kxpu_cdi_parse_vf_vgpu
        return self._parse(fn, VFVGPUCDI_DTYPE, fmt, doc, kind)

    def cdi_parse_raw(self, fmt, doc, kind, cap, mdev=False, offset=0, cdev=False, typed=False):
        """The bare call: doc placed at `offset` bytes past a 16-byte aligned host buffer, out of `cap` records.
        Returns (status, n, records) with n and the records as the call left them (n = -1: not stored).
        mdev and cdev: kxpu_cdi_parse_mdev_cdev, mdev: kxpu_cdi_parse_mdev, cdev: kxpu_cdi_parse_cdev, neither:
        kxpu_cdi_parse; typed: kxpu_cdi_parse_vf_vgpu, or with cdev kxpu_cdi_parse_vf_vgpu_cdev."""
        if typed:
            dtype = VFVGPUCDI_DTYPE
            fn = self.L.kxpu_cdi_parse_vf_vgpu_cdev if cdev else self.L.kxpu_cdi_parse_vf_vgpu
        elif mdev and cdev:
            dtype, fn = MDEVCDEV_DTYPE, self.L.kxpu_cdi_parse_mdev_cdev
        else:
            dtype = MDEVCDI_DTYPE if mdev else CDIDEV_DTYPE
            fn = self.L.kxpu_cdi_parse_mdev if mdev else self.L.kxpu_cdi_parse_cdev if cdev else self.L.kxpu_cdi_parse
        buf = np.zeros(len(doc) + offset + 16, np.uint8)
        base = (-buf.ctypes.data) % 16
        buf = buf[base:]
        buf[offset:offset + len(doc)] = np.frombuffer(bytes(doc), np.uint8)
        out = np.zeros(max(cap, 1), dtype)
        n = C.c_size_t((1 << 64) - 1)
        rc = fn(self.ctx, fmt, _kind(kind), buf.ctypes.data + offset if len(doc) else None, len(doc),
                _ptr(out) if cap else None, cap, C.byref(n))
        return rc, (-1 if n.value == (1 << 64) - 1 else n.value), out[:cap]

    def _parse(self, fn, dtype, fmt, doc, kind):
        doc = bytes(doc)
        cap = len(doc) // CDI_FRAG_MIN
        out = np.zeros(max(cap, 1), dtype)
        n = C.c_size_t(0)
        self._chk(fn(self.ctx, fmt, _kind(kind), doc, len(doc), _ptr(out), cap, C.byref(n)))
        return out[:n.value].copy()

    def cdi_emit_len(self, fmt, devs, kind=None):
        """Sizing call of the two-call protocol: out = NULL, returns the required length."""
        devs = np.ascontiguousarray(devs)
        need = C.c_size_t(0)
        kb = _kind(kind)
        dp = _ptr(devs) if len(devs) else None
        if kb is None:
            rc = self.L.kxpu_cdi_emit(self.ctx, fmt, dp, len(devs), None, 0, C.byref(need))
        else:
            rc = self.L.kxpu_cdi_emit_kind(self.ctx, fmt, kb, dp, len(devs), None, 0, C.byref(need))
        if rc not in (KXPU_OK, E_NOSPACE):
            self._chk(rc)
        return need.value

    def alloc_names(self, idx, kind=None):
        """kind=None: kxpu_alloc_names ("nvidia.com/gpu=<idx>"); else kxpu_alloc_names_kind ("<kind>=<idx>")."""
        idx = np.ascontiguousarray(idx, dtype=np.uint64)
        offs = np.empty(len(idx) + 1, np.uint32)
        need = C.c_size_t(0)
        kb = _kind(kind)
        cap = (22 + (len(kb) if kb else 14)) * len(idx) + 16
        out = np.empty(cap, np.uint8)
        if kb is None:
            self._chk(self.L.kxpu_alloc_names(self.ctx, _ptr(idx), len(idx), _ptr(out), cap, _ptr(offs), C.byref(need)))
        else:
            self._chk(self.L.kxpu_alloc_names_kind(self.ctx, kb, _ptr(idx), len(idx), _ptr(out), cap, _ptr(offs),
                                                   C.byref(need)))
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


def reconcile_outputs(n_prev, n_cur, fill=0):
    """Caller buffers of kxpu_reconcile (one spare element each, so that every pointer is valid), filled with `fill`."""
    return dict(index=np.full(max(n_cur, 1), fill, np.uint64), cur_state=np.full(max(n_cur, 1), fill & 0xFF, np.uint8),
                prev_state=np.full(max(n_prev, 1), fill & 0xFF, np.uint8), counts=np.zeros(1, RC_COUNTS_DTYPE),
                n_prev=n_prev, n_cur=n_cur)


def reconcile_result(out):
    c = out["counts"][0]
    return dict(index=out["index"][:out["n_cur"]].copy(), cur_state=out["cur_state"][:out["n_cur"]].copy(),
                prev_state=out["prev_state"][:out["n_prev"]].copy(),
                counts={k: int(c[k]) for k in RC_COUNTS_DTYPE.names})


def pref_requests(requests):
    """[(available, must-include, size)] -> the CSR arrays of kxpu_preferred_allocation (a one-element array stands in
    for an empty list, so that every pointer is valid)."""
    na = [len(r[0]) for r in requests]
    nm = [len(r[1]) for r in requests]
    avail_off = np.zeros(len(requests) + 1, np.uint32)
    must_off = np.zeros(len(requests) + 1, np.uint32)
    avail_off[1:] = np.cumsum(na, dtype=np.int64)
    must_off[1:] = np.cumsum(nm, dtype=np.int64)
    avail = np.zeros(max(int(avail_off[-1]), 1), np.uint32)
    must = np.zeros(max(int(must_off[-1]), 1), np.uint32)
    for q, (av, mu, _) in enumerate(requests):
        avail[avail_off[q]:avail_off[q + 1]] = av
        must[must_off[q]:must_off[q + 1]] = mu
    return dict(avail_off=avail_off, avail=avail, must_off=must_off, must=must,
                size=np.array([r[2] for r in requests], np.uint32).reshape(-1))


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
