/*
 * kxpu.h -- C ABI of libkxpu.so: the H100-native (sm_90a) implementation of the
 * kata-xpu-device-plugin discovery hot path.
 *
 * The reference (Apokleos/kata-xpu-device-plugin) is one Go binary with no FFI of its
 * own; this header is the boundary a cgo shim binds (see INTEGRATION.md).  Every entry
 * point names the reference code it replaces (file:line, paths relative to the
 * reference repository root).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only.
 *   - every function returns an int32 status: KXPU_OK (0) or a negative KXPU_E_* code.
 *   - inputs are borrowed for the duration of the call (cgo rule: no Go pointer is
 *     retained); outputs are caller-allocated, `cap` is passed, and when `cap` is too
 *     small the call returns KXPU_E_NOSPACE after storing the required size.
 *   - two calls take a struct that CONTAINS pointers (kxpu_classify_out: seven output arrays;
 *     kxpu_shard: device pointers).  From Go the arrays a kxpu_classify_out points at must be
 *     pinned for the call (runtime.Pinner) or C-allocated: cgo rejects a Go struct holding
 *     pointers to unpinned Go memory.  kxpu_shard only carries device addresses (not Go
 *     pointers) and needs nothing.  See INTEGRATION.md.
 *   - opaque handles (kxpu_ctx, kxpu_table) are owned by the library.
 *   - there is NO CPU fallback: without a usable sm_90 GPU kxpu_ctx_create fails with
 *     KXPU_E_NOGPU and nothing else can be called.
 *   - a kxpu_ctx may be used from several OS threads; calls on one ctx are serialised
 *     by an internal mutex (grpc-go runs Allocate handlers concurrently,
 *     pkg/device_plugin/generic_device_plugin.go:320).
 */
#ifndef KXPU_H
#define KXPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KXPU_ABI_VERSION 14

/* status codes */
#define KXPU_OK             0
#define KXPU_E_INVALID     -1  /* bad argument */
#define KXPU_E_CUDA        -2  /* CUDA runtime/driver error (see kxpu_last_error) */
#define KXPU_E_NOGPU       -3  /* no CUDA device / not an sm_90 part */
#define KXPU_E_NOSPACE     -4  /* caller buffer too small; required size was stored */
#define KXPU_E_CAPACITY    -5  /* internal table capacity exceeded after growth limit */
#define KXPU_E_NCCL        -6  /* NCCL / peer-memory exchange missing, failed or timed out */
#define KXPU_E_UNSUPPORTED -7  /* input outside the supported domain (documented per call) */
#define KXPU_E_NOMEM       -8

#define KXPU_ROW_MISS  (-1)            /* kxpu_lookup: key not present (reference: "") */
#define KXPU_REJECTED  0xFFFFFFFFu     /* kxpu_classify: record not accepted */

typedef struct kxpu_ctx   kxpu_ctx;
typedef struct kxpu_table kxpu_table;

/* ------------------------------------------------------------------ context */

/* Bind to one GPU (ordinal as in CUDA_VISIBLE_DEVICES order).  Fails with
 * KXPU_E_NOGPU when there is no device or its compute capability is not 9.0. */
int32_t kxpu_ctx_create(int32_t gpu_ordinal, kxpu_ctx **out);
int32_t kxpu_ctx_destroy(kxpu_ctx *ctx);
const char *kxpu_strerror(int32_t status);
/* Detailed message of the last failing call on this ctx (static storage inside ctx). */
const char *kxpu_last_error(kxpu_ctx *ctx);
/* Number of kernel launches issued by this ctx so far (bench accounting). */
uint64_t kxpu_launch_count(kxpu_ctx *ctx);
/* Device time in ms of the most recent call's kernels, per stage (parse, finalize,
 * lookup, ...).  Index with KXPU_T_*.  Measured with CUDA events on the ctx stream. */
#define KXPU_T_PARSE    0
#define KXPU_T_FINALIZE 1
#define KXPU_T_LOOKUP   2  /* 0 after kxpu_pciids_join(_device): the join runs beside the names, under KXPU_T_FINALIZE */
#define KXPU_T_NAMES    3
#define KXPU_T_CLASSIFY 4  /* also kxpu_reconcile's, kxpu_pcie_tree[_sriov / _mdev]'s and kxpu_sriov's kernels: the slot holds the most recent call's */
#define KXPU_T_EMIT     5  /* also kxpu_cdi_parse[_mdev|_cdev|_mdev_cdev|_vf_vgpu[_cdev]]: decode, re-emit and compare of the most recent call */
#define KXPU_T_MERGE    6
#define KXPU_T_RESOLVE  7  /* parse: second pass over the chunks whose governing line was not known */
#define KXPU_T_COUNT    8
int32_t kxpu_last_timings(kxpu_ctx *ctx, float ms_out[KXPU_T_COUNT]);
/* The per-stage events cost a few microseconds per call; on = 0 drops them (kxpu_last_timings
 * then reports nothing), on = 1 (default) restores them. */
int32_t kxpu_set_stage_timing(kxpu_ctx *ctx, int32_t on);
/* Device-side stopwatch over an arbitrary sequence of calls on this ctx: begin records a
 * CUDA event on the ctx stream, end records a second one, waits for it and returns the
 * elapsed milliseconds (bench.py times its K steps with this pair). */
int32_t kxpu_timer_begin(kxpu_ctx *ctx);
int32_t kxpu_timer_end(kxpu_ctx *ctx, float *ms_out);

/* Device / pinned memory helpers so a host program without a CUDA binding can keep
 * inputs resident (used by bench.py for the HBM-resident `value` measurement and for
 * pinned staging buffers of the `e2e` measurement). */
int32_t kxpu_dev_alloc(kxpu_ctx *ctx, size_t bytes, void **d_out);
int32_t kxpu_dev_free(kxpu_ctx *ctx, void *d_ptr);
int32_t kxpu_dev_upload(kxpu_ctx *ctx, void *d_dst, const void *h_src, size_t bytes);
int32_t kxpu_dev_download(kxpu_ctx *ctx, void *h_dst, const void *d_src, size_t bytes);
/* d_dst[i*n .. (i+1)*n) = d_src[0..n) for i in [0,copies): builds the "pci.ids x1000"
 * text of BASELINE.json configs[3] on the device. */
int32_t kxpu_dev_replicate(kxpu_ctx *ctx, void *d_dst, const void *d_src, size_t n, size_t copies);
/* page-locked host memory the GPU can address (cudaMallocHost): fast H2D source, zero-copy input of
 * kxpu_pciids_join */
int32_t kxpu_pinned_alloc(kxpu_ctx *ctx, size_t bytes, void **h_out);
int32_t kxpu_pinned_free(kxpu_ctx *ctx, void *h_ptr);
int32_t kxpu_sync(kxpu_ctx *ctx);

/* ----------------------------------------------- S2: pci.ids parse + lookup */

/* Parse a pci.ids text once and build the (vendor,device) -> row table.
 * Replaces the per-call file scan of getDeviceName/locateVendor
 * (pkg/device_plugin/device_plugin.go:208-275): for every key the table answers
 * exactly what that scan would answer on the same text --
 *   - the vendor anchor is the FIRST line whose first four bytes equal the vendor id
 *     (device_plugin.go:263-267),
 *   - its block is the run of following lines that start with '#' or '\t'
 *     (device_plugin.go:229-236); the first block line starting with "\t"+device wins
 *     (device_plugin.go:237),
 *   - bufio.Scanner semantics: a line of >= 65536 bytes ends the scan
 *     (device_plugin.go:262, bufio.MaxScanTokenSize).
 * Keys are (vendor<<16)|device rendered as four lowercase hex digits each, which is
 * what sysfs provides (device_plugin.go:142,164).
 * `text` is host memory; it is copied to the GPU inside the call and may be freed
 * afterwards (the table keeps sanitised names, not the text). */
int32_t kxpu_pciids_load(kxpu_ctx *ctx, const uint8_t *text, size_t n, kxpu_table **out);
/* Same, text already resident in device memory (16-byte aligned pointer). */
int32_t kxpu_pciids_load_device(kxpu_ctx *ctx, const void *d_text, size_t n, kxpu_table **out);
int32_t kxpu_table_free(kxpu_ctx *ctx, kxpu_table *t);
/* Number of (vendor,device) rows that a lookup can hit. */
int32_t kxpu_table_rows(kxpu_ctx *ctx, kxpu_table *t, uint32_t *n_rows);
/* Dump the table in file order (ascending line offset).  Arrays hold `cap` entries;
 * on KXPU_E_NOSPACE *n_rows holds the required count. */
int32_t kxpu_table_export(kxpu_ctx *ctx, kxpu_table *t, uint32_t *keys, uint64_t *line_off,
                          int32_t *rows, size_t cap, uint32_t *n_rows);

/* Batched join: rows_out[i] = row handle of keys[i] or KXPU_ROW_MISS.
 * Replaces one getDeviceName call per key (device_plugin.go:99). */
int32_t kxpu_lookup(kxpu_ctx *ctx, kxpu_table *t, const uint32_t *keys, size_t n,
                    int32_t *rows_out);
int32_t kxpu_lookup_device(kxpu_ctx *ctx, kxpu_table *t, const uint32_t *d_keys, size_t n,
                           int32_t *d_rows_out);
/* Parse and join in one call: what createDevicePlugins does for all device ids at start-up
 * (getDeviceName per id, device_plugin.go:99 -> :208-259).  Same results as
 * kxpu_pciids_load_device followed by kxpu_lookup_device; the join is enqueued behind the
 * parse without a host round trip in between.  Text, keys and rows are device pointers. */
int32_t kxpu_pciids_join_device(kxpu_ctx *ctx, const void *d_text, size_t n, const uint32_t *d_keys,
                                size_t nq, int32_t *d_rows_out, kxpu_table **out);

/* The same from host buffers: text and keys are copied to the GPU, the row handles come back in
 * rows_out, ONE host round trip.  This is the start-up path of the plugin: createDevicePlugins needs
 * the name of every device id once (device_plugin.go:91-105).  A small text (the real pci.ids is
 * 1.4 MB) is parsed, folded, finalized and joined by one cooperative kernel launch.
 * Zero-copy: when text, keys AND rows_out lie in pinned host memory the GPU can address
 * (kxpu_pinned_alloc, cudaHostAlloc, cudaHostRegister) and the text is 16-byte aligned, nothing is
 * copied: that kernel pulls the text over PCIe itself and writes the row handles to rows_out; the
 * call is one launch and one stream synchronisation.  Pageable buffers take the copying path with
 * the same results.  (A Go host reads the file into a kxpu_pinned_alloc buffer instead of
 * os.ReadFile's Go slice: C memory, nothing to pin for cgo.) */
int32_t kxpu_pciids_join(kxpu_ctx *ctx, const uint8_t *text, size_t n, const uint32_t *keys, size_t nq,
                         int32_t *rows_out, kxpu_table **out);

/* Sanitised resource names for row handles (device_plugin.go:241-251: TrimPrefix,
 * TrimSpace, ToUpper, '/'->'_', '.'->'_', \s+ -> '_', strip [^a-zA-Z0-9_.]).
 * Name i occupies out[offsets[i] .. offsets[i+1]); a miss row yields an empty name
 * (reference returns "" and the caller falls back to the raw id, :100-103).
 * *need receives the total bytes required. */
int32_t kxpu_names(kxpu_ctx *ctx, kxpu_table *t, const int32_t *rows, size_t n,
                   uint8_t *out, size_t cap, uint32_t *offsets, size_t *need);

/* ------------------------------- the rest of the pci.ids model (SURVEY 8(f) row 4) */

/* Subsystem rows and the class / subclass / prog-if section of the same text, on top of a finished
 * (vendor,device) table.  The reference scans these lines and ignores them
 * (device_plugin.go:229-237); their meaning is the file's own format statement
 * (utils/pci.ids:23-27, :38195-38200), taken with the reference's matching rules one level down:
 * raw byte prefixes, the FIRST line wins at every level (vendor / class line, device / subclass line
 * inside it, subsystem / prog-if line inside that), bufio line semantics.
 *   kind 0  vendor     key = vendor
 *   kind 1  subsystem  key = vendor<<48 | device<<32 | subvendor<<16 | subdevice
 *   kind 2  class section: class 1<<24 | c<<16;  subclass 2<<24 | c<<16 | s<<8;  prog-if 3<<24 | c<<16 | s<<8 | p
 * A row is (key, offset of its line in the text); names are the rest of that line.
 * d_text / n / t: the text the table `t` was built from (device memory, still resident); `t` must
 * outlive the returned object. */
typedef struct kxpu_full kxpu_full;
int32_t kxpu_pciids_full_load_device(kxpu_ctx *ctx, const void *d_text, size_t n, kxpu_table *t, kxpu_full **out);
int32_t kxpu_full_free(kxpu_ctx *ctx, kxpu_full *f);
/* rows of one kind in file order; on KXPU_E_NOSPACE *n_rows holds the required count */
int32_t kxpu_full_export(kxpu_ctx *ctx, kxpu_full *f, int32_t kind, uint64_t *keys, uint64_t *line_off, size_t cap,
                         uint32_t *n_rows);
/* batched probe (host buffers): line_off_out[i] = offset of the line of keys[i], or -1 */
int32_t kxpu_full_lookup(kxpu_ctx *ctx, kxpu_full *f, int32_t kind, const uint64_t *keys, size_t n, int64_t *line_off_out);

/* ------------------------------------------------------------- multi-GPU */

/* The pci.ids text shards by vendor-id range (SURVEY.md 8(e)): a cut may only fall where a
 * TOP-LEVEL line starts (first byte neither '\t' nor '#'), so no vendor block spans two shards.
 * Host-side planner: cuts_out[0] = 0 <= cuts_out[1] <= ... <= cuts_out[nranks] = n; rank r owns
 * text[cuts_out[r] .. cuts_out[r+1]).  A few memchr calls per cut; not part of the parse. */
int32_t kxpu_plan_shards(const uint8_t *text, size_t n, int32_t nranks, uint64_t *cuts_out /* nranks+1 */);

/* --- one process per rank (torchrun-style launch).  NCCL is loaded lazily (dlopen libnccl.so.2);
 * single-GPU users never need it.  kxpu_comm_init also maps every peer's exchange region through
 * CUDA IPC; the data plane of the sharded load is then peer-memory stores over NVLink, NCCL is the
 * fallback transport (KXPU_NO_P2P=1 forces it). */
#define KXPU_COMM_ID_BYTES 128
int32_t kxpu_comm_unique_id(uint8_t id_out[KXPU_COMM_ID_BYTES]);
int32_t kxpu_comm_init(kxpu_ctx *ctx, int32_t nranks, int32_t rank,
                       const uint8_t id[KXPU_COMM_ID_BYTES]);
int32_t kxpu_comm_destroy(kxpu_ctx *ctx);
/* Collective.  Each rank passes its shard of one logical text: bytes
 * [global_base, global_base+n) as planned by kxpu_plan_shards (16-byte aligned device pointer).
 * Every rank parses its shard; "first anchor wins" (device_plugin.go:263-267) is decided across
 * shards by an all-reduce(min) of the per-vendor first anchors, then only the winning rows and
 * their sanitised names are exchanged and inserted, and every rank returns the same table, equal
 * to kxpu_pciids_load on the concatenated text (same row handles on every rank).
 * A time-out (a rank missing for 4 s) or a CUDA error leaves the communicator unusable:
 * KXPU_E_NCCL until kxpu_comm_destroy + kxpu_comm_init. */
int32_t kxpu_pciids_load_sharded(kxpu_ctx *ctx, const void *d_text_shard, size_t n,
                                 uint64_t global_base, kxpu_table **out);
/* Collective: the sharded load plus the join of BASELINE configs[3].  Rank r probes its slice
 * d_keys[0..nq) = keys[key_offset .. key_offset+nq) of one logical key array of nq_total keys and
 * stores every hit into every rank's result buffer (the all-gather of hits rides on the probe
 * kernel); d_rows_all (device, [nq_total], may be NULL) receives all nq_total row handles on
 * every rank.  nq_total <= 2^21 on the peer-memory transport; the NCCL transport needs equal
 * slices in rank order. */
int32_t kxpu_pciids_join_sharded(kxpu_ctx *ctx, const void *d_text_shard, size_t n, uint64_t global_base,
                                 const uint32_t *d_keys, size_t nq, size_t key_offset, size_t nq_total,
                                 int32_t *d_rows_all, kxpu_table **out);

/* --- one process, N GPUs: what the reference's single Go process (cmd/main.go:5-7) binds.
 * The contexts of a group see each other's exchange regions through direct peer pointers
 * (cudaDeviceEnablePeerAccess), no IPC, no NCCL.  The same ordinal may appear more than once
 * (several contexts on one GPU: used by the single-GPU parity tests of the sharded path). */
typedef struct kxpu_multi kxpu_multi;
int32_t kxpu_ctx_create_multi(const int32_t *ordinals, int32_t n, kxpu_multi **out);
int32_t kxpu_multi_destroy(kxpu_multi *m);          /* destroys its contexts too */
int32_t kxpu_multi_size(kxpu_multi *m);
kxpu_ctx *kxpu_multi_ctx(kxpu_multi *m, int32_t i);  /* borrowed: usable with every single-ctx call */
typedef struct kxpu_shard {
    const void     *d_text;      /* shard on GPU i, 16-byte aligned                    */
    size_t          n;
    uint64_t        global_base;
    const uint32_t *d_keys;      /* key slice of rank i on GPU i (NULL: no join)       */
    size_t          nq;
    size_t          key_offset;
    int32_t        *d_rows_all;  /* [nq_total] on GPU i, may be NULL                   */
} kxpu_shard;
/* kxpu_pciids_join_sharded for all ranks of the group from ONE host thread: the kernels of every
 * rank are enqueued phase by phase, then all streams are awaited once.  tables_out[i] belongs to
 * kxpu_multi_ctx(m, i).  nq_total = 0: load only.
 * Limit: the ranks of a group exchange their winner rows through fixed peer slabs of 65 536 rows
 * and 2 MiB of names per rank.  A text whose shard holds more winners (or more name bytes)
 * fails with KXPU_E_CAPACITY ("winner rows outgrow the peer slab"); the group stays usable for
 * smaller texts.  Load such a text with one context (kxpu_pciids_load_device) instead. */
int32_t kxpu_multi_pciids_join(kxpu_multi *m, const kxpu_shard *shards /* [size] */, size_t nq_total,
                               kxpu_table **tables_out /* [size] */);

/* ----------------------------------------------- S1/S4: discovery classify */

/* One sysfs entry under /sys/bus/pci/devices, raw bytes as the Go host gathered them
 * (readIDFromFile / readLink, device_plugin.go:183-202), in filepath.Walk order
 * (device_plugin.go:132).  64 bytes. */
typedef struct kxpu_devrec {
    char     bdf[16];        /* entry name (info.Name()), NUL padded, <= 15 bytes      */
    uint8_t  vendor_txt[8];  /* first 8 bytes of the `vendor` file, e.g. "0x10de\n"     */
    uint8_t  device_txt[8];  /* first 8 bytes of the `device` file                      */
    char     driver[16];     /* basename of the `driver` link, NUL padded               */
    uint32_t iommu_group;    /* basename of the `iommu_group` link, decimal             */
    uint8_t  vendor_len;     /* length of the vendor file (0..8; longer => set flag)    */
    uint8_t  device_len;
    uint8_t  flags;          /* KXPU_REC_* */
    uint8_t  numa_node;      /* NUMA node of the function (0..63), valid only with KXPU_REC_NUMA (ABI v5) */
    uint32_t reserved1[2];
} kxpu_devrec;

#define KXPU_REC_VENDOR_ERR 0x01u /* readIDFromFile(vendor) failed  (device_plugin.go:143) */
#define KXPU_REC_DRIVER_ERR 0x02u /* readLink(driver) failed        (device_plugin.go:152) */
#define KXPU_REC_IOMMU_ERR  0x04u /* readLink(iommu_group) failed   (device_plugin.go:158) */
#define KXPU_REC_DEVICE_ERR 0x08u /* readIDFromFile(device) failed  (device_plugin.go:165) */
#define KXPU_REC_IS_DIR     0x10u /* info.IsDir()                   (device_plugin.go:137) */
/* numa_node holds a known NUMA node (kxpu_devrec and kxpu_mdevrec).  Without it the record's node is unknown,
 * so a zero-filled record -- every record built before ABI v5 -- means "no topology".
 *
 * NUMA node of a record: the host reads <entry>/numa_node (/sys/bus/pci/devices/<bdf>/numa_node for a PCI
 * function, <uuid>/../numa_node -- the parent's -- for an mdev), strips ONE trailing '\n', and sets the flag
 * only when what is left is a canonical decimal 0..63 (no sign, no leading zero except "0" itself).  Anything
 * else -- "-1" (no node), a failed read, 64 and above, "01", an empty file, junk -- leaves the node unknown and
 * is never an error.  The read changes nothing else: whether a record is accepted, its busIndex, its group and
 * every other output of kxpu_classify / _rules / _mdev and kxpu_mdev_names ignore numa_node and this flag.
 * A record whose flag is set with numa_node >= 64 counts as unknown. */
#define KXPU_REC_NUMA       0x40u
#define KXPU_MAX_NUMA_NODES 64
/* The entry is bound to a driver outside the caller's viability list, and iommu_group holds its group (ABI v8; see
 * kxpu_classify_viable).  Only kxpu_classify_viable reads it: every other call ignores the flag. */
#define KXPU_REC_BLOCKS     0x80u

/* Caller-allocated outputs of kxpu_classify; every array has room for n entries
 * (group_off / dev_off: n+1). */
typedef struct kxpu_classify_out {
    uint32_t *accept_index;  /* [n] busIndex of record i, or KXPU_REJECTED               */
    /* iommuMap (device_plugin.go:31,171): groups in first-seen walk order               */
    uint32_t *group_ids;     /* [n_groups]                                                */
    uint32_t *group_off;     /* [n_groups+1] into group_members                           */
    uint32_t *group_members; /* [n_accepted] record indices, walk order inside a group    */
    /* deviceMap (device_plugin.go:34,169): device ids in first-seen walk order; each
     * lists the groups whose FIRST member has that device id, in first-seen order.
     * dev_ids holds the id string bytes (little-endian packed, NUL padded, <= 8).       */
    uint64_t *dev_ids;       /* [n_devids]                                                */
    uint32_t *dev_off;       /* [n_devids+1] into dev_groups                              */
    uint32_t *dev_groups;    /* [n_groups] group ids == pluginapi.Device.ID (:94)         */
    uint32_t  n_accepted;
    uint32_t  n_groups;
    uint32_t  n_devids;
} kxpu_classify_out;

/* createIommuDeviceMap (device_plugin.go:126-180) + the device-list build of
 * createDevicePlugins (device_plugin.go:91-98) over a flat record table. */
int32_t kxpu_classify(kxpu_ctx *ctx, const kxpu_devrec *recs, size_t n, kxpu_classify_out *out);

/* One accepted (vendor, driver) pair of kxpu_classify_rules.  32 bytes. */
typedef struct kxpu_xpu_rule {
    char     vendor[8];    /* vendor id exactly as readIDFromFile returns it (data[2:], '\n' trimmed), e.g. "1002"; NUL padded */
    char     driver[16];   /* basename of the driver link, e.g. "vfio-pci"; NUL padded */
    uint32_t reserved[2];
} kxpu_xpu_rule;
#define KXPU_MAX_RULES 16

/* kxpu_classify for accelerators of any configured vendor (the reference's README TODO "To support other
 * GPUs", README.md:34-39).  The walk is createIommuDeviceMap's (device_plugin.go:126-180) with the two
 * NVIDIA constants replaced by a rule list:
 *   - a record is a candidate iff the conditions of :137-161 hold for some rule r, where the `10de` test
 *     of :149 reads "read_id(vendor) equals rules[r].vendor byte for byte, length included" and the
 *     `vfio-pci` test of :156 reads "driver equals rules[r].driver".  Rules are pairwise distinct, so at
 *     most one rule matches a record;
 *   - ONE walk and ONE busIndex counter (:130, :171-175) over all rules: accept_index, group_ids,
 *     group_off and group_members mean what they mean for kxpu_classify;
 *   - a group belongs to its FIRST member (:162-170) and to that member's rule; the members of one group
 *     may match different rules;
 *   - the key of a deviceMap entry (:169) is (rule of the group's first member, device id): one device
 *     id under two vendors gives two entries.  dev_ids keeps its meaning, dev_rule[d] (caller array of
 *     n entries, may be NULL) receives the rule index of entry d.
 * Invalid rule lists return KXPU_E_INVALID: n_rules is 0 or more than KXPU_MAX_RULES; a vendor is empty,
 * longer than 6 bytes (the longest id a record can carry after data[2:]), contains '\n' or has a
 * non-NUL byte after its first NUL; a driver is empty, 16 bytes or longer, contains '/' or has a non-NUL
 * byte after its first NUL; two rules are the same (vendor, driver) pair.
 * With rules = {{"10de", "vfio-pci"}} every array equals kxpu_classify's and dev_rule is all 0. */
int32_t kxpu_classify_rules(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                            size_t n, kxpu_classify_out *out, uint8_t *dev_rule /* [n] */);

/* ------------------------------------------------- S1/S4 for mediated vGPUs */

/* One entry under /sys/bus/mdev/devices (the reference's README TODO "To support vGPUs", README.md:34-39), raw
 * bytes as the host gathered them with the reference's read semantics (readIDFromFile = data[2:] with '\n'
 * trimmed, readLink = basename), entries in lexical order (the order filepath.Walk gives the PCI walk,
 * device_plugin.go:132).  Each entry <uuid> is a symlink into its parent PCI device's directory.  128 bytes, a
 * multiple of 16: the classify kernel reads a record with eight 16-byte vector loads. */
typedef struct kxpu_mdevrec {
    char     uuid[36];             /* entry name; anything but a 36-byte name is stored as 36 NUL bytes     */
    char     parent[16];           /* basename of the parent directory (its PCI address), NUL padded        */
    uint8_t  parent_vendor_txt[8]; /* first 8 bytes of <uuid>/../vendor                                     */
    char     driver[16];           /* basename of the mdev's `driver` link, NUL padded                      */
    uint8_t  type_name[40];        /* first 40 bytes of <uuid>/mdev_type/name                               */
    uint32_t iommu_group;          /* basename of the mdev's `iommu_group` link, decimal                    */
    uint8_t  vendor_len;           /* length of the parent's vendor file (a file over 8 bytes: a failed read) */
    uint8_t  name_len;             /* length of the type name file (0..40)                                  */
    uint8_t  flags;                /* KXPU_REC_VENDOR_ERR / _DRIVER_ERR / _IOMMU_ERR / _IS_DIR / _NAME_ERR / _NUMA */
    uint8_t  numa_node;            /* the parent's NUMA node, valid only with KXPU_REC_NUMA (ABI v5)        */
    uint32_t reserved1;
} kxpu_mdevrec;
#define KXPU_REC_NAME_ERR 0x20u /* reading mdev_type/name failed (kxpu_mdevrec only)                       */

/* kxpu_classify for mediated devices (vGPUs).  The semantics follow the shape of kubevirt-gpu-device-plugin, the
 * model the reference names, and keep the rest of this plugin's model: device ID = IOMMU group, one busIndex per
 * walk, CDI names <kind>=<index>.
 *   - a record is a CANDIDATE for rule r when it is not a directory, its uuid is a canonical lowercase UUID
 *     (8-4-4-4-12 hex digits [0-9a-f] with '-' between), read_id(parent_vendor_txt) equals rules[r].vendor, driver
 *     equals rules[r].driver (the matching of kxpu_classify_rules, "vendor" meaning the parent's vendor) and the
 *     vendor, driver and iommu_group reads succeeded;
 *   - the TYPE KEY of a record plays the part of the PCI `device` file: type_name[0..name_len) with the bytes
 *     "\t\n\v\f\r " trimmed from both ends, every ' ' replaced by '_', then every byte outside [A-Za-z0-9_.-]
 *     deleted.  It is at most 40 bytes and is the resource-name suffix (kubevirt: "GRID T4-1Q" -> GRID_T4-1Q);
 *   - a group comes into existence only at a candidate whose name read succeeded and whose type key is non-empty
 *     (the "device read works" rule of device_plugin.go:162-170); later members of an existing group are
 *     accepted without it;
 *   - grouping and indexing are kxpu_classify_rules': a group belongs to its first good record and that record's
 *     rule, busIndex counts accepted records over all rules in one walk, the iommuMap is a CSR in walk order;
 *   - a deviceMap entry is keyed by (rule of the group's first member, type key), entries in first-seen order.
 *     Two raw names with the same type key share one entry (one resource).
 * Domain restrictions; a record outside them is skipped like the corresponding read error, so this call never
 * returns KXPU_E_UNSUPPORTED:
 *   - name_len > 40 (a longer name file) counts as KXPU_REC_NAME_ERR;
 *   - vendor_len > 8 counts as KXPU_REC_VENDOR_ERR;
 *   - iommu_group must be the canonical decimal basename of the link and below 4294967295 (the host marks
 *     anything else KXPU_REC_IOMMU_ERR; iommu_group = 0xFFFFFFFF counts as that error here too);
 *   - parent is at most 15 bytes over [0-9a-f:.] (the host marks anything else KXPU_REC_VENDOR_ERR: the parent
 *     cannot be named in a CDI spec).
 * Outputs: `out` is filled with kxpu_classify_rules' meaning, EXCEPT dev_ids: here dev_ids[d] is the index of the
 * first record (lowest index) that is a candidate of any rule and carries entry d's type key, so the host reads
 * the type name (kxpu_mdev_names) and the UUID from its own records.  dev_rule as in kxpu_classify_rules.
 * Invalid rule lists return KXPU_E_INVALID, as in kxpu_classify_rules. */
int32_t kxpu_classify_mdev(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs,
                           size_t n, kxpu_classify_out *out, uint8_t *dev_rule /* [n] */);

/* The type keys (see kxpu_classify_mdev) of records recs[rec_idx[j]], j < k, with kxpu_names' two-call sizing:
 * key j occupies out[offsets[j] .. offsets[j+1]), *need receives the total.  A record whose name read failed
 * (KXPU_REC_NAME_ERR or name_len > 40) yields an empty key.  rec_idx[j] >= n is KXPU_E_INVALID. */
int32_t kxpu_mdev_names(kxpu_ctx *ctx, const kxpu_mdevrec *recs, size_t n, const uint32_t *rec_idx, size_t k,
                        uint8_t *out, size_t cap, uint32_t *offsets /* [k+1] */, size_t *need);

/* ------------------------------------------------------- NUMA topology of the groups */

/* kxpu_classify_rules / kxpu_classify_mdev plus the NUMA nodes of every group.  group_numa (caller array of n
 * entries) receives, for group ordinal g < n_groups:
 *   group_numa[g] = OR of (1 << numa_node) over the ACCEPTED members of group g that carry KXPU_REC_NUMA with
 *                   numa_node < 64;
 * 0 means "no topology" (no member's node is known).  Every other output is bitwise what kxpu_classify_rules /
 * kxpu_classify_mdev return for the same arguments (with rules = {{"10de", "vfio-pci"}}: what kxpu_classify
 * returns), and the calls run the same launches: the mask is folded into the pass that already visits every
 * accepted record with its group ordinal. */
int32_t kxpu_classify_topo(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, size_t n,
                           kxpu_classify_out *out, uint8_t *dev_rule /* [n] */, uint64_t *group_numa /* [n] */);
int32_t kxpu_classify_mdev_topo(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs,
                                size_t n, kxpu_classify_out *out, uint8_t *dev_rule /* [n] */,
                                uint64_t *group_numa /* [n] */);

/* ------------------------------------------------- IOMMU group viability (ABI v8) */

/* Whether VFIO can open each group.  The kernel lets VFIO take a group only when every PCI function in it is unbound
 * or bound to a driver that leaves DMA to its owner (vfio-pci and its variant drivers, pci-stub, pcieport); a group
 * that breaks this is offered to the kubelet, allocated, and then fails in QEMU with "group is not viable".
 * Host side: for a non-directory entry that is not a class candidate, the host reads its `driver` link; when that
 * driver is bound and not in the caller's viability list (the class drivers always count as allowed), it reads
 * `iommu_group`, and when that is a canonical decimal below 4294967295 it stores the group and the driver (first 15
 * bytes) and sets KXPU_REC_BLOCKS.
 *   - a record is a BLOCKER when it carries KXPU_REC_BLOCKS, is not KXPU_REC_IS_DIR and is not a candidate of any rule
 *     (a candidate ignores the flag: a class driver is always allowed);
 *   - group_blocker[o], for each group ordinal o < n_groups, is min{ i : record i is a blocker and
 *     iommu_group(i) == group_ids[o] }, or KXPU_VIABLE when there is none.  The minimum is walk order, so the host
 *     names the first blocking function.  A blocker may come before or after the group's first accepted record;
 *     blockers of groups that never come into existence (no candidate, or none whose device read works) produce
 *     nothing;
 *   - a blocker with iommu_group = 0xFFFFFFFF is outside the domain: KXPU_E_UNSUPPORTED, as for a candidate.
 * group_numa == NULL: every other output equals kxpu_classify_rules'; otherwise kxpu_classify_topo's (group_numa then
 * receives the masks).  KXPU_REC_BLOCKS changes nothing else, in this call or in any other.  Argument checks are
 * kxpu_classify_topo's, with group_blocker required instead of group_numa.
 * GPU: the candidate pass inserts a blocker's group into the same group table and lowers a spare word of its slot
 * with an atomic min; the per-group pass reads that word.  Same launches as kxpu_classify_rules / _topo.
 * vGPUs are out of scope: an mdev's IOMMU group is its own. */
#define KXPU_VIABLE 0xFFFFFFFFu
int32_t kxpu_classify_viable(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                             size_t n, kxpu_classify_out *out, uint8_t *dev_rule /* [n] */,
                             uint64_t *group_numa /* [n] or NULL */, uint32_t *group_blocker /* [n] */);

/* GetPreferredAllocation (the reference returns nil, nil: generic_device_plugin.go:378-386), batched over the
 * container requests of one PreferredAllocationRequest.  dev_numa[d] is the NUMA mask of the plugin's device d (the
 * group_numa of its group); positions are indices into that device list.  Request q:
 *   available      = avail[avail_off[q] .. avail_off[q+1])
 *   must-include   = must[must_off[q] .. must_off[q+1])
 *   size           = size[q]
 * Let home(d) = lowest set bit of dev_numa[d], or 64 when the mask is 0; U = the home nodes below 64 of the
 * must-include devices; candidates = available minus must-include; c[k] = the number of candidates with home k;
 * r = size - |must|.  The bins are ordered
 *   1. bins k in U with c[k] > 0, by c[k] descending, then k ascending;
 *   2. the other bins k < 64 with c[k] > 0, in the same order;
 *   3. bin 64 (unknown node) last.
 * The answer of request q, out[out_off[q] .. out_off[q+1]) with out_off[q+1] - out_off[q] = size[q], is the
 * must-include positions in request order followed by the first r candidates taken bin by bin, ascending position
 * inside a bin (position order is walk order: adjacent addresses stay together).  out_off is computed by the call.
 * KXPU_E_INVALID (and no output) when any request has a position >= n_devs, a duplicate inside available or inside
 * must-include, a must-include position that is not available, size < |must| or size > |available|.
 * Requests of up to 256 available positions run one warp each in a single launch; a larger request runs a
 * histogram pass, then a stable per-bin rank and scatter over the device positions with a decoupled look-back.
 * Limits (else KXPU_E_UNSUPPORTED): n_devs, n_req and the total of avail / must below 2^31. */
int32_t kxpu_preferred_allocation(kxpu_ctx *ctx, const uint64_t *dev_numa, size_t n_devs,
                                  const uint32_t *avail_off /* [n_req+1] */, const uint32_t *avail,
                                  const uint32_t *must_off /* [n_req+1] */, const uint32_t *must,
                                  const uint32_t *size /* [n_req] */, size_t n_req,
                                  uint32_t *out /* [sum of size] */, uint32_t *out_off /* [n_req+1] */);

/* ------------------------------------------------- PCIe topology of the groups (ABI v7) */

/* The PCIe path of one kxpu_devrec, a side record at the same index.  128 bytes.  len == 0 means "unknown", so a
 * zero-filled record is unknown.
 * Host side: readlink(<basePath>/<bdf>) (on real sysfs e.g.
 * "../../../devices/pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0"); path holds the target from its
 * first path component whose name begins with "pci" to the end, len its length.  No such component, a target longer
 * than 120 bytes from there, or a failed readlink store len = 0; none of these is an error.
 * Grammar (anything else makes the path unknown, never an error, like numa_node): components separated by a single
 * '/', no empty component, no trailing '/'; hex digits lowercase;
 *   host bridge  "pci" <domain> ":" <bus>
 *   function     <domain> ":" <bus> ":" <dev> "." <fn>
 * domain = exactly 4 digits, or 5..8 digits with a non-zero first digit (VMD domains such as 10000); bus = 2 digits;
 * dev = 2 digits, at most 1f; fn = one digit 0..7.  The first component is a host bridge; each later one is a
 * function or a host bridge (VMD puts pci10000:e0 below an endpoint); the last equals recs[i].bdf byte for byte
 * (up to its first NUL).  The components before the last are the record's CHAIN, 1..KXPU_PCIE_MAX_DEPTH long; the
 * depth of a component is its index in the chain.  Node key of a component:
 *   function     domain << 16 | bus << 8 | dev << 3 | fn
 *   host bridge  1 << 63 | domain << 16 | bus << 8 */
typedef struct kxpu_pcipath {
    char    path[120];
    uint8_t len;            /* 0..120; 0 = unknown; above 120 counts as unknown */
    uint8_t reserved[7];
} kxpu_pcipath;
#define KXPU_PCIE_MAX_DEPTH 8
#define KXPU_PCIE_NO_NODE   0xFFFFFFFFu

/* The PCIe forest of a walk.  recs / paths: the n records and paths the classify call saw; group_off [n_groups+1] /
 * group_members: its iommuMap CSR (kxpu_classify_out).
 *   - chain of group g = the longest common prefix, key by key, of the chains of its members whose path is known; a
 *     group none of whose members has a known path has no node;
 *   - a NODE is a distinct chain prefix (the whole prefix, not its last key), numbered in first-seen order: groups in
 *     ordinal order, each chain root to leaf, so parent[v] < v;
 *   - group_node[g] = the last node of g's chain, or KXPU_PCIE_NO_NODE;
 *   - key[v], parent[v] (KXPU_PCIE_NO_NODE for a root), depth[v] for v < *n_nodes.  key / parent / depth hold
 *     KXPU_PCIE_MAX_DEPTH * n_groups entries, which bounds the node count.
 * KXPU_E_INVALID (nothing written) when group_off decreases or a member index is >= n.
 * GPU: a parse of each path by 16 lanes (vector loads), one longest-common-prefix pass per group, a hash table of
 * the prefixes (keys compared prefix by prefix on a hit) with an atomic min of the first group, and the ordinals
 * from the single-pass scan.  Limit (else KXPU_E_UNSUPPORTED): n and n_groups below 2^28. */
int32_t kxpu_pcie_tree(kxpu_ctx *ctx, const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n,
                       const uint32_t *group_off /* [n_groups+1] */, const uint32_t *group_members, size_t n_groups,
                       uint32_t *group_node /* [n_groups] */, uint64_t *key, uint32_t *parent, uint8_t *depth,
                       uint32_t *n_nodes);

/* kxpu_preferred_allocation that keeps an allocation under as few PCIe switches as it can.  dev_node[d] is the node
 * of device d's group (kxpu_pcie_tree's group_node) or KXPU_PCIE_NO_NODE; parent / depth (n_nodes entries) are the
 * forest.  Device d lies in node v when v is on the path from dev_node[d] to its root.  Per request, with M the
 * must-include set, C the candidates (available minus M) and r = size - |M| as in kxpu_preferred_allocation:
 *   1. avail(v) = the available devices in v, mustin(v) = the must-include devices in v.  v qualifies when
 *      mustin(v) = |M| and avail(v) >= size.  X is the qualifying node with the smallest key
 *        (avail(v), -depth(v), avail(parent(v)), avail(grandparent(v)), ..., avail(root), lowest available position in v)
 *      -- a best fit at every level -- or all devices when no node qualifies.
 *   2. The candidates in X are ranked by lca, deepest first, then by NUMA bin (kxpu_preferred_allocation's order,
 *      c[k] counted over the candidates in X), then by position.  lca(c) = the greatest depth of a node holding c and
 *      at least one must-include device; "none" (every candidate when M is empty) ranks after depth 0.
 *   3. The answer is M in request order followed by the first r candidates of X in that order.
 * KXPU_E_INVALID (and no output): every case of kxpu_preferred_allocation; dev_node[d] >= n_nodes other than
 * KXPU_PCIE_NO_NODE; parent[v] >= v other than KXPU_PCIE_NO_NODE; depth[v] != depth[parent[v]] + 1, or != 0 for a
 * root; depth[v] >= KXPU_PCIE_MAX_DEPTH.
 * dev_node == NULL, or every entry KXPU_PCIE_NO_NODE, gives kxpu_preferred_allocation's answer byte for byte.
 * Shapes, limits and out_off as kxpu_preferred_allocation; n_nodes below 2^31.
 * The forest may be any walk's: kxpu_pcie_tree's, kxpu_pcie_tree_sriov's, or kxpu_pcie_tree_mdev's for vGPUs. */
int32_t kxpu_preferred_allocation_pcie(kxpu_ctx *ctx, const uint64_t *dev_numa, const uint32_t *dev_node, size_t n_devs,
                                       const uint32_t *parent, const uint8_t *depth, size_t n_nodes,
                                       const uint32_t *avail_off /* [n_req+1] */, const uint32_t *avail,
                                       const uint32_t *must_off /* [n_req+1] */, const uint32_t *must,
                                       const uint32_t *size /* [n_req] */, size_t n_req,
                                       uint32_t *out /* [sum of size] */, uint32_t *out_off /* [n_req+1] */);

/* ------------------------------------------- SR-IOV virtual functions (additions to ABI v14) */

/* These calls and kxpu_sriovrec were added to ABI v14 without a version bump: a caller detects them by symbol (dlsym), as
 * the ctypes binding and the Go shim do.  A virtual function (VF) bound to vfio-pci is a PCI function like any other, so
 * a passthrough class serves it.  What makes VFs different rests on sysfs ABI (Documentation/ABI/testing/sysfs-bus-pci:
 * physfn, virtfnN, sriov_numvfs) and on these facts:
 *   [assumed] since Linux 5.7, vfio-pci refuses to open a VF whose physical function (PF) is bound to vfio-pci unless
 *             the opener presents the PF's VF token ("VF token required to access device"), and refuses a PF on
 *             vfio-pci whose VFs are in use in the same way;
 *   [assumed] Kata's QEMU command line presents no VF token;
 *   [assumed] a VF reports its PF's vendor ID, so the PF's record, with its driver, is in the same walk;
 *   [assumed] <bdf>/physfn is a symlink whose basename is the PF's PCI address.
 * Host side: for every record that is a candidate of a passthrough class (vendor and driver of some class), the host
 * reads readlink(<bdf>/physfn) (basename) and the first 8 bytes of <bdf>/sriov_numvfs into a side record at the same
 * index; every other record gets a zero-filled one.  A missing link or file is not an error: the function is no VF, or
 * has no SR-IOV capability. */
typedef struct kxpu_sriovrec {
    char    physfn[16];     /* basename of the `physfn` link, NUL padded; empty: no link              */
    uint8_t numvfs_txt[8];  /* first 8 bytes of `sriov_numvfs`                                       */
    uint8_t numvfs_len;     /* length of the file (0..8; longer => 9)                                */
    uint8_t flags;          /* KXPU_SR_*                                                             */
    uint8_t reserved[6];
} kxpu_sriovrec;            /* 32 bytes: the kernel reads one with two 16-byte vector loads          */
#define KXPU_SR_PHYSFN_ERR 0x01u  /* readlink(physfn) failed for a reason other than "no such link"      */
#define KXPU_SR_NUMVFS_ERR 0x02u  /* reading sriov_numvfs failed for a reason other than "no such file"   */
#define KXPU_NO_PF 0xFFFFFFFFu

/* The SR-IOV verdict of a walk.  recs / srs: the n records and side records a classify call saw; group_ids / group_off /
 * group_members / n_groups: that call's iommuMap CSR (kxpu_classify_out of kxpu_classify_rules, _topo or _viable with the
 * same rules).  Outputs:
 *   - numvfs[i] = sriov_numvfs of record i: numvfs_txt[0..numvfs_len) with at most one trailing '\n' removed must be a
 *     canonical decimal 0..65535 (no sign, no leading zero except "0" itself); anything else -- empty, "07", "65536",
 *     "-1", junk, numvfs_len > 8, KXPU_SR_NUMVFS_ERR -- counts as 0 and is never an error (the numa_node rule);
 *   - pf_of[i] = p, the lowest index whose bdf (up to its first NUL) equals physfn (up to its first NUL), or KXPU_NO_PF
 *     when physfn is not a canonical lowercase "dddd:bb:dd.f" (4 hex digits, 2, 2 at most 1f, one digit 0..7), carries
 *     KXPU_SR_PHYSFN_ERR, no record matches, or p == i (a record never resolves to itself).  A VF whose PF is outside
 *     the walk gets KXPU_NO_PF, no verdict, and is served as any function is;
 *   - group_sriov[o], o < n_groups: the lowest member index i of group o (members are the accepted records) for which
 *       (a) pf_of[i] != KXPU_NO_PF and the PF record's driver equals the driver of some rule and the PF does not carry
 *           KXPU_REC_DRIVER_ERR (a class driver is a VFIO driver, so the VF needs the PF's VF token), or
 *       (b) numvfs[i] > 0 (a PF with VFs enabled: its tenant would own the device other tenants' VFs live on);
 *     KXPU_VIABLE when no member qualifies.
 * group_ids is not read (a group's ordinal is its position in the CSR) and may be NULL.
 * Argument checks are kxpu_classify_viable's (the rule list included); KXPU_E_INVALID, and nothing written, when
 * group_off decreases or a member index is >= n.  Limit (else KXPU_E_UNSUPPORTED, checked before any array is read): n
 * and n_groups below 2^30 (the address table has a power-of-two size of at least 2n slots).
 * GPU: three launches timed under KXPU_T_CLASSIFY -- (1) one thread per record parses sriov_numvfs and inserts its
 * canonical bdf, packed as domain << 16 | bus << 8 | dev << 3 | fn, into an open-addressing table holding the lowest
 * index per key (atomic min); (2) one thread per record probes its physfn; (3) one thread per group member folds the
 * verdict with an atomic min.  The records are read with 16-byte vector loads. */
int32_t kxpu_sriov(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                   const kxpu_sriovrec *srs, size_t n, const uint32_t *group_ids, const uint32_t *group_off /* [n_groups+1] */,
                   const uint32_t *group_members, size_t n_groups, uint32_t *pf_of /* [n] */, uint32_t *numvfs /* [n] */,
                   uint32_t *group_sriov /* [n_groups] */);

/* kxpu_pcie_tree with the VFs of a PF placed below it.  pf_of: kxpu_sriov's (n entries, each < n or KXPU_NO_PF).  The
 * chain of a member i with pf_of[i] = p != KXPU_NO_PF, where p's path is known and p's chain is shorter than
 * KXPU_PCIE_MAX_DEPTH, is p's chain followed by p's own node key (the function key of p's bdf): the PF becomes a node and
 * its VFs sit below it, whatever the VF's own path says.  When p's chain already has KXPU_PCIE_MAX_DEPTH keys the longer
 * chain would not fit, and i keeps its own chain, as in kxpu_pcie_tree; so does i when p's path is unknown.  Only one
 * level is followed: p's own pf_of is not read.  With pf_of all KXPU_NO_PF every output is bitwise kxpu_pcie_tree's.
 * KXPU_E_INVALID (nothing written): kxpu_pcie_tree's cases, pf_of == NULL with n > 0, or pf_of[i] >= n other than
 * KXPU_NO_PF.  kxpu_preferred_allocation_pcie needs no change: its best fit then packs a request's VFs by PF.
 * GPU: kxpu_pcie_tree's kernels; the parse keeps each record's own key and the longest-common-prefix pass reads a VF's
 * chain through its PF (compile-time variants: kxpu_pcie_tree's kernels are unchanged). */
int32_t kxpu_pcie_tree_sriov(kxpu_ctx *ctx, const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n,
                             const uint32_t *group_off /* [n_groups+1] */, const uint32_t *group_members, size_t n_groups,
                             uint32_t *group_node /* [n_groups] */, uint64_t *key, uint32_t *parent, uint8_t *depth,
                             uint32_t *n_nodes, const uint32_t *pf_of /* [n] */);

/* ------------------------------------------ PCIe forest of the mdev walk (addition to ABI v14) */

/* kxpu_pcie_tree for the mdev walk's records: same outputs, same CSR inputs (a kxpu_classify_mdev[_topo] call's), same
 * limits and errors.  Added to ABI v14 without a version bump: a caller detects it by symbol, as for kxpu_pcie_tree_sriov.
 * paths[i] is readlink(<mdevBasePath>/<uuid>) of record i, cut as kxpu_pcipath states: from its first component that
 * begins with "pci", unknown when over 120 bytes from there.  An mdev is a child device of its parent in the driver model, so the
 * target runs through the parent function, e.g.
 *   "../../../devices/pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0/<uuid>".
 * Grammar: kxpu_pcipath's, except for the leaf (anything else makes the path unknown, never an error):
 *   - the last component equals recs[i].uuid, all 36 bytes, and is a canonical lowercase UUID (8-4-4-4-12 over
 *     [0-9a-f] with '-' between);
 *   - the component before it is a function (not a host bridge) equal to recs[i].parent (up to its first NUL);
 *   - the CHAIN is every component before the UUID, the parent included, 1..KXPU_PCIE_MAX_DEPTH keys.  So the parent
 *     function is the deepest node of a group whose members share it, and every vGPU of one GPU sits below one node.
 *     With the first component a host bridge, a known chain has at least 2 keys; the 120-byte cap, 37 bytes of which
 *     the UUID takes, bounds it at 7 (a host bridge and 5 functions at most, on paths of host bridge and functions).
 * Node keys, VMD domains, the per-group longest common prefix and first-seen numbering are kxpu_pcie_tree's.  An mdev
 * whose parent is a VF needs nothing more: the VF is its chain's last key, below the PF's upstream port; the PF itself
 * (physfn) is not consulted.
 * Host-side policy, Plugin::vgpuPcieTopologyAware (off by default), rests on one fact:
 *   [assumed] the vGPU manager accepts several vGPUs of one physical GPU in one VM for the profiles a class serves, so
 *             packing a request under its parent GPU (kxpu_preferred_allocation_pcie's best fit) is what the user wants.
 * GPU: kxpu_pcie_tree's launches, the parse a compile-time variant for this record type and leaf (kxpu_pcie_tree's and
 * kxpu_pcie_tree_sriov's kernels are unchanged). */
int32_t kxpu_pcie_tree_mdev(kxpu_ctx *ctx, const kxpu_mdevrec *recs, const kxpu_pcipath *paths, size_t n,
                            const uint32_t *group_off /* [n_groups+1] */, const uint32_t *group_members, size_t n_groups,
                            uint32_t *group_node /* [n_groups] */, uint64_t *key, uint32_t *parent, uint8_t *depth,
                            uint32_t *n_nodes);

/* ------------------------------------ vGPUs on SR-IOV virtual functions (additions to ABI v14) */

/* These calls and their records were added to ABI v14 without a version bump: a caller detects them by symbol, as for
 * kxpu_sriov.  On a host with NVIDIA's vendor-specific VFIO framework (vGPU 17 and later on Linux 6.8 and later) no mdev
 * exists: each vGPU is an SR-IOV virtual function of the GPU whose profile the admin picks by writing a type ID to
 * <vf>/nvidia/current_vgpu_type, and the VF is then handed to the VM as a VFIO PCI function.  These facts are taken as
 * given, since no such host and no vendor document were at hand; a different layout only needs a different reader:
 *   [assumed] each such vGPU is a VF (<vf>/physfn exists) of an NVIDIA PF;
 *   [assumed] <vf>/nvidia/current_vgpu_type holds the VF's vGPU type ID as a decimal, and 0 when no vGPU is created on it;
 *   [assumed] <vf>/nvidia/creatable_vgpu_types holds a header line ("ID    : vGPU Name") and then one "<id> : <name>"
 *             line for each type the VF can take now.  A VF that already carries a type, and every VF of a full GPU,
 *             may list nothing, so the name of a type cannot be taken from the VF that carries it;
 *   [assumed] a type ID means the same name on every GPU of one host under one driver;
 *   [assumed] writing current_vgpu_type sends no bind uevent, so a type change does not move the uevent generation.
 * The driver a vGPU-carrying VF is bound to is configuration (the class's driver), not an assumption.
 * Host side: for every non-directory record whose vendor and driver match a class that serves vGPUs on VFs and that has
 * a physfn link, the host reads the first 16 bytes of nvidia/current_vgpu_type into a side record at the same index; every
 * other record gets a zero-filled one. */
typedef struct kxpu_vfvgpurec {
    uint8_t cur_txt[16];   /* first 16 bytes of nvidia/current_vgpu_type                                   */
    uint8_t cur_len;       /* length of the file (0..16; longer => 17)                                      */
    uint8_t flags;         /* KXPU_VT_READ / KXPU_VT_CUR_ERR                                                */
    uint8_t reserved[14];
} kxpu_vfvgpurec;          /* 32 bytes: the kernel reads one with two 16-byte vector loads                  */
#define KXPU_VT_READ    0x01u  /* the host read this record's files                                          */
#define KXPU_VT_CUR_ERR 0x02u  /* reading current_vgpu_type failed ("no such file" included)                 */
#define KXPU_VGPU_FILE_MAX 16384  /* the host uses no creatable_vgpu_types text longer than this (it logs it)   */

/* One record's type key: the layout of kxpu_classify_mdev's per-record key rows.  48 bytes. */
typedef struct kxpu_vgpukey {
    uint8_t key[40];       /* the type key, zero padded                                                     */
    uint8_t zero[7];       /* always 0: nothing else may live in the row, which is hashed and compared whole */
    uint8_t len;           /* key length, 0 = no key                                                        */
} kxpu_vgpukey;
/* kxpu_vf_vgpu_types' per-record status */
#define KXPU_VT_NONE    0u  /* the record was not read (no KXPU_VT_READ), or its type is 0                  */
#define KXPU_VT_NAMED   1u  /* a type ID that some table names: keys_out holds the key of that name          */
#define KXPU_VT_UNNAMED 2u  /* a type ID that no line of any table names                                     */
#define KXPU_VT_BAD     3u  /* KXPU_VT_CUR_ERR, cur_len > 16, or a text that is not a canonical decimal       */

/* The type join of a walk's vGPU VFs.  recs_vt: n side records.  blob: n_tables name tables, table t being
 * blob[table_off[t] .. table_off[t+1]), in priority order (the host sends the class's configured names, then the
 * creatable_vgpu_types text of every VF it read in walk order, then the names it learned in earlier walks; the call
 * treats them all alike).
 *   - a LINE ends at '\n' (the last line of a table may not); one trailing '\r' is dropped.  A line NAMES a type when it
 *     is [blanks] ID [blanks] ':' [blanks] NAME [blanks], blanks being ' ' and '\t', ID a canonical decimal
 *     1..4294967295 (no sign, no leading zero), NAME non-empty, at most 40 bytes, with a non-empty type key.  Every other
 *     line (the header included) is skipped;
 *   - the TYPE KEY of a NAME is kxpu_classify_mdev's: trim "\t\n\v\f\r " at both ends, ' ' -> '_', drop every byte
 *     outside [A-Za-z0-9_.-].  The rule is idempotent, so a key written back as a NAME gives the same key;
 *   - the name of an ID is the first line, in table order and then line order, that names it;
 *   - the current type of record i: cur_txt[0..cur_len) with at most one trailing '\n' removed must be a canonical
 *     decimal below 2^32 ("0" included).
 * Outputs, per record i:
 *   - status[i]: KXPU_VT_NONE when the record lacks KXPU_VT_READ or its type is 0; else KXPU_VT_BAD for
 *     KXPU_VT_CUR_ERR, cur_len > 16 or a text that is not canonical; else KXPU_VT_NAMED or KXPU_VT_UNNAMED;
 *   - type_id[i]: the parsed ID of a NAMED or UNNAMED record, else 0;
 *   - keys_out[i]: the key of the ID's name for a NAMED record, else all zero.
 * Limits (else KXPU_E_UNSUPPORTED): n below 2^30, checked before any array is read; table_off[n_tables] below 2^40,
 * checked before anything else is read; the number of lines below 2^30, counted on the GPU, with nothing written.
 * KXPU_E_INVALID, and nothing written: a table_off that decreases, a NULL array that is needed.
 * GPU: launches timed under KXPU_T_CLASSIFY -- (1) one warp per 2 KiB chunk of the blob finds the lines that start in
 * it, parses each and inserts its ID into an open-addressing table that keeps the lowest line offset per ID with an
 * atomic min (a line's blob offset orders lines by table, then by line); (2) one thread per record parses its current
 * type, probes the table, re-parses the winning line and writes the key row with three 16-byte stores.  The table starts
 * with 4096 slots; when more than half of them hold distinct IDs, both launches run again with room for every naming
 * line (four launches instead of two).  KXPU_T_CLASSIFY spans every run, table resets included. */
int32_t kxpu_vf_vgpu_types(kxpu_ctx *ctx, const kxpu_vfvgpurec *recs_vt, size_t n, const uint8_t *blob,
                           const uint64_t *table_off /* [n_tables+1] */, size_t n_tables, kxpu_vgpukey *keys_out /* [n] */,
                           uint32_t *type_id /* [n] */, uint8_t *status /* [n] */);

/* kxpu_classify_rules with one resource per vGPU type for the rules whose bit is set in vgpu_rules.  keys: n rows in
 * kxpu_vf_vgpu_types' layout (keys_out of that call).
 *   - a record that matches rule r with bit r set is a candidate only when its key row is non-empty (len > 0).  That
 *     test also stands in for the "device read works" rule: such a group comes into existence at its first candidate;
 *   - the deviceMap key of such a record is (r, type key), interned from the key rows as kxpu_classify_mdev interns its
 *     keys, so two IDs with one key share one entry; dev_ids[d] of such an entry is the lowest index of a candidate
 *     that carries the key (kxpu_classify_mdev's convention), dev_rule[d] its rule;
 *   - rules whose bit is clear behave exactly as in kxpu_classify_rules.
 * With vgpu_rules == 0 (keys may then be NULL) every output is bitwise that of kxpu_classify_rules (group_numa and
 * group_blocker NULL), kxpu_classify_topo (group_numa only) or kxpu_classify_viable (group_blocker given).
 * KXPU_E_INVALID: those calls' cases, a bit at or above n_rules, or vgpu_rules != 0 with keys == NULL.
 * GPU: compile-time variants of the candidate, intern and per-group kernels; every existing kernel is unchanged. */
int32_t kxpu_classify_vf_vgpu(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, uint32_t vgpu_rules,
                              const kxpu_devrec *recs, size_t n, const kxpu_vgpukey *keys /* [n] or NULL */,
                              kxpu_classify_out *out, uint8_t *dev_rule /* [n] */, uint64_t *group_numa /* [n] or NULL */,
                              uint32_t *group_blocker /* [n] or NULL */);

/* ------------------------------------------------- runtime rediscovery (ABI v6) */

/* One accepted entry of a walk, as a rediscovery compares two walks.  64 bytes. */
typedef struct kxpu_snaprec {
    char     key[40];       /* PCI address (PCI walk) or UUID (mdev walk), NUL padded, 1..39 bytes          */
    uint32_t iommu_group;
    uint32_t klass;         /* index of the class (xpuClasses / vgpuClasses) the entry itself matched       */
    uint64_t tag;           /* opaque identity word, compared for equality only                             */
    uint64_t index;         /* prev: its index; cur: ignored                                                */
} kxpu_snaprec;

#define KXPU_RC_KEPT    0u  /* same key, group, klass and tag in both walks: keeps its index           */
#define KXPU_RC_NEW     1u  /* cur only: the key is absent from prev                                   */
#define KXPU_RC_CHANGED 2u  /* the key is in both walks, but its group, klass or tag differs           */
#define KXPU_RC_RETIRED 3u  /* prev only: the key is absent from cur                                   */

typedef struct kxpu_reconcile_counts {
    uint64_t n_kept, n_new, n_changed, n_retired;  /* n_changed counts pairs: one cur and one prev entry each */
    uint64_t next_index_out;                       /* next_index + n_new + n_changed                          */
} kxpu_reconcile_counts;

/* Index reconciliation of a rediscovery: which entries of the new walk `cur` are the entries of the previous
 * snapshot `prev`, and which CDI index each gets.  Allocate hands out <kind>=<index> and the container runtime
 * resolves that name against the spec file later, so an index must never name two different devices while the
 * process lives:
 *   - cur[i] is KEPT iff some prev[j] has the same 40 key bytes, iommu_group, klass and tag; then
 *     index_out[i] = prev[j].index and prev_state[j] = KXPU_RC_KEPT;
 *   - every other cur[i] gets index_out[i] = next_index + (number of non-kept cur entries before i): fresh
 *     indices in walk order, never one handed out before (every prev index is below next_index);
 *   - cur_state[i]: KXPU_RC_KEPT, KXPU_RC_NEW (no prev entry has its key) or KXPU_RC_CHANGED (one has, with
 *     another group, klass or tag: the entry gets a fresh index);
 *   - prev_state[j]: KXPU_RC_KEPT, KXPU_RC_RETIRED (no cur entry has its key) or KXPU_RC_CHANGED;
 *   - counts: the four counts and next_index_out = next_index + (number of non-kept cur entries).
 * KXPU_E_INVALID, and nothing is written to any output, when: a key occurs twice within prev or within cur; a key is
 * empty (first byte NUL) or has a non-NUL byte after its first NUL; some prev[j].index >= next_index;
 * next_index + n_cur overflows 64 bits.
 * Two identities tie the call to the walk: n_prev = 0 with next_index = 0 gives index_out[i] = i (kxpu_classify's
 * busIndex when cur is the accepted records in walk order), and prev = the output of a call over the same cur (index
 * = index_out) gives all KEPT, the same indices and next_index_out = next_index.
 * The join is a hash table of at least 2 * (n_prev + n_cur) 16-byte slots (keys compared byte for byte on a hash
 * hit), one probe per cur entry, and the fresh indices come from the single-pass scan of the classify kernels.
 * Limit (else KXPU_E_UNSUPPORTED): n_prev + n_cur <= 2^30.  cur_state / prev_state / counts may be NULL. */
int32_t kxpu_reconcile(kxpu_ctx *ctx, const kxpu_snaprec *prev, size_t n_prev, uint64_t next_index,
                       const kxpu_snaprec *cur, size_t n_cur, uint64_t *index_out /* [n_cur] */,
                       uint8_t *cur_state /* [n_cur] */, uint8_t *prev_state /* [n_prev] */,
                       kxpu_reconcile_counts *counts);

/* ------------------------------------------------------- S3: CDI spec emit */

/* One accepted device as generateCDISpec sees it (device_plugin.go:59-76). 32 bytes. */
typedef struct kxpu_cdidev {
    char     bdf[16];       /* dev.addr, NUL padded                                       */
    uint32_t iommu_group;   /* devName (decimal)                                          */
    uint32_t vfio_cdev;     /* N of the function's VFIO cdev /dev/vfio/devices/vfio<N>: read by
                               kxpu_cdi_emit_cdev only (returned by kxpu_cdi_parse_cdev); the
                               other calls ignore it, and kxpu_cdi_parse returns 0 (ABI v14)  */
    uint64_t index;         /* dev.index                                                  */
} kxpu_cdidev;

#define KXPU_FMT_YAML 0  /* yaml.v3 encoder, SetIndent(2)   (cdi/spec.go:104-112)          */
#define KXPU_FMT_JSON 1  /* json.MarshalIndent(spec,"","  ") (cdi/spec.go:114-123)         */

/* generateCDISpec + CdiSpec.Save (device_plugin.go:55-80, cdi/spec.go:85-127) into a
 * caller buffer; devices are emitted in array order (canonical order: ascending index).
 * Call with out==NULL/cap==0 to obtain *len.  The host writes the file. */
int32_t kxpu_cdi_emit(kxpu_ctx *ctx, int32_t format, const kxpu_cdidev *devs, size_t n,
                      uint8_t *out, size_t cap, size_t *len);

/* kxpu_cdi_emit with the CDI kind as an argument: `kind` replaces "nvidia.com/gpu" (CdiVendorClass,
 * generic_device_plugin.go:31) in the `kind:` field (device_plugin.go:78), in the cdi.k8s.io/vfio<g>
 * annotation value (:66) and, for kind = "nvidia.com/gpu", the bytes equal kxpu_cdi_emit's.
 * Supported domain (else KXPU_E_UNSUPPORTED): a NUL-terminated "vendor/class" of at most 63 bytes;
 * vendor = a letter, then [A-Za-z0-9_.-], ending in a letter or digit; class = a letter, then
 * [A-Za-z0-9_-], ending in a letter or digit.  This is a subset of what the CDI v0.8.0 pkg/parser
 * vendor / class rules accept.  Inside it the kind is always written as it is:
 *   - YAML: it starts with a letter and contains '/', so yaml.v3's resolve cannot read it as an int,
 *     float, bool, null or timestamp, and neither isBase60Float nor isOldBool matches it (both need a
 *     leading digit / sign or a whole-word boolean); no character of it is an indicator that forces
 *     quoting in a plain scalar.  "kind=<index>" stays plain for the same reasons.
 *   - JSON: it holds no '"', '\\', control byte, '<', '>' or '&', so encoding/json escapes nothing.
 * The bdf domain of every kxpu_cdi_emit* call (kxpu_cdi_emit included; the parent of the vGPU calls alike), in both
 * formats (else KXPU_E_UNSUPPORTED, nothing written, the sizing call included): the bytes before the first NUL (all 16
 * when there is none), 1..16 of them over [0-9a-f:.], that yaml.v3 writes either plain or, when isBase60Float matches
 * them, double-quoted.  Restated from yaml.v3 v3.0.1 (resolve.go, encode.go, emitterc.go) for this alphabet, which
 * holds no sign, '_', 'x', 'o', letter of a bool / null word or '-' of a timestamp; refused are the bdfs that
 *   - are all decimal digits (resolve reads an int, or a float for 08 / 09 ...; the encoder would double-quote them);
 *   - are "0b" and one or more binary digits (an int: double-quoted);
 *   - match [0-9]+(\.[0-9]*)?(e[0-9]+)? or \.[0-9]+(e[0-9]+)? (a float, e.g. 1.5, .5, 0., 1e3: double-quoted);
 *   - end in ':' (the emitter's analysis forbids a plain scalar there and yaml.v3 single-quotes it);
 *   - start with "..." (a document end marker: single-quoted).
 * The last two would need a quoting style this library neither writes nor parses; refusing all five keeps the YAML
 * document's bdf a plain string to every YAML loader (a YAML 1.1 one such as PyYAML reads fewer of these as numbers, and
 * none of the accepted ones), and keeps both formats to one domain.  Every PCI address sysfs names is inside it.
 * Kinds up to 22 bytes run on the same kernel configuration as kxpu_cdi_emit; longer ones on a variant
 * with a larger per-device fragment bound (fewer CTAs per SM, DESIGN.md K6). */
int32_t kxpu_cdi_emit_kind(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_cdidev *devs, size_t n,
                           uint8_t *out, size_t cap, size_t *len);

/* One accepted vGPU as its CDI spec names it.  64 bytes. */
typedef struct kxpu_mdevcdi {
    char     uuid[36];      /* the mdev's UUID, canonical lowercase form                     */
    uint32_t iommu_group;   /* the mdev's own IOMMU group: /dev/vfio/<g>                      */
    char     parent[16];    /* PCI address of the parent device, NUL padded                   */
    uint64_t index;         /* busIndex                                                       */
} kxpu_mdevcdi;

/* The CDI spec of a vGPU class: kxpu_cdi_emit_kind's document (same head, tail, device order, zero-device form
 * and kind domain, KXPU_E_UNSUPPORTED outside it) with one annotation more per device.  The annotations, in
 * sorted key order for both encoders (yaml.v3 and encoding/json sort map keys; these four sort the same either
 * way):
 *   attach-pci: "true"
 *   bdf: <parent address>             (yaml.v3's isBase60Float quoting, as for kxpu_cdi_emit)
 *   cdi.k8s.io/vfio<g>: <kind>=<index>
 *   mdev: <uuid>
 * and the device node is /dev/vfio/<g> with g = iommu_group.  A uuid outside the canonical lowercase form
 * (8-4-4-4-12 over [0-9a-f], '-' between) or a parent outside kxpu_cdi_emit_kind's bdf domain (empty, a byte outside
 * [0-9a-f:.], or one of the five YAML classes listed there) is KXPU_E_UNSUPPORTED.
 * A canonical UUID is always written as it is:
 *   - YAML: it has exactly four '-' and 32 hex digits.  yaml.v3's resolve reads a plain scalar as int / float
 *     only when it is [-+]?digits (with an optional 0x / 0o / 0b prefix, '_' separators) or a float of the form
 *     [-+]?(\.[0-9]+|[0-9]+(\.[0-9]*)?)([eE][-+]?[0-9]+)? -- none has a '-' after the first byte; as a
 *     timestamp only in the forms 2006-01-02 ... which need a 4-digit group first (the UUID has 8 before its first
 *     '-'); never as bool / null (whole words: true, false, yes, no, on, off, y, n, null, ~) and never as base 60
 *     (that needs ':').  Its first byte is a hex digit, not an indicator, and it holds no ':', '#', space or
 *     quote, so the encoder emits it plain (a UUID of only decimal digits and '-', e.g.
 *     12345678-1234-1234-1234-123456789012, stays plain too).
 *   - JSON: it holds no '"', '\\', control byte, '<', '>' or '&', so encoding/json escapes nothing. */
int32_t kxpu_cdi_emit_mdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_mdevcdi *devs, size_t n,
                           uint8_t *out, size_t cap, size_t *len);

/* ------------------------------------------------- CDI spec parse (ABI v13) */

/* The shortest device fragment of any document kxpu_cdi_emit_kind / kxpu_cdi_emit_mdev write (YAML, a 3-byte kind,
 * one-digit index and group, a one-byte bdf such as "a", which stays plain): a document of len bytes names at most len / KXPU_CDI_FRAG_MIN devices,
 * so cap = len / KXPU_CDI_FRAG_MIN needs no second call. */
#define KXPU_CDI_FRAG_MIN 166

/* The inverse of kxpu_cdi_emit_kind: the records of a CDI spec this library wrote, so that a restarted plugin can read
 * back the indices it handed out (the container runtime resolves <kind>=<index> against these very bytes).
 *   - KXPU_OK with *n records exactly when kxpu_cdi_emit_kind(format, kind, out, *n) returns doc byte for byte.  The
 *     records come back in document order; any device order is accepted, not only ascending index.  bdf is NUL padded
 *     and vfio_cdev is 0, as the emitter's input would hold them.  The zero-device documents (YAML "devices: []", JSON
 *     "devices": null) give *n = 0.
 *   - KXPU_E_INVALID for every other document (nothing written to out, *n untouched), and for ctx, n or kind NULL, doc
 *     NULL with len > 0, out NULL with cap > 0, or a format other than KXPU_FMT_YAML / KXPU_FMT_JSON.  A document whose
 *     bdf the emitter refuses (KXPU_E_UNSUPPORTED) is not one it writes: KXPU_E_INVALID.
 *   - cap < *n: *n is stored and the call returns KXPU_E_NOSPACE, nothing written to out (KXPU_CDI_FRAG_MIN bounds *n).
 *   - KXPU_E_UNSUPPORTED: kind outside kxpu_cdi_emit_kind's domain, or len >= 2^32.
 * GPU: one decode kernel over the document in 8 KiB tiles (device starts by ballot, record slots by the decoupled
 * look-back), then the emitter's own kernel re-emits the decoded records into device scratch and a compare kernel
 * holds them against the document, so "accepted" and "round-trips" are the same statement.  The span from the decode
 * to the compare (one host read of the device count in between) is timed under KXPU_T_EMIT. */
int32_t kxpu_cdi_parse(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                       kxpu_cdidev *out, size_t cap, size_t *n);

/* The same for kxpu_cdi_emit_mdev's documents: KXPU_OK with *n records exactly when kxpu_cdi_emit_mdev(format, kind, out,
 * *n) returns doc byte for byte; a uuid outside the canonical lowercase form or a parent the emitter refuses makes the
 * document KXPU_E_INVALID.  Everything else as kxpu_cdi_parse. */
int32_t kxpu_cdi_parse_mdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                            kxpu_mdevcdi *out, size_t cap, size_t *n);

/* ------------------------------------------ CDI specs naming VFIO device cdevs (ABI v14) */

/* A function bound to vfio-pci can also be opened through its own VFIO character device instead of its group's
 * /dev/vfio/<g>:
 *   [assumed] since Linux 6.6 such a function has /dev/vfio/devices/vfio<N>, and its sysfs directory holds vfio-dev/
 *             with the one entry vfio<N>;
 *   [assumed] a kernel built with CONFIG_VFIO_GROUP=n has no /dev/vfio/<g> at all;
 *   [assumed] a VMM opens the cdev through iommufd (/dev/iommu), which the runtime opens itself, as it opens
 *             /dev/vfio/vfio for a group; Kata attaches a /dev/vfio/devices/vfio<N> node through QEMU's iommufd
 *             backend.  So the spec names no /dev/iommu node;
 *   [assumed] cdev numbers are handed out at bind time and reused: two functions unbound and re-bound in the other order
 *             swap numbers.
 * The IOMMU group stays the unit of allocation (iommufd claims DMA ownership for the whole group). */

/* kxpu_cdi_emit_kind's document, byte for byte, except that the device node of device i is
 * /dev/vfio/devices/vfio<N> with N = devs[i].vfio_cdev (every uint32 is valid) in place of /dev/vfio/<g>.  The
 * annotations (cdi.k8s.io/vfio<g> included), head, tail, zero-device form, device order, kind and bdf domains, sizing
 * protocol and KXPU_E_UNSUPPORTED cases are kxpu_cdi_emit_kind's.
 * GPU: the kernel of kxpu_cdi_emit_kind with the node literal and number compiled in; the longest fragment is 12 bytes
 * longer, and kinds up to 22 bytes still run at four CTAs per SM (DESIGN.md K6).  Timed under KXPU_T_EMIT. */
int32_t kxpu_cdi_emit_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_cdidev *devs, size_t n,
                           uint8_t *out, size_t cap, size_t *len);

/* The inverse of kxpu_cdi_emit_cdev: KXPU_OK with *n records exactly when kxpu_cdi_emit_cdev(format, kind, out, *n)
 * returns doc byte for byte; vfio_cdev holds each device's N.  A document of kxpu_cdi_emit_kind (a group node) is
 * KXPU_E_INVALID here, as a document of kxpu_cdi_emit_cdev is for kxpu_cdi_parse; the zero-device documents are the same
 * bytes in both layouts, and both calls return *n = 0 for them.  KXPU_CDI_FRAG_MIN still bounds *n.  Everything else as
 * kxpu_cdi_parse. */
int32_t kxpu_cdi_parse_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                            kxpu_cdidev *out, size_t cap, size_t *n);

/* ------------------------------- CDI specs naming the VFIO cdevs of vGPUs (additions to ABI v14) */

/* These two calls were added to ABI v14 without a version bump: a caller detects them by symbol (dlsym), as the ctypes
 * binding and the Go shim do.  An mdev can be opened through its own VFIO character device like a PCI function:
 *   [assumed] on a kernel with CONFIG_VFIO_DEVICE_CDEV=y, an mdev whose vendor driver registers a VFIO device gets
 *             /dev/vfio/devices/vfio<N>, and <mdevBasePath>/<uuid>/vfio-dev/ holds the one entry vfio<N>, the layout of
 *             a PCI function.  With CONFIG_IOMMUFD the kernel requires iommufd ops of every VFIO driver, so a working
 *             vGPU driver has a cdev; only the operator knows whether the node's vGPU driver does, so a vGPU class
 *             opts in on its own;
 *   [assumed] mdev and PCI cdev numbers come from one number space and are reused: re-creating an mdev with the same
 *             UUID can give it another N;
 *   [assumed] Kata attaches an mdev cdev through QEMU's iommufd backend, as it does a function's, so the spec names no
 *             /dev/iommu node (the runtime opens it itself). */

/* One accepted vGPU of a class served through VFIO cdevs.  80 bytes (16-byte strides for the kernels' vector loads). */
typedef struct kxpu_mdevcdev {
    kxpu_mdevcdi dev;        /* exactly what kxpu_cdi_emit_mdev reads                    */
    uint32_t     vfio_cdev;  /* N of /dev/vfio/devices/vfio<N>; every uint32 is valid    */
    uint32_t     reserved[3];/* ignored by the emitter, written 0 by the parser           */
} kxpu_mdevcdev;

/* kxpu_cdi_emit_mdev's document for devs[i].dev, byte for byte, except that the device node of device i is
 * /dev/vfio/devices/vfio<N> with N = devs[i].vfio_cdev in place of /dev/vfio/<g>.  The four annotations (cdi.k8s.io/vfio<g>
 * and mdev: <uuid> included), head, tail, zero-device form, device order, kind domain, uuid and parent refusals
 * (KXPU_E_UNSUPPORTED; the parent has kxpu_cdi_emit_kind's bdf domain) and sizing protocol are kxpu_cdi_emit_mdev's.
 * GPU: the kernel of kxpu_cdi_emit_mdev with the node literal and number compiled in; the longest fragment is 12 bytes
 * longer (492), and the tile still runs three CTAs per SM (DESIGN.md K6).  Timed under KXPU_T_EMIT. */
int32_t kxpu_cdi_emit_mdev_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_mdevcdev *devs, size_t n,
                                uint8_t *out, size_t cap, size_t *len);

/* The inverse of kxpu_cdi_emit_mdev_cdev: KXPU_OK with *n records exactly when kxpu_cdi_emit_mdev_cdev(format, kind, out,
 * *n) returns doc byte for byte; vfio_cdev holds each device's N and reserved is 0.  A document of kxpu_cdi_emit_mdev,
 * kxpu_cdi_emit_kind or kxpu_cdi_emit_cdev is KXPU_E_INVALID here (and each of their parsers refuses this call's
 * documents); the zero-device documents are the same bytes in every layout, and every parser returns *n = 0 for them.
 * KXPU_CDI_FRAG_MIN still bounds *n.  Everything else as kxpu_cdi_parse_mdev. */
int32_t kxpu_cdi_parse_mdev_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                                 kxpu_mdevcdev *out, size_t cap, size_t *n);

/* ------------------------- CDI specs that carry the vGPU type of each SR-IOV VF (additions to ABI v14) */

/* These four calls were added to ABI v14 without a version bump: a caller detects them by symbol (dlsym), as the ctypes
 * binding and the Go shim do.  A VF that carries a vGPU type lists nothing in creatable_vgpu_types, so a restarted
 * plugin on a full GPU cannot learn the names of the types it serves from sysfs; and a spec that does not hold each VF's
 * type cannot tell a restarted plugin that a VF changed type while it was down.  These layouts put the type ID and the
 * type key of each VF in two more device annotations, so the spec itself carries both facts across a restart.
 *   [assumed] the container runtime's CDI registry accepts any string value of a device annotation and ignores keys it
 *             does not know (the bdf and mdev annotations already rest on this). */

/* One served VF of a class that serves vGPUs on SR-IOV VFs.  80 bytes (16-byte strides for the kernels' vector loads). */
typedef struct kxpu_vfvgpucdi {
    kxpu_cdidev dev;         /* exactly what kxpu_cdi_emit_kind / kxpu_cdi_emit_cdev read                    */
    uint32_t    type_id;     /* the VF's vGPU type ID, 1 .. 2^32-1                                            */
    uint8_t     key_len;     /* 1 .. 40                                                                       */
    uint8_t     reserved[3]; /* ignored by the emitters, written 0 by the parsers                             */
    char        key[40];     /* its type key (kxpu_vgpukey.key): bytes past key_len are ignored, written 0    */
} kxpu_vfvgpucdi;

/* kxpu_cdi_emit_kind's document for devs[i].dev, byte for byte, except for two more annotations per device.  The
 * annotations, in sorted key order (the same for yaml.v3 and encoding/json):
 *   attach-pci: "true"
 *   bdf: <address>                    (yaml.v3's isBase60Float quoting, as for kxpu_cdi_emit)
 *   cdi.k8s.io/vfio<g>: <kind>=<index>
 *   vgpu-type: "<type_id>"            (canonical decimal)
 *   vgpu-type-key: "<key>"
 * Both new values are always double-quoted, in YAML too: this is this project's canonical form.  A plain 557, or a key
 * such as 1e5, true, No, 0x1F, .inf or 2024-01-01, would resolve as a non-string, and a CDI registry that reads
 * annotations as map[string]string would then refuse the whole spec.  Over the key alphabet [A-Za-z0-9_.-] and the
 * digits a quoted value needs no escape in either format.
 * KXPU_E_UNSUPPORTED, with nothing written: every case kxpu_cdi_emit_kind refuses (its bdf domain included), type_id 0,
 * key_len 0 or above 40, or a key byte (of the first key_len) outside [A-Za-z0-9_.-].
 * GPU: the kernel of kxpu_cdi_emit_kind with the annotations compiled in; each record is read with five 16-byte loads
 * and a warp copies the key straight from the device array.  The longest fragment grows by 104 bytes, and kinds up to 22
 * bytes run at three CTAs per SM, longer ones at two (DESIGN.md K6).  Timed under KXPU_T_EMIT. */
int32_t kxpu_cdi_emit_vf_vgpu(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_vfvgpucdi *devs, size_t n,
                              uint8_t *out, size_t cap, size_t *len);
/* kxpu_cdi_emit_vf_vgpu's document, except that the device node of device i is /dev/vfio/devices/vfio<N> with
 * N = devs[i].dev.vfio_cdev in place of /dev/vfio/<g> (kxpu_cdi_emit_cdev's node).  Everything else as
 * kxpu_cdi_emit_vf_vgpu. */
int32_t kxpu_cdi_emit_vf_vgpu_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_vfvgpucdi *devs, size_t n,
                                   uint8_t *out, size_t cap, size_t *len);

/* The inverses: KXPU_OK with *n records exactly when kxpu_cdi_emit_vf_vgpu (_cdev: kxpu_cdi_emit_vf_vgpu_cdev) given
 * them returns doc byte for byte.  dev is what kxpu_cdi_parse (_cdev: kxpu_cdi_parse_cdev) returns; type_id, key_len and
 * key come from the annotations, reserved and the key bytes past key_len are 0.  The six CDI layouts (kind, cdev, mdev,
 * mdev cdev and these two) refuse each other's documents with KXPU_E_INVALID; the zero-device documents are the same
 * bytes in every layout, and every parser returns *n = 0 for them.  KXPU_CDI_FRAG_MIN still bounds *n.  Everything else
 * as kxpu_cdi_parse. */
int32_t kxpu_cdi_parse_vf_vgpu(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                               kxpu_vfvgpucdi *out, size_t cap, size_t *n);
int32_t kxpu_cdi_parse_vf_vgpu_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                                    kxpu_vfvgpucdi *out, size_t cap, size_t *n);

/* ------------------------------------------------------ S5: Allocate names */

/* updateResponseForCDI / QualifiedName (generic_device_plugin.go:274-299,
 * cdi/cdi-utils.go:9): name i = "nvidia.com/gpu=" + decimal(idx[i]). */
int32_t kxpu_alloc_names(kxpu_ctx *ctx, const uint64_t *idx, size_t n, uint8_t *out,
                         size_t cap, uint32_t *offsets, size_t *need);
/* The same with the CDI kind as an argument (QualifiedName(vendor, class, idx), cdi-utils.go:9):
 * name i = kind + "=" + decimal(idx[i]).  `kind` has kxpu_cdi_emit_kind's domain (else
 * KXPU_E_UNSUPPORTED); kind = "nvidia.com/gpu" gives kxpu_alloc_names' bytes. */
int32_t kxpu_alloc_names_kind(kxpu_ctx *ctx, const char *kind, const uint64_t *idx, size_t n, uint8_t *out,
                              size_t cap, uint32_t *offsets, size_t *need);

/* ListAndWatchResponse wire bytes for a device list (generic_device_plugin.go:224):
 * repeated field 1 { string ID = 1 (decimal group); string health = 2 }.
 * healthy[i] != 0 -> "Healthy" else "Unhealthy"; healthy == NULL -> all healthy. */
int32_t kxpu_lw_encode(kxpu_ctx *ctx, const uint32_t *group_ids, const uint8_t *healthy,
                       size_t n, uint8_t *out, size_t cap, size_t *len);

/* kxpu_lw_encode with the NUMA topology of every device (v1beta1 Device.topology, what the kubelet Topology
 * Manager aligns on).  Device i, fields in number order as kubelet v0.30's gogo-generated api.pb.go marshals them:
 *   string ID = 1; string health = 2;
 *   when numa_mask[i] != 0: TopologyInfo topology = 3 { repeated NUMANode nodes = 1 { int64 ID = 1 } },
 *   one node per set bit, ascending.
 * proto3 omits a zero int64, so node 0 is an empty NUMANode (0a 00).  A topology of many nodes makes a Device longer
 * than 127 bytes: both lengths are varints.  numa_mask == NULL or all masks 0 gives kxpu_lw_encode's bytes.
 * Limit (else KXPU_E_UNSUPPORTED): n below 2^32 / 283 (the longest Device is 283 bytes). */
int32_t kxpu_lw_encode_topo(kxpu_ctx *ctx, const uint32_t *group_ids, const uint8_t *healthy, const uint64_t *numa_mask,
                            size_t n, uint8_t *out, size_t cap, size_t *len);

/* ------------------------------------------- DRA ResourceSlices (ABI v9) */

/* Kubernetes Dynamic Resource Allocation publishes devices as ResourceSlice objects (resource.k8s.io/v1).  Facts about
 * that API are stated from memory of the upstream Go types, not checked against k8s.io/api; each is marked [assumed]:
 *   [assumed] resource.k8s.io/v1 is GA since Kubernetes 1.34;
 *   [assumed] the v1 ResourceSlice field order is kind, apiVersion, metadata, spec; ResourceSliceSpec is driver, pool,
 *             nodeName, ..., devices; ResourcePool is name, generation, resourceSliceCount; Device is name, attributes;
 *             DeviceAttribute holds exactly one of int, bool, string, version;
 *   [assumed] a slice lists at most 128 devices; a device has at most 32 attributes; an attribute name is a C
 *             identifier of at most 32 bytes, optionally qualified by a DNS subdomain; a string value is at most 64
 *             bytes; a device name is a DNS label;
 *   [assumed] the driver name is a lowercase DNS subdomain of at most 63 bytes; pool and node names are lowercase DNS
 *             subdomains of at most 253 bytes;
 *   [assumed] resource.kubernetes.io/pcieRoot is the standard attribute that aligns devices of different drivers
 *             under one PCIe root complex;
 *   [assumed] without taints (ABI v11, below) a published device is schedulable: the v9 / v10 calls publish no
 *             per-device health. */

/* One published device (one IOMMU group of one class).  128 bytes: the kernel reads it with eight 16-byte loads. */
typedef struct kxpu_dradev {
    uint8_t  product[64];   /* productName bytes, NUL padded                                                 */
    char     bdf[16];       /* PCI address of the group's first accepted member                              */
    char     pcie_root[16]; /* "pci<domain>:<bus>", the first component of that member's path; "" = unknown */
    char     vendor[8];     /* read_id(vendor) of that member, NUL padded                                    */
    char     device[8];     /* read_id(device)                                                               */
    uint64_t numa_mask;     /* the group's NUMA mask (kxpu_classify_topo)                                    */
    uint32_t iommu_group;
    uint8_t  product_len;   /* 0..64                                                                         */
    uint8_t  reserved[3];
} kxpu_dradev;
#define KXPU_DRA_SLICE_DEVICES 128       /* devices per slice: the v1 limit [assumed]                          */
#define KXPU_DRA_MAX_DEVICES   (1u << 24) /* n must be below this                                               */

/* The ResourceSlices of one pool: S = max(1, ceil(n / 128)) slices, slice s holding devs[128 s .. min(n, 128 s + 128))
 * in array order.  out receives S compact JSON objects (no spaces), each followed by one '\n' (a JSON Lines file);
 * object s is out[slice_off[s] .. slice_off[s+1] - 1) and its '\n' is the byte before slice_off[s+1].  With out == NULL
 * or cap < *len the call stores *len and *n_slices and returns KXPU_E_NOSPACE, as kxpu_cdi_emit does.  slice_off (may be
 * NULL) has S + 1 entries and is written only on KXPU_OK.
 *
 * Every object is
 *   {"kind":"ResourceSlice","apiVersion":"resource.k8s.io/v1","metadata":{"generateName":"<node>-<driver>-"},
 *    "spec":{"driver":"<driver>","pool":{"name":"<pool>","generation":<generation>,"resourceSliceCount":<S>},
 *    "nodeName":"<node>","devices":[<device>,<device>,...]}}
 * (one line; fields in the declaration order of the Go v1 types [assumed]).  A device is
 *   {"name":"vfio<g>","attributes":{<attributes>}}
 * with g = iommu_group in decimal: a DNS label that mirrors the cdi.k8s.io/vfio<g> annotation of the CDI spec.  The
 * attributes, keys sorted bytewise as encoding/json sorts map keys:
 *   "deviceID":{"string":"<device>"}                                  always
 *   "iommuGroup":{"int":<g>}                                          always
 *   "numaNode":{"int":<k>}                                            only when numa_mask has exactly one bit k set
 *   "pciAddress":{"string":"<bdf>"}                                   always; a driver-local name on purpose
 *   "productName":{"string":"<product[0..product_len)>"}              only when product_len > 0
 *   "resource.kubernetes.io/pcieRoot":{"string":"<pcie_root>"}        only when pcie_root is not empty
 *   "vendorID":{"string":"<vendor>"}                                  always
 * n = 0 gives one slice with "devices":[]: a pool without devices still tells the scheduler the node has none.
 * These bytes are this project's canonical form (the checker pins them); they are not claimed to equal Go's, which
 * would also write "creationTimestamp":null.
 *
 * KXPU_E_INVALID, nothing written (not even *len): ctx, len or n_slices NULL, devs NULL with n > 0; driver not a
 * lowercase DNS subdomain (labels of [a-z0-9-] that start and end with [a-z0-9], joined by '.', each at most 63 bytes)
 * of at most 63 bytes; pool or node not such a subdomain of at most 253 bytes; generation >= 2^63.  These checks mean
 * that no string needs JSON escaping.
 * KXPU_E_UNSUPPORTED, with *len, the output and slice_off untouched: n >= KXPU_DRA_MAX_DEVICES, or a record outside
 * the domain:
 *   - product[0..product_len) over [A-Za-z0-9_.-] (the resource-name sanitiser's output and a raw hex id both fit);
 *     bytes past product_len are ignored; product_len <= 64;
 *   - bdf: the bytes before its first NUL (all 16 when there is none), 1..16 of them, over [0-9a-f:.];
 *   - pcie_root: empty (first byte NUL), or "pci" followed by 1..13 bytes over [0-9a-f:] before its first NUL;
 *   - vendor, device: 1..6 bytes over [0-9a-f] before the first NUL;
 *   - iommu_group below 4294967295.
 * GPU: one CTA per slice.  One thread per device computes its fragment length, a block scan places the devices in
 * the slice, the slice's offset is the exclusive prefix of a decoupled look-back over the slice totals (which is
 * slice_off[s]), and the slice is staged in shared memory at its destination's 16-byte phase and written with one
 * bulk store.  The header and tail, the same for every slice, are built on the host once per call.  Timed under
 * KXPU_T_EMIT. */
int32_t kxpu_dra_slices(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                        const kxpu_dradev *devs, size_t n, uint8_t *out, size_t cap, size_t *len,
                        uint64_t *slice_off /* [n_slices+1] */, size_t *n_slices);

/* ------------------------------------------- DRA ResourceSlices of vGPUs (ABI v10) */

/* One published vGPU (one IOMMU group of one vGPU class, described by its first mdev).  208 bytes, a multiple of 16;
 * alignof 8.  No new fact about the Kubernetes API is used: the [assumed] list above covers this call too. */
typedef struct kxpu_dramdev {
    uint8_t  product[64];   /* the PARENT's productName bytes, NUL padded                                    */
    char     mdev_type[40]; /* the type key of kxpu_classify_mdev, NUL padded                                */
    char     uuid[36];      /* the mdev's UUID                                                               */
    uint32_t iommu_group;
    char     parent[16];    /* parent PCI address                                                            */
    char     pcie_root[16]; /* "pci<domain>:<bus>", the first component of the mdev entry's link; "" = unknown */
    char     vendor[8];     /* the parent's vendor id, NUL padded                                            */
    char     device[8];     /* the parent's device id; "" = not read                                         */
    uint64_t numa_mask;     /* the group's NUMA mask (kxpu_classify_mdev_topo)                               */
    uint8_t  product_len;   /* 0..64                                                                         */
    uint8_t  reserved[7];
} kxpu_dramdev;

/* The ResourceSlices of one pool of vGPUs.  Everything but the device is kxpu_dra_slices' contract, unchanged: the
 * slices, their header and tail, 128 devices per slice and one empty slice for n = 0, slice_off, the two-call sizing
 * and KXPU_E_NOSPACE, the KXPU_E_INVALID argument checks, KXPU_DRA_MAX_DEVICES, and nothing written on KXPU_E_INVALID
 * or KXPU_E_UNSUPPORTED.  A device is
 *   {"name":"vfio<g>","attributes":{<attributes>}}
 * with g = iommu_group in decimal (it mirrors the cdi.k8s.io/vfio<g> annotation of the mdev CDI spec), and the
 * attributes, keys sorted bytewise:
 *   "iommuGroup":{"int":<g>}                                          always
 *   "mdevType":{"string":"<mdev_type>"}                               always
 *   "numaNode":{"int":<k>}                                            only when numa_mask has exactly one bit k set
 *   "parentAddress":{"string":"<parent>"}                             always
 *   "parentDeviceID":{"string":"<device>"}                            only when device is not empty
 *   "parentVendorID":{"string":"<vendor>"}                            always
 *   "productName":{"string":"<product[0..product_len)>"}              only when product_len > 0
 *   "resource.kubernetes.io/pcieRoot":{"string":"<pcie_root>"}        only when pcie_root is not empty
 *   "uuid":{"string":"<uuid>"}                                        always
 * KXPU_E_UNSUPPORTED, with *len, the output and slice_off untouched: n >= KXPU_DRA_MAX_DEVICES, or a record outside
 * the domain:
 *   - product[0..product_len) over [A-Za-z0-9_.-]; bytes past product_len are ignored; product_len <= 64;
 *   - mdev_type: 1..40 bytes over [A-Za-z0-9_.-] before its first NUL (all 40 when there is none);
 *   - uuid: the canonical lowercase 8-4-4-4-12 form;
 *   - parent: 1..16 bytes over [0-9a-f:.] before its first NUL;
 *   - pcie_root: empty, or "pci" followed by 1..13 bytes over [0-9a-f:] before its first NUL;
 *   - vendor: 1..6 bytes over [0-9a-f] before the first NUL; device: 0..6 such bytes;
 *   - iommu_group below 4294967295.
 * GPU: the kernel of kxpu_dra_slices, instantiated for this record layout.  Timed under KXPU_T_EMIT. */
int32_t kxpu_dra_slices_mdev(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                             const kxpu_dramdev *devs, size_t n, uint8_t *out, size_t cap, size_t *len,
                             uint64_t *slice_off /* [n_slices+1] */, size_t *n_slices);

/* ------------------------------------------- DRA device taints (ABI v11) */

/* A device that must not be allocated is published with a taint (KEP-5055), the DRA counterpart of ListAndWatch's
 * Unhealthy.  These facts refine the list above; the "no per-device health" line there holds for the v9 / v10 calls,
 * which never write taints:
 *   [assumed] v1 Device has taints []DeviceTaint, declared after attributes.  The fields declared between them
 *             (capacity, consumesCounters, nodeName, nodeSelector, allNodes) are never emitted here;
 *   [assumed] DeviceTaint is key, value, effect, timeAdded in that order; effect is NoSchedule or NoExecute; a device
 *             has at most 4 taints; the key is a qualified name and the value a label value;
 *   [assumed] taints take effect only with the DRADeviceTaints feature gate.  With the gate off the API server drops
 *             the field and the device looks untainted, which is what the v9 / v10 calls publish;
 *   [assumed] a slice in which any device has taints lists at most 64 devices. */
#define KXPU_DRA_TAINT_SLICE_DEVICES 64           /* devices per slice of the _taint calls with taint_since    */
#define KXPU_DRA_TAINT_SINCE_MAX     253402300799ll /* 9999-12-31T23:59:59Z                                     */

/* kxpu_dra_slices with at most one taint per device.  The contract is kxpu_dra_slices', with these additions:
 *   - taint_since == NULL: the output, *len, slice_off and *n_slices are byte for byte kxpu_dra_slices'; the taint
 *     arguments are not read.
 *   - taint_since[i] < 0: device i has no taint.
 *   - 0 <= taint_since[i] <= KXPU_DRA_TAINT_SINCE_MAX: device i carries one taint, a member after "attributes":
 *       {"name":"vfio<g>","attributes":{...},"taints":[{"key":"<key>","value":"<value>","effect":"<effect>",
 *        "timeAdded":"<YYYY-MM-DDTHH:MM:SSZ>"}]}
 *     "value" is left out when taint_value is empty; timeAdded is taint_since[i] as RFC 3339 in UTC with whole
 *     seconds, as metav1.Time marshals.
 *   - With taint_since != NULL a slice holds at most KXPU_DRA_TAINT_SLICE_DEVICES devices: S = max(1, ceil(n / 64)),
 *     also when no device is tainted, so the slice layout does not move when a device's health flips.
 * KXPU_E_INVALID, nothing written: the checks of kxpu_dra_slices, and with taint_since != NULL: taint_key not a
 * qualified name of at most 127 bytes (an optional lowercase DNS subdomain and '/', then a name of 1..63 bytes that
 * starts and ends with [A-Za-z0-9] and holds [-A-Za-z0-9_.] between; 127 is this project's bound); taint_value NULL, or
 * not empty and not such a name of at most 63 bytes; taint_effect not exactly "NoSchedule" or "NoExecute".
 * KXPU_E_UNSUPPORTED, nothing written: the cases of kxpu_dra_slices, or a taint_since[i] above
 * KXPU_DRA_TAINT_SINCE_MAX.
 * GPU: kxpu_dra_slices_taints with this taint as a one-entry table: the kernel of kxpu_dra_slices with a taint list
 * of one entry compiled in, one CTA per 64-device slice; the thread of a device range-checks its taint_since and
 * formats timeAdded into shared memory.  Timed under KXPU_T_EMIT. */
int32_t kxpu_dra_slices_taint(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                              const kxpu_dradev *devs, size_t n, const char *taint_key, const char *taint_value,
                              const char *taint_effect, const int64_t *taint_since /* [n] or NULL */, uint8_t *out,
                              size_t cap, size_t *len, uint64_t *slice_off /* [n_slices+1] */, size_t *n_slices);
/* The same for a pool of vGPUs: kxpu_dra_slices_mdev's devices with kxpu_dra_slices_taint's taints, slices and checks;
 * taint_since == NULL gives kxpu_dra_slices_mdev's bytes. */
int32_t kxpu_dra_slices_mdev_taint(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node,
                                   uint64_t generation, const kxpu_dramdev *devs, size_t n, const char *taint_key,
                                   const char *taint_value, const char *taint_effect,
                                   const int64_t *taint_since /* [n] or NULL */, uint8_t *out, size_t cap, size_t *len,
                                   uint64_t *slice_off /* [n_slices+1] */, size_t *n_slices);

/* ------------------------------------------- PCIe AER health and several taints per device (ABI v12) */

/* The uncorrectable PCIe errors a function has reported (Documentation/ABI/testing/sysfs-bus-pci-devices-aer_stats):
 *   [assumed] /sys/bus/pci/devices/<bdf>/aer_dev_fatal and aer_dev_nonfatal exist since Linux 4.19;
 *   [assumed] they exist only on functions that have an AER capability;
 *   [assumed] each line is "<name> <count>", and a name may contain spaces;
 *   [assumed] the total is the line "TOTAL_ERR_FATAL <n>" (aer_dev_fatal) or "TOTAL_ERR_NONFATAL <n>" (aer_dev_nonfatal);
 *   [assumed] on firmware-first platforms the OS does not handle AER, and the counters may never move. */
#define KXPU_AER_FATAL    1u  /* some member's known fatal count is above fatal_limit        */
#define KXPU_AER_NONFATAL 2u  /* some member's known non-fatal count is above nonfatal_limit */
#define KXPU_AER_UNKNOWN  4u  /* some member has an unknown count                            */
#define KXPU_AER_FILE_MAX 4096 /* a longer file gives an unknown count                       */

/* The AER counts of n records, folded per group.  Record i has two files: its fatal file is
 * text[file_off[2i], +file_len[2i]) and its non-fatal file is entry 2i+1.  Files may share bytes (a vGPU uses its
 * parent's files).  The count of a file:
 *   - the last line of the file that begins with "TOTAL_ERR_FATAL " (fatal file) or "TOTAL_ERR_NONFATAL " (non-fatal
 *     file), the space included;
 *   - what follows the prefix, up to '\n' or the end of the file, is a canonical decimal: 1 to 20 digits, no leading
 *     zero except "0" itself, value below 2^64 - 1;
 *   - anything else makes the count UNKNOWN, never an error (like numa_node): no such line, a '\r', a bad number,
 *     file_len == 0 (the host's failed read) or file_len > KXPU_AER_FILE_MAX.
 * totals (may be NULL): totals[2i] / totals[2i+1] = the fatal / non-fatal count of record i, UINT64_MAX when unknown.
 * group_aer[o], over the members group_members[group_off[o] .. group_off[o+1]) of group o: KXPU_AER_FATAL when some
 * member's known fatal count is greater than fatal_limit, KXPU_AER_NONFATAL the same for the non-fatal count and
 * nonfatal_limit, KXPU_AER_UNKNOWN when some member has an unknown count.  A group without members gets 0.
 * KXPU_E_INVALID, nothing written: ctx NULL, text NULL with text_len > 0, file_off / file_len NULL with n > 0,
 * group_off NULL, group_members NULL with members, group_aer NULL with n_groups > 0; a file range outside text_len;
 * group_off decreasing; a member >= n.
 * Limit (else KXPU_E_UNSUPPORTED): n and n_groups below 2^28.
 * GPU: one warp per file reads its tail backward in 32-byte windows: a ballot finds the line starts, each starting lane
 * tests the prefix and parses its number, and the highest match decides; then one warp per group ORs its members'
 * bits.  Timed under KXPU_T_CLASSIFY. */
int32_t kxpu_aer_health(kxpu_ctx *ctx, const uint8_t *text, size_t text_len, const uint64_t *file_off /* [2n] */,
                        const uint32_t *file_len /* [2n] */, size_t n, uint64_t fatal_limit, uint64_t nonfatal_limit,
                        const uint32_t *group_off /* [n_groups+1] */, const uint32_t *group_members, size_t n_groups,
                        uint64_t *totals /* [2n] or NULL */, uint8_t *group_aer /* [n_groups] */);

/* Several taints per device: a table of up to KXPU_DRA_MAX_TAINTS entries, each with the _taint calls' key, value and
 * effect rules.
 *   [assumed] the API rejects a device that carries two taints with the same key and effect. */
typedef struct kxpu_dra_taint {
    const char *key, *value, *effect;
} kxpu_dra_taint;
#define KXPU_DRA_MAX_TAINTS 4

/* kxpu_dra_slices_taint with a table of n_taints taints.  The contract is kxpu_dra_slices_taint's, with these changes:
 *   - taint_since == NULL: the output, *len, slice_off and *n_slices are byte for byte kxpu_dra_slices'; the taint
 *     arguments are not read.
 *   - taint_since[i * n_taints + t] < 0: device i does not carry taint t; 0 .. KXPU_DRA_TAINT_SINCE_MAX: it carries
 *     taint t with that timeAdded.
 *   - a device that carries some taint gets "taints":[{...},{...}], its taints in table order, each written as the
 *     _taint call writes its one taint ("value" left out when empty).  n_taints == 1 gives kxpu_dra_slices_taint's bytes
 *     for that key, value and effect.
 *   - with taint_since != NULL a slice holds at most KXPU_DRA_TAINT_SLICE_DEVICES devices.
 * KXPU_E_INVALID, nothing written: the checks of kxpu_dra_slices, and with taint_since != NULL: taints NULL, n_taints 0
 * or above KXPU_DRA_MAX_TAINTS, or an entry whose key, value or effect fails kxpu_dra_slices_taint's checks.
 * KXPU_E_UNSUPPORTED, nothing written: the cases of kxpu_dra_slices, a taint_since above KXPU_DRA_TAINT_SINCE_MAX, or a
 * device that carries two entries with the same key and effect.
 * GPU: the kernel of kxpu_dra_slices with the taint list compiled in, its shared memory sized for the table's capacity:
 * one entry for n_taints == 1, KXPU_DRA_MAX_TAINTS for more.  Timed under KXPU_T_EMIT. */
int32_t kxpu_dra_slices_taints(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                               const kxpu_dradev *devs, size_t n, const kxpu_dra_taint *taints, size_t n_taints,
                               const int64_t *taint_since /* [n * n_taints], device-major, or NULL */, uint8_t *out,
                               size_t cap, size_t *len, uint64_t *slice_off /* [n_slices+1] */, size_t *n_slices);
/* The same for a pool of vGPUs: taint_since == NULL gives kxpu_dra_slices_mdev's bytes, n_taints == 1
 * kxpu_dra_slices_mdev_taint's. */
int32_t kxpu_dra_slices_mdev_taints(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node,
                                    uint64_t generation, const kxpu_dramdev *devs, size_t n, const kxpu_dra_taint *taints,
                                    size_t n_taints, const int64_t *taint_since /* [n * n_taints] or NULL */, uint8_t *out,
                                    size_t cap, size_t *len, uint64_t *slice_off /* [n_slices+1] */, size_t *n_slices);

#ifdef __cplusplus
}
#endif
#endif /* KXPU_H */
