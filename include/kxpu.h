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

#define KXPU_ABI_VERSION 2

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
#define KXPU_T_LOOKUP   2
#define KXPU_T_NAMES    3
#define KXPU_T_CLASSIFY 4
#define KXPU_T_EMIT     5
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
    uint8_t  reserved0;
    uint32_t reserved1[2];
} kxpu_devrec;

#define KXPU_REC_VENDOR_ERR 0x01u /* readIDFromFile(vendor) failed  (device_plugin.go:143) */
#define KXPU_REC_DRIVER_ERR 0x02u /* readLink(driver) failed        (device_plugin.go:152) */
#define KXPU_REC_IOMMU_ERR  0x04u /* readLink(iommu_group) failed   (device_plugin.go:158) */
#define KXPU_REC_DEVICE_ERR 0x08u /* readIDFromFile(device) failed  (device_plugin.go:165) */
#define KXPU_REC_IS_DIR     0x10u /* info.IsDir()                   (device_plugin.go:137) */

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

/* ------------------------------------------------------- S3: CDI spec emit */

/* One accepted device as generateCDISpec sees it (device_plugin.go:59-76). 32 bytes. */
typedef struct kxpu_cdidev {
    char     bdf[16];       /* dev.addr, NUL padded                                       */
    uint32_t iommu_group;   /* devName (decimal)                                          */
    uint32_t reserved;
    uint64_t index;         /* dev.index                                                  */
} kxpu_cdidev;

#define KXPU_FMT_YAML 0  /* yaml.v3 encoder, SetIndent(2)   (cdi/spec.go:104-112)          */
#define KXPU_FMT_JSON 1  /* json.MarshalIndent(spec,"","  ") (cdi/spec.go:114-123)         */

/* generateCDISpec + CdiSpec.Save (device_plugin.go:55-80, cdi/spec.go:85-127) into a
 * caller buffer; devices are emitted in array order (canonical order: ascending index).
 * Call with out==NULL/cap==0 to obtain *len.  The host writes the file. */
int32_t kxpu_cdi_emit(kxpu_ctx *ctx, int32_t format, const kxpu_cdidev *devs, size_t n,
                      uint8_t *out, size_t cap, size_t *len);

/* ------------------------------------------------------ S5: Allocate names */

/* updateResponseForCDI / QualifiedName (generic_device_plugin.go:274-299,
 * cdi/cdi-utils.go:9): name i = "nvidia.com/gpu=" + decimal(idx[i]). */
int32_t kxpu_alloc_names(kxpu_ctx *ctx, const uint64_t *idx, size_t n, uint8_t *out,
                         size_t cap, uint32_t *offsets, size_t *need);

/* ListAndWatchResponse wire bytes for a device list (generic_device_plugin.go:224):
 * repeated field 1 { string ID = 1 (decimal group); string health = 2 }.
 * healthy[i] != 0 -> "Healthy" else "Unhealthy"; healthy == NULL -> all healthy. */
int32_t kxpu_lw_encode(kxpu_ctx *ctx, const uint32_t *group_ids, const uint8_t *healthy,
                       size_t n, uint8_t *out, size_t cap, size_t *len);

#ifdef __cplusplus
}
#endif
#endif /* KXPU_H */
