// comm.cu -- multi-GPU pci.ids load + join: one rank per GPU (one process per rank, or one
// process driving all ranks through kxpu_ctx_create_multi), shards cut at vendor-line boundaries.
//
// BASELINE.json configs[3] / SURVEY.md 8(e).  Every rank parses its byte range of one logical
// text with GLOBAL offsets, which yields for every (vendor,device) key the earliest candidate
// line of the shard and for every vendor prefix its earliest anchor.  "First anchor wins"
// (device_plugin.go:263-267) is then decided across shards in two exchange phases:
//
//   A  all-reduce(min) of vendor_first (+ the bufio.ErrTooLong cut-off and status bits), done as an
//      all-gather with the min taken by the reader (pushed by extra CTAs of resolve_chunks_kernel while the others
//      fold -- vendor_first is final since the parse kernel): every rank stores
//      its dense first-anchor array
//      (512 KB, plain 16-byte stores over NVLink -- remote 64-bit atomics cost ~10 ns apiece, the
//      copy is one streaming write) into ITS block of every rank's exchange region; nothing is ever
//      cleared, the block is overwritten whole each epoch.  After phase A every rank knows the
//      global first anchor of every vendor id (min over the R blocks), so a row is a WINNER iff
//      its anchor equals it -- and winners are globally unique per key (the first block sits in
//      exactly one shard).
//   B  winners only, as a PULL: each rank sanitises the names of its winner rows straight into its own slab
//      (finalize kernel); the last CTA of that kernel writes the slab header and raises "slab ready" on every
//      rank.  Shards that hold no first block publish an empty slab.  Every rank's merge kernel then reads the
//      slabs of all ranks over NVLink (uncached loads) and inserts the winners into the table it parsed into
//      -- no second table, no min-merge, row handles are global (rank prefix + index).  (Until round 2 a push
//      kernel copied the slab into every peer: the same step time -- the cost is the fence + flag latency at
//      the phase boundary, not the copy -- but one kernel and R slab copies more.)
//   C  (join) every rank probes its slice of the keys and stores each result into every rank's
//      result buffer: the all-gather of hits rides on the probe kernel.
//
// A phase boundary is a flag per (phase, buffer, rank) in every region, raised by the last CTA
// of the producing kernel after a system fence, and a wait in the prologue of the consumer kernel (a
// one-warp wait kernel when several contexts share a GPU).  Two buffers alternate by epoch: a rank
// can only start epoch e + 2 after every peer delivered e + 1, i.e. finished reading epoch e.
// The epoch is bumped before anything can fail, statuses travel WITH the data (min-encoded words
// in phase A, slab headers in phase B), so every rank takes the same retry decision; a time-out
// or a CUDA error marks the exchange broken (re-init required).
//
// Transports: peer memory (CUDA IPC mappings across processes, direct pointers inside one
// process) is the product path; NCCL (ncclAllGather for every phase, loaded lazily with
// dlopen) runs the same kernels against a local staging region when peer mapping is impossible
// (KXPU_NO_P2P=1 forces it) or a slab outgrows the fixed peer region.
#include <dlfcn.h>

#include <algorithm>
#include <new>

#include "exchange.cuh"
#include "internal.cuh"
#include "parse_common.cuh"

namespace kxx {

// ------------------------------------------------------------------ NCCL (lazy)
typedef int (*fn_get_unique_id)(void *);
typedef int (*fn_comm_destroy)(void *);
typedef int (*fn_all_gather)(const void *, void *, size_t, int, void *, cudaStream_t);
typedef const char *(*fn_err_string)(int);
struct UniqueId { char internal[128]; };
typedef int (*fn_comm_init_rank)(void **, int, UniqueId, int);  // ncclUniqueId is passed by value (128 bytes)

struct NcclApi {
    void *handle = nullptr;
    fn_get_unique_id get_unique_id = nullptr;
    fn_comm_init_rank comm_init_rank = nullptr;
    fn_comm_destroy comm_destroy = nullptr;
    fn_all_gather all_gather = nullptr;
    fn_err_string err_string = nullptr;
};
static NcclApi g_nccl;
static std::mutex g_nccl_mu;
constexpr int NCCL_UINT8 = 1;

static bool nccl_load() {
    std::lock_guard<std::mutex> g(g_nccl_mu);
    if (g_nccl.handle) return true;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    void *h = nullptr;
    for (const char *nm : names) {
        h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
        if (h) break;
    }
    if (!h) return false;
    g_nccl.get_unique_id = (fn_get_unique_id)dlsym(h, "ncclGetUniqueId");
    g_nccl.comm_init_rank = (fn_comm_init_rank)dlsym(h, "ncclCommInitRank");
    g_nccl.comm_destroy = (fn_comm_destroy)dlsym(h, "ncclCommDestroy");
    g_nccl.all_gather = (fn_all_gather)dlsym(h, "ncclAllGather");
    g_nccl.err_string = (fn_err_string)dlsym(h, "ncclGetErrorString");
    if (!g_nccl.get_unique_id || !g_nccl.comm_init_rank || !g_nccl.comm_destroy || !g_nccl.all_gather) return false;
    g_nccl.handle = h;
    return true;
}

// ------------------------------------------------------------------ exchange region
constexpr size_t FLAGS_BYTES = 1024;  // u32 flag[3 phases][2 buffers][KX_MAX_RANKS]

struct XCaps { uint32_t rows, blob, join; };  // per-rank slab rows / name bytes, keys of one sharded join

struct XLayout {
    size_t o_a[2], a_stride, o_slab[2], slab_stride, o_res[2], total;  // o_a[b]: phase-A block of rank 0, rank r at + r * a_stride
};
__host__ __device__ static inline size_t x_align(size_t x) { return (x + 255) / 256 * 256; }
static XLayout x_layout(const XCaps &c, int R) {
    XLayout L;
    size_t off = FLAGS_BYTES;
    L.a_stride = x_align((size_t)A_WORDS * 8);
    for (int b = 0; b < 2; b++) { L.o_a[b] = off; off += (size_t)R * L.a_stride; }
    L.slab_stride = x_align(sizeof(SlabHeader) + (size_t)c.rows * sizeof(SlabRow) + c.blob + 16);
    for (int b = 0; b < 2; b++) { L.o_slab[b] = off; off += (size_t)R * L.slab_stride; }
    for (int b = 0; b < 2; b++) { L.o_res[b] = off; off = x_align(off + (size_t)c.join * 4); }
    L.total = off;
    return L;
}
__host__ __device__ static inline size_t slab_rows_off() { return sizeof(SlabHeader); }
__host__ __device__ static inline size_t slab_blob_off(uint32_t rows_cap) { return sizeof(SlabHeader) + (size_t)rows_cap * sizeof(SlabRow); }
__host__ __device__ static inline size_t flag_off(int phase, int b, int rank) { return (size_t)((phase * 2 + b) * KX_MAX_RANKS + rank) * 4; }

static const XCaps kPeerCaps{65536u, 2u << 20, 1u << 21};

}  // namespace kxx

struct KxExchange {
    int nranks = 1, rank = 0;
    bool p2p = false;     // peer-memory transport available
    bool ipc = false;     // peers mapped through CUDA IPC (else direct pointers of this process)
    bool broken = false;  // a time-out / CUDA error desynchronised the ranks: re-init required
    bool use_nccl = false;  // transport of the current/next attempt
    bool fuse_waits = false;  // every rank has its own GPU: consumer kernels wait for the flags in their prologue
    uint8_t *local = nullptr;
    uint8_t *peer[KX_MAX_RANKS] = {};
    kxx::XLayout L{};
    kxx::XCaps caps{};
    uint32_t epoch = 0;
    uint32_t *scratch = nullptr;  // device: [0..2] last-CTA counters of the three pushing kernels, [8] time-out flag
    // uniform across ranks (only changed by decisions every rank takes alike)
    uint32_t x_cap = 1u << 16, x_blob_cap = 4u << 20;
    // NCCL transport: staging region with the same layout (R slabs contiguous = all-gather target)
    uint8_t *stage = nullptr;
    uint8_t *send_slab = nullptr;
    kxx::XLayout SL{};
    kxx::XCaps scaps{};
};

namespace kxx {

// ------------------------------------------------------------------ kernels
// one warp: lane q waits for rank q's flag of this epoch (used when the wait cannot ride on the
// consumer kernel: several contexts share one GPU and many spinning CTAs could starve the peers)
__global__ void wait_flags_kernel(const WaitSpec W) { wait_flags_lane(W, (int)threadIdx.x); }

// keys a table may hold after the merge: the bound (winners + the most losers any rank keeps) is the
// same on every rank and usually counts the winners' keys twice, so it may go well beyond the 50 %
// load the parse is held to
__host__ __device__ static inline uint32_t merged_key_limit(uint32_t cap) { return cap - cap / 8; }

struct MergeParams {
    const uint8_t *slab_of[KX_MAX_RANKS];  // rank r's slab: peer memory (read over NVLink) or the all-gathered staging copy
    int R;
    uint32_t slab_rows_cap;
    MinView mv;  // the phase-A blocks of all ranks (status words)
    KxTableDev tab;
    uint32_t *row_key, *row_name_off, *row_name_len;
    unsigned long long *row_line, *row_anchor;
    uint8_t *blob;
    uint32_t rows_cap, blob_cap;
    const uint32_t *timeout_flag;
    WaitSpec wait;
};

// The winners of all ranks go into the table this rank parsed into: row arrays and names at their
// global positions (rank prefix + index), key -> global row handle in the hash.  Winners are unique
// per key, so this is an insert, not a min-merge.  Every rank computes the same summary
// (KX_C_X*) from the same headers and takes the same retry decision from it.
__global__ void __launch_bounds__(256) merge_kernel(const MergeParams P) {
    __shared__ uint32_t rpre[KX_MAX_RANKS + 1], bpre[KX_MAX_RANKS + 1], s_status, s_maxkeys;
    wait_flags_cta(P.wait);
    // the R headers: one lane each (remote reads, all in flight together)
    __shared__ uint32_t h_rows[KX_MAX_RANKS], h_blob[KX_MAX_RANKS], h_status[KX_MAX_RANKS], h_nkeys[KX_MAX_RANKS];
    if (threadIdx.x < (unsigned)P.R) {
        const uint4 hv = __ldcv(reinterpret_cast<const uint4 *>(P.slab_of[threadIdx.x]));  // n_rows, blob_bytes, status, nkeys
        h_rows[threadIdx.x] = hv.x; h_blob[threadIdx.x] = hv.y; h_status[threadIdx.x] = hv.z; h_nkeys[threadIdx.x] = hv.w;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t st = min_view_status(P.mv), mk = 0, racc = 0, bacc = 0;
        for (int r = 0; r < P.R; r++) {
            rpre[r] = racc; bpre[r] = bacc;
            racc += h_rows[r];
            bacc += (h_blob[r] + 15u) & ~15u;
            st |= h_status[r];
            const uint32_t losers = h_nkeys[r] > h_rows[r] ? h_nkeys[r] - h_rows[r] : 0u;  // local keys that are not winners
            mk = losers > mk ? losers : mk;
        }
        rpre[P.R] = racc; bpre[P.R] = bacc;
        if (P.timeout_flag && *P.timeout_flag) st |= 0x80000000u;
        s_status = st; s_maxkeys = mk;
        if (blockIdx.x == 0) {
            P.tab.counters[KX_C_XSTATUS] = st;
            P.tab.counters[KX_C_XROWS] = racc;
            P.tab.counters[KX_C_XBLOB] = bacc;
            P.tab.counters[KX_C_XMAXKEYS] = mk;
        }
    }
    __syncthreads();
    const uint32_t total_rows = rpre[P.R], total_b16 = bpre[P.R] / 16u;
    // uniform on every rank: table capacities are kept equal across ranks (KxExchange::x_cap)
    if (s_status != 0u || total_rows > P.rows_cap || bpre[P.R] > P.blob_cap || total_rows + s_maxkeys > merged_key_limit(P.tab.cap)) return;
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
    uint32_t nfresh = 0;
    for (size_t g = tid; g < total_rows; g += nth) {
        int r = 0;
        while (r + 1 < P.R && g >= rpre[r + 1]) r++;
        // a 32-byte row in two uncached 16-byte loads (peer memory: never out of a stale cache line)
        const uint4 *rp = reinterpret_cast<const uint4 *>(P.slab_of[r] + slab_rows_off()) + 2 * (size_t)(g - rpre[r]);
        const uint4 ra = __ldcv(rp), rb = __ldcv(rp + 1);
        SlabRow row;
        row.key = ra.x; row.name_len = ra.y; row.line = ((unsigned long long)ra.w << 32) | ra.z;
        row.anchor = ((unsigned long long)rb.y << 32) | rb.x; row.name_off = rb.z; row.pad = rb.w;
        P.row_key[g] = row.key; P.row_line[g] = row.line; P.row_anchor[g] = row.anchor;
        P.row_name_off[g] = bpre[r] + row.name_off; P.row_name_len[g] = row.name_len;
        const uint32_t slot = kxparse::table_claim(P.tab, row.key, nfresh);
        if (slot != 0xffffffffu) P.tab.slots[slot].row = (int32_t)g;
    }
    if (nfresh) atomicAdd(&P.tab.counters[KX_C_NKEYS], nfresh);
    for (size_t j = tid; j < total_b16; j += nth) {
        int r = 0;
        while (r + 1 < P.R && j * 16u >= bpre[r + 1]) r++;
        const uint8_t *src = P.slab_of[r] + slab_blob_off(P.slab_rows_cap);
        reinterpret_cast<uint4 *>(P.blob)[j] = __ldcv(reinterpret_cast<const uint4 *>(src) + (j - bpre[r] / 16u));
    }
}

// rows that lost (their anchor is not the global first one) keep a handle from the local finalize
// only if they were selected, and selection already used the global minima: nothing to undo.

struct JoinParams {
    const uint32_t *keys;
    size_t n, key_offset;
    const KxSlot *slots;
    uint32_t cap, shift;
    Targets tg;
    size_t o_res, o_flag;
    int raise_flags;
    uint32_t epoch;
    uint32_t *done;
};

// Phase C: probe this rank's key slice; a CTA stages its 1024 hits in shared memory and warp w
// streams the block into the result buffer of rank w, w + 8, ... (512 contiguous bytes per store
// instruction over NVLink) -- probe and all-gather of hits in one kernel.  key_offset is a multiple
// of 4 (16-byte alignment of every block) or the scalar tail path is used.
constexpr int JOIN_PER_CTA = 1024;
__global__ void __launch_bounds__(256) join_gather_kernel(const JoinParams P) {
    __shared__ __align__(16) int32_t res[JOIN_PER_CTA];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    for (size_t b0 = (size_t)blockIdx.x * JOIN_PER_CTA; b0 < P.n; b0 += (size_t)gridDim.x * JOIN_PER_CTA) {
        const uint32_t cnt = P.n - b0 < (size_t)JOIN_PER_CTA ? (uint32_t)(P.n - b0) : (uint32_t)JOIN_PER_CTA;
        {
            static_assert(JOIN_PER_CTA == 4 * 256, "four keys per thread");
            uint32_t key[4] = {0u, 0u, 0u, 0u}, on = 0;
            int32_t row[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t j = tid + 256u * k;
                if (j < cnt) { key[k] = P.keys[b0 + j]; on |= 1u << k; }
            }
            kxparse::table_probe4(P.slots, P.cap, P.shift, key, on, row);  // the four probes of a thread run side by side
#pragma unroll
            for (int k = 0; k < 4; k++)
                if ((on >> k) & 1u) res[tid + 256u * k] = row[k];
        }
        __syncthreads();
        const size_t o = P.key_offset + b0;
        for (int q = (int)w; q < P.tg.n; q += 8) {
            int32_t *dst = reinterpret_cast<int32_t *>(P.tg.region[q] + P.o_res) + o;
            if (cnt == (uint32_t)JOIN_PER_CTA && (o & 3u) == 0u) {
#pragma unroll
                for (int k = 0; k < JOIN_PER_CTA / 128; k++)
                    reinterpret_cast<uint4 *>(dst)[lane + 32 * k] = reinterpret_cast<const uint4 *>(res)[lane + 32 * k];
            } else {
                for (uint32_t j = lane; j < cnt; j += 32u) dst[j] = res[j];
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        kx_fence_sys();
        const uint32_t prev = atomicAdd(P.done, 1u);
        if (prev == gridDim.x - 1u) {
            *P.done = 0u;
            kx_fence_sys();
            if (P.raise_flags)
                for (int q = 0; q < P.tg.n; q++) *reinterpret_cast<volatile uint32_t *>(P.tg.region[q] + P.o_flag) = P.epoch;
        }
    }
}

// everybody's hits have landed in my result buffer: hand them to the caller's buffer
__global__ void __launch_bounds__(256) gather_copy_kernel(const WaitSpec W, const uint4 *src, uint4 *dst, size_t n16, const int32_t *src_tail,
                                                          int32_t *dst_tail, uint32_t n_tail) {
    wait_flags_cta(W);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) dst[i] = src[i];
    if (blockIdx.x == 0 && threadIdx.x < n_tail) dst_tail[threadIdx.x] = src_tail[threadIdx.x];
}

// ------------------------------------------------------------------ region set-up
static int32_t region_alloc(kxpu_ctx *ctx, KxExchange *x, const XCaps &caps) {
    x->caps = caps;
    x->L = x_layout(caps, x->nranks);
    if (cudaMalloc((void **)&x->local, x->L.total) != cudaSuccess) { cudaGetLastError(); x->local = nullptr; return KXPU_E_NOMEM; }
    bool ok = cudaMemsetAsync(x->local, 0, FLAGS_BYTES, ctx->stream) == cudaSuccess;
    ok = ok && cudaMalloc((void **)&x->scratch, 256) == cudaSuccess && cudaMemsetAsync(x->scratch, 0, 256, ctx->stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(ctx->stream) == cudaSuccess;
    if (!ok) { cudaGetLastError(); return KXPU_E_CUDA; }
    return KXPU_OK;
}

static void exchange_free(kxpu_ctx *ctx) {
    KxExchange *x = ctx->xch;
    if (!x) return;
    cudaSetDevice(ctx->device);
    if (x->ipc)
        for (int q = 0; q < x->nranks; q++)
            if (q != x->rank && x->peer[q]) cudaIpcCloseMemHandle(x->peer[q]);
    if (x->local) cudaFree(x->local);
    if (x->scratch) cudaFree(x->scratch);
    if (x->stage) cudaFree(x->stage);
    if (x->send_slab) cudaFree(x->send_slab);
    cudaGetLastError();
    delete x;
    ctx->xch = nullptr;
}

// Map every peer's exchange region through CUDA IPC (one process per rank).  Any failure leaves
// p2p false on EVERY rank (the ranks agree through one more tiny all-gather): NCCL transport.
static void ipc_setup(kxpu_ctx *ctx, KxExchange *x) {
    x->p2p = false;
    const int R = x->nranks;
    if (R < 2 || R > KX_MAX_RANKS || getenv("KXPU_NO_P2P")) return;
    bool ok = region_alloc(ctx, x, kPeerCaps) == KXPU_OK;
    cudaIpcMemHandle_t mine, all[KX_MAX_RANKS];
    memset(&mine, 0, sizeof mine);
    ok = ok && cudaIpcGetMemHandle(&mine, x->local) == cudaSuccess;
    const size_t hb = sizeof(cudaIpcMemHandle_t);
    uint8_t *d_x = nullptr;
    if (cudaMalloc((void **)&d_x, hb * (size_t)(R + 1) + 64) != cudaSuccess) { d_x = nullptr; ok = false; }
    uint8_t okbyte[KX_MAX_RANKS + 1] = {};
    if (d_x) {  // exchange the handles with the communicator that exists already
        cudaMemcpyAsync(d_x, &mine, hb, cudaMemcpyHostToDevice, ctx->stream);
        const int nrc = g_nccl.all_gather(d_x, d_x + hb, hb, NCCL_UINT8, ctx->nccl_comm, ctx->stream);
        cudaMemcpyAsync(all, d_x + hb, hb * (size_t)R, cudaMemcpyDeviceToHost, ctx->stream);
        if (nrc != 0 || cudaStreamSynchronize(ctx->stream) != cudaSuccess) ok = false;
    }
    bool opened[KX_MAX_RANKS] = {};
    if (ok) {
        for (int q = 0; q < R && ok; q++) {
            if (q == x->rank) { x->peer[q] = x->local; continue; }
            void *pp = nullptr;
            if (cudaIpcOpenMemHandle(&pp, all[q], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = false; cudaGetLastError(); break; }
            x->peer[q] = (uint8_t *)pp;
            opened[q] = true;
        }
    }
    if (d_x) {  // agreement: all ranks or none
        const uint8_t mineok = ok ? 1 : 0;
        uint8_t *d_ok = d_x + hb * (size_t)(R + 1);
        cudaMemcpyAsync(d_ok, &mineok, 1, cudaMemcpyHostToDevice, ctx->stream);
        const int nrc = g_nccl.all_gather(d_ok, d_ok + 16, 1, NCCL_UINT8, ctx->nccl_comm, ctx->stream);
        cudaMemcpyAsync(okbyte, d_ok + 16, (size_t)R, cudaMemcpyDeviceToHost, ctx->stream);
        if (nrc != 0 || cudaStreamSynchronize(ctx->stream) != cudaSuccess) ok = false;
        for (int q = 0; q < R; q++) ok = ok && okbyte[q] == 1;
        cudaFree(d_x);
    }
    if (!ok) {
        for (int q = 0; q < R; q++)
            if (opened[q]) cudaIpcCloseMemHandle(x->peer[q]);
        memset(x->peer, 0, sizeof x->peer);
        if (x->local) { cudaFree(x->local); x->local = nullptr; }
        if (x->scratch) { cudaFree(x->scratch); x->scratch = nullptr; }
        cudaGetLastError();
        if (getenv("KXPU_TRACE_MERGE")) fprintf(stderr, "[kxpu] rank %d: peer-memory exchange unavailable, using NCCL\n", x->rank);
        return;
    }
    x->ipc = true;
    x->p2p = true;
    x->fuse_waits = true;  // one process per rank, one GPU per process
    if (getenv("KXPU_TRACE_MERGE")) fprintf(stderr, "[kxpu] rank %d: peer-memory exchange over %d ranks, %zu B per rank\n", x->rank, R, x->L.total);
}

// NCCL transport: a staging region of the same layout whose R slabs form the all-gather target
static int32_t stage_reserve(kxpu_ctx *ctx, KxExchange *x, const XCaps &want) {
    if (x->stage && x->scaps.rows >= want.rows && x->scaps.blob >= want.blob) return KXPU_OK;
    cudaStreamSynchronize(ctx->stream);
    if (x->stage) { cudaFree(x->stage); x->stage = nullptr; }
    if (x->send_slab) { cudaFree(x->send_slab); x->send_slab = nullptr; }
    // zeroed on the ctx stream: the stream is non-blocking, so a legacy-stream cudaMemset would not be ordered
    // in front of the kernels that read these counters
    if (!x->scratch && (cudaMalloc((void **)&x->scratch, 256) != cudaSuccess ||
                        cudaMemsetAsync(x->scratch, 0, 256, ctx->stream) != cudaSuccess)) {
        cudaGetLastError();
        if (x->scratch) { cudaFree(x->scratch); x->scratch = nullptr; }
        return KXPU_E_NOMEM;
    }
    x->scaps = want;
    x->scaps.join = 0;
    x->SL = x_layout(x->scaps, x->nranks);
    if (cudaMalloc((void **)&x->stage, x->SL.total) != cudaSuccess || cudaMalloc((void **)&x->send_slab, x->SL.slab_stride) != cudaSuccess) {
        cudaGetLastError();
        KX_SET_ERR(ctx, "NCCL staging region (%zu B) could not be allocated", x->SL.total);
        return KXPU_E_NOMEM;
    }
    return KXPU_OK;
}

// ------------------------------------------------------------------ one sharded load (+ join)
struct ShardArgs {
    const uint8_t *d_text;
    size_t n;
    unsigned long long base;
    const uint32_t *d_keys;  // join slice of this rank (may be null)
    size_t nq, key_offset, nq_total;
    int32_t *d_rows_all;     // [nq_total] on this rank (may be null)
};

struct ShardOp {
    kxpu_ctx *ctx = nullptr;
    KxExchange *x = nullptr;
    ShardArgs a{};
    kxpu_table *t = nullptr;
    bool have_trunc = false;
    int b = 0;
    uint32_t epoch = 0;
    bool nccl = false;
    int32_t rc = KXPU_OK;  // first failure of an enqueue phase (the remaining phases are skipped)
};

// KXPU_TRACE_MERGE=1: device time between the enqueue points of one sharded load, averaged over 16 loads
struct PhaseTrace {
    static constexpr int N = 10;
    cudaEvent_t ev[N] = {};
    bool on = false, made = false;
    double acc[N] = {};
    int calls = 0;
    const char *name[N] = {"trunc", "parse+resolve+xa", "waitA", "select+finalize+tail", "-", "waitB", "merge (pull)", "join", "waitC+copy", ""};
    void init() {
        on = getenv("KXPU_TRACE_MERGE") != nullptr;
        if (on && !made) { for (auto &e : ev) cudaEventCreate(&e); made = true; }
    }
    void mark(int i, cudaStream_t s) { if (on) cudaEventRecord(ev[i], s); }
    void report(int rank, int nranks) {
        if (!on) return;
        for (int i = 0; i + 1 < N; i++) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, ev[i], ev[i + 1]) == cudaSuccess) acc[i] += ms;
        }
        cudaGetLastError();
        if (++calls % 16 == 0) {
            fprintf(stderr, "[kxpu shard trace] rank %d/%d:", rank, nranks);
            for (int i = 0; i + 1 < N; i++) fprintf(stderr, " %s %.1f us |", name[i], acc[i] / 16 * 1e3);
            fprintf(stderr, "\n");
            for (auto &a : acc) a = 0;
        }
    }
};
static thread_local PhaseTrace g_trace;

static Targets targets(const ShardOp &op) {
    Targets tg;
    memset(&tg, 0, sizeof tg);
    if (op.nccl) { tg.n = 1; tg.region[0] = op.x->stage; }
    else {
        tg.n = op.x->nranks;
        for (int q = 0; q < tg.n; q++) tg.region[q] = op.x->peer[q];
    }
    return tg;
}
static const XLayout &layout(const ShardOp &op) { return op.nccl ? op.x->SL : op.x->L; }
static uint8_t *my_region(const ShardOp &op) { return op.nccl ? op.x->stage : op.x->local; }

static void nccl_fail(ShardOp &op, const char *what, int nrc) {
    KX_SET_ERR(op.ctx, "%s: %s", what, g_nccl.err_string ? g_nccl.err_string(nrc) : "error");
    op.x->broken = true;
    op.rc = KXPU_E_NCCL;
}

// phase 1: acquire + parse + push of the shard's minima.  Nothing here waits for a peer.
static void shard_phase1(ShardOp &op) {
    kxpu_ctx *ctx = op.ctx;
    KxExchange *x = op.x;
    op.rc = KXPU_OK;
    op.t = nullptr;
    op.epoch = ++x->epoch;  // before anything can fail: the ranks stay in step
    op.nccl = x->use_nccl || !x->p2p;
    op.b = op.nccl ? 0 : (int)(op.epoch & 1u);
    if (x->broken) { KX_SET_ERR(ctx, "the exchange is broken (an earlier time-out or error): kxpu_comm_destroy + kxpu_comm_init"); op.rc = KXPU_E_NCCL; return; }
    if ((reinterpret_cast<uintptr_t>(op.a.d_text) & 15u) != 0) { KX_SET_ERR(ctx, "device text pointer must be 16-byte aligned"); op.rc = KXPU_E_INVALID; return; }
    if (op.a.base + op.a.n >= (1ull << 44)) { op.rc = KXPU_E_UNSUPPORTED; return; }
    if (op.nccl) {
        XCaps want{std::max<uint32_t>(x->x_cap, 65536u), std::max<uint32_t>(x->x_blob_cap / 2, 2u << 20), 0u};
        if (x->scaps.rows > want.rows) want.rows = x->scaps.rows;
        if (x->scaps.blob > want.blob) want.blob = x->scaps.blob;
        op.rc = stage_reserve(ctx, x, want);
        if (op.rc != KXPU_OK) return;
    }
    const uint32_t num_chunks = (uint32_t)((op.a.n + kxparse::CW - 1) / kxparse::CW);
    op.rc = kx_table_acquire(ctx, x->x_cap, x->x_blob_cap, num_chunks, &op.t);
    if (op.rc != KXPU_OK) return;
    kxpu_table *t = op.t;
    g_trace.init();
    g_trace.mark(0, ctx->stream);
    // exact bufio.ErrTooLong cut-off of the shard (second attempt only; independent of the parse)
    if (op.have_trunc) op.rc = kx_launch_trunc(ctx, t, op.a.d_text, op.a.n, op.a.base);
    if (op.rc != KXPU_OK) return;
    g_trace.mark(1, ctx->stream);
    // parse + resolve; extra CTAs of resolve_chunks_kernel push the shard's minima (phase A)
    const XLayout &L = layout(op);
    KxXaHook hook;
    memset(&hook, 0, sizeof hook);
    XaParams &P = hook.p;
    P.tg = targets(op);
    P.o_a = L.o_a[op.b] + (size_t)x->rank * L.a_stride;  // my block (of this buffer) in every region
    P.o_flag = flag_off(0, op.b, x->rank); P.raise_flags = op.nccl ? 0 : 1; P.epoch = op.epoch;
    P.vendor_first = t->dev.vendor_first; P.trunc = t->dev.trunc; P.counters = t->dev.counters;
    P.max_keys = t->dev.max_keys; P.have_trunc = op.have_trunc ? 1 : 0;
    hook.done = x->scratch + 0;
    op.rc = kx_launch_parse(ctx, t, op.a.d_text, op.a.n, op.a.base, 0, &hook);
    if (ctx->stage_timing) cudaEventRecord(ctx->ev[2 * KXPU_T_MERGE], ctx->stream);  // exchange: wait A .. winners inserted
    g_trace.mark(2, ctx->stream);
}

// phase 2: global minima are there -> winners, their names, push of the winner slab
static void shard_phase2(ShardOp &op) {
    if (op.rc != KXPU_OK) return;
    kxpu_ctx *ctx = op.ctx;
    KxExchange *x = op.x;
    kxpu_table *t = op.t;
    const XLayout &L = layout(op);
    uint8_t *mine = my_region(op);
    WaitSpec ws{nullptr, x->nranks, op.epoch, x->scratch + 8};
    if (op.nccl) {
        uint8_t *a0 = mine + L.o_a[0];  // the R phase-A blocks are contiguous: in-place all-gather of mine
        const int nrc = g_nccl.all_gather(a0 + (size_t)x->rank * L.a_stride, a0, L.a_stride, NCCL_UINT8, ctx->nccl_comm, ctx->stream);
        if (nrc != 0) { nccl_fail(op, "ncclAllGather(phase A)", nrc); return; }
    } else {
        ws.flags = reinterpret_cast<const uint32_t *>(mine + flag_off(0, op.b, 0));
        if (!x->fuse_waits) {
            wait_flags_kernel<<<1, 32, 0, ctx->stream>>>(ws);
            KX_LAUNCHED(ctx);
            ws.flags = nullptr;
        }
    }
    g_trace.mark(3, ctx->stream);
    const MinView mv{reinterpret_cast<const unsigned long long *>(mine + L.o_a[op.b]), L.a_stride / 8, x->nranks, nullptr};
    // winners (judged against the minima over all ranks' blocks) are sanitised straight into my own slab
    const uint32_t rows_cap = op.nccl ? x->scaps.rows : x->caps.rows, blob_cap = op.nccl ? x->scaps.blob : x->caps.blob;
    uint8_t *own_slab = op.nccl ? x->send_slab : mine + L.o_slab[op.b] + (size_t)x->rank * L.slab_stride;
    KxSlabOut so;
    memset(&so, 0, sizeof so);
    so.rows = own_slab + slab_rows_off(); so.rows_cap = rows_cap; so.blob = own_slab + slab_blob_off(rows_cap); so.blob_cap = blob_cap;
    // the last CTA of the finalize writes the slab header and tells every peer that the slab can be read
    so.tail.on = 1; so.tail.done = x->scratch + 1; so.tail.header = reinterpret_cast<SlabHeader *>(own_slab);
    if (!op.nccl) { so.tail.tg = targets(op); so.tail.o_flag = flag_off(1, op.b, x->rank); }
    so.tail.epoch = op.epoch; so.tail.rows_cap = rows_cap; so.tail.blob_cap = blob_cap;
    op.rc = kx_launch_finalize(ctx, t, op.a.d_text, op.a.n, op.a.base, &mv, &ws, &so);
    if (op.rc != KXPU_OK) return;
    g_trace.mark(4, ctx->stream);
    g_trace.mark(5, ctx->stream);
}

// phase 3: winners of all ranks -> my table; join of my key slice, results to every rank
static void shard_phase3(ShardOp &op) {
    if (op.rc != KXPU_OK) return;
    kxpu_ctx *ctx = op.ctx;
    KxExchange *x = op.x;
    kxpu_table *t = op.t;
    const XLayout &L = layout(op);
    uint8_t *mine = my_region(op);
    WaitSpec ws{nullptr, x->nranks, op.epoch, x->scratch + 8};
    if (op.nccl) {
        const int nrc = g_nccl.all_gather(x->send_slab, mine + L.o_slab[0], L.slab_stride, NCCL_UINT8, ctx->nccl_comm, ctx->stream);
        if (nrc != 0) { nccl_fail(op, "ncclAllGather(winner slabs)", nrc); return; }
    } else {
        ws.flags = reinterpret_cast<const uint32_t *>(mine + flag_off(1, op.b, 0));
        if (!x->fuse_waits) {
            wait_flags_kernel<<<1, 32, 0, ctx->stream>>>(ws);
            KX_LAUNCHED(ctx);
            ws.flags = nullptr;
        }
    }
    g_trace.mark(6, ctx->stream);
    MergeParams M;
    memset(&M, 0, sizeof M);
    M.wait = ws;
    M.R = x->nranks;
    for (int r = 0; r < x->nranks; r++)  // rank r's slab sits in ITS region (peer memory); NCCL: in my staging copy
        M.slab_of[r] = (op.nccl ? mine : x->peer[r]) + L.o_slab[op.b] + (size_t)r * L.slab_stride;
    M.slab_rows_cap = op.nccl ? x->scaps.rows : x->caps.rows;
    M.mv = MinView{reinterpret_cast<const unsigned long long *>(mine + L.o_a[op.b]), L.a_stride / 8, x->nranks, nullptr};
    M.tab = t->dev; M.row_key = t->row_key; M.row_name_off = t->row_name_off; M.row_name_len = t->row_name_len;
    M.row_line = t->row_line; M.row_anchor = t->row_anchor; M.blob = t->blob; M.rows_cap = t->rows_cap; M.blob_cap = t->blob_cap;
    M.timeout_flag = x->scratch + 8;
    merge_kernel<<<2 * ctx->sm_count, 256, 0, ctx->stream>>>(M);
    KX_LAUNCHED(ctx);
    if (ctx->stage_timing) { cudaEventRecord(ctx->ev[2 * KXPU_T_MERGE + 1], ctx->stream); ctx->ev_used[KXPU_T_MERGE] = true; }
    g_trace.mark(7, ctx->stream);
    if (op.a.nq_total == 0) return;
    KxTimer tm(ctx, KXPU_T_LOOKUP);
    if (op.nccl) {
        // probe straight into my slice of the caller's buffer; the all-gather of hits follows in phase 4
        if (op.a.nq) op.rc = kx_launch_lookup(ctx, t, op.a.d_keys, op.a.nq, op.a.d_rows_all + op.a.key_offset);
        return;
    }
    JoinParams J;
    memset(&J, 0, sizeof J);
    J.keys = op.a.d_keys; J.n = op.a.nq; J.key_offset = op.a.key_offset; J.slots = t->dev.slots; J.cap = t->cap; J.shift = t->shift;
    J.tg = targets(op); J.o_res = L.o_res[op.b]; J.o_flag = flag_off(2, op.b, x->rank); J.raise_flags = 1; J.epoch = op.epoch;
    J.done = x->scratch + 2;
    size_t blocks = std::max<size_t>((op.a.nq + JOIN_PER_CTA - 1) / JOIN_PER_CTA, 1);
    blocks = std::min<size_t>(blocks, (size_t)ctx->sm_count * 8);
    join_gather_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(J);
    KX_LAUNCHED(ctx);
    g_trace.mark(8, ctx->stream);
}

// phase 4: everybody's hits have landed -> caller's buffer; counters to the host
static void shard_phase4(ShardOp &op) {
    if (op.rc != KXPU_OK) return;
    kxpu_ctx *ctx = op.ctx;
    KxExchange *x = op.x;
    const XLayout &L = layout(op);
    uint8_t *mine = my_region(op);
    if (op.a.nq_total) {
        if (op.nccl) {
            const int nrc = g_nccl.all_gather(op.a.d_rows_all + op.a.key_offset, op.a.d_rows_all, op.a.nq * 4, NCCL_UINT8, ctx->nccl_comm, ctx->stream);
            if (nrc != 0) { nccl_fail(op, "ncclAllGather(hits)", nrc); return; }
        } else {
            WaitSpec ws{reinterpret_cast<const uint32_t *>(mine + flag_off(2, op.b, 0)), x->nranks, op.epoch, x->scratch + 8};
            if (!x->fuse_waits || !op.a.d_rows_all) {
                wait_flags_kernel<<<1, 32, 0, ctx->stream>>>(ws);
                KX_LAUNCHED(ctx);
                ws.flags = nullptr;
            }
            if (op.a.d_rows_all) {
                const int32_t *src = reinterpret_cast<const int32_t *>(mine + L.o_res[op.b]);
                if ((reinterpret_cast<uintptr_t>(op.a.d_rows_all) & 15u) == 0) {
                    const size_t n16 = op.a.nq_total / 4;
                    gather_copy_kernel<<<(unsigned)std::min<size_t>(std::max<size_t>((n16 + 255) / 256, 1), 2u * ctx->sm_count), 256, 0, ctx->stream>>>(
                        ws, reinterpret_cast<const uint4 *>(src), reinterpret_cast<uint4 *>(op.a.d_rows_all), n16, src + n16 * 4,
                        op.a.d_rows_all + n16 * 4, (uint32_t)(op.a.nq_total & 3));
                    KX_LAUNCHED(ctx);
                } else {
                    if (ws.flags) { wait_flags_kernel<<<1, 32, 0, ctx->stream>>>(ws); KX_LAUNCHED(ctx); }
                    cudaMemcpyAsync(op.a.d_rows_all, src, op.a.nq_total * 4, cudaMemcpyDeviceToDevice, ctx->stream);
                }
            }
        }
    }
    g_trace.mark(9, ctx->stream);
    cudaMemcpyAsync(ctx->h_ctl, op.t->dev.counters, KX_C_COUNT * 4, cudaMemcpyDeviceToHost, ctx->stream);
    if (!op.nccl) cudaMemcpyAsync(ctx->h_ctl + KX_C_COUNT, x->scratch + 8, 4, cudaMemcpyDeviceToHost, ctx->stream);
}

enum { SH_DONE = 0, SH_RETRY = 1, SH_FAIL = 2 };

// The one host round trip of the load.  Every rank reads the same summary and decides alike.
static int shard_complete(ShardOp &op, kxpu_table **out, int32_t *rc_out) {
    kxpu_ctx *ctx = op.ctx;
    KxExchange *x = op.x;
    auto fail = [&](int32_t rc) {
        if (op.t) { kx_table_release(ctx, op.t); op.t = nullptr; }
        *rc_out = rc;
        return (int)SH_FAIL;
    };
    if (op.rc != KXPU_OK) {
        // an enqueue phase failed on this rank only: the peers are waiting for pushes that never
        // come and will time out -- the exchange cannot be used any more
        if (op.rc != KXPU_E_INVALID && op.rc != KXPU_E_UNSUPPORTED) x->broken = true;
        else if (x->nranks > 1) x->broken = true;
        cudaStreamSynchronize(ctx->stream);
        return fail(op.rc);
    }
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        KX_SET_ERR(ctx, "sharded load failed: %s", cudaGetErrorString(e));
        x->broken = true;
        return fail(KXPU_E_CUDA);
    }
    if (op.a.nq_total && x->ipc) g_trace.report(x->rank, x->nranks);
    const uint32_t *h = ctx->h_ctl;
    const uint32_t st = h[KX_C_XSTATUS];
    if ((st & 0x80000000u) || (!op.nccl && h[KX_C_COUNT])) {
        KX_SET_ERR(ctx, "peer-memory exchange: a rank did not deliver within 4 s (epoch %u)", op.epoch);
        x->broken = true;
        cudaMemsetAsync(x->scratch + 8, 0, 4, ctx->stream);
        return fail(KXPU_E_NCCL);
    }
    kxpu_table *t = op.t;
    const uint32_t total_rows = h[KX_C_XROWS], total_blob = h[KX_C_XBLOB], maxkeys = h[KX_C_XMAXKEYS];
    const bool grow_cap = (st & XS_GROW) || total_rows + maxkeys > merged_key_limit(t->cap) || total_rows > t->rows_cap;
    const bool grow_blob = (st & XS_GROW_BLOB) || total_blob > t->blob_cap;
    const bool need_trunc = (st & XS_NEED_TRUNC) != 0;
    const bool slab_over = (st & XS_SLAB_OVERFLOW) != 0;
    if (grow_cap || grow_blob || need_trunc || slab_over) {
        kx_table_release(ctx, t);
        op.t = nullptr;
        if (grow_cap) {
            uint32_t cap = x->x_cap;
            if (!kx_grow_cap(&cap, (st & XS_FULL) != 0)) { *rc_out = KXPU_E_CAPACITY; return SH_FAIL; }
            x->x_cap = cap;
        }
        if (grow_blob) {
            if (x->x_blob_cap >= (1u << 31)) { *rc_out = KXPU_E_CAPACITY; return SH_FAIL; }
            x->x_blob_cap <<= 2;
        }
        if (need_trunc) op.have_trunc = true;
        if (slab_over) {
            if (op.nccl) { x->scaps.rows = std::max<uint32_t>(x->scaps.rows, 65536u) << 2; x->scaps.blob = std::max<uint32_t>(x->scaps.blob, 2u << 20) << 2; }
            else if (ctx->multi) { KX_SET_ERR(ctx, "winner rows outgrow the peer slab (%u rows / %u name bytes per rank)", x->caps.rows, x->caps.blob); *rc_out = KXPU_E_CAPACITY; return SH_FAIL; }
            else x->use_nccl = true;  // the fixed peer slab is too small for this text: NCCL transport with a growing slab
        }
        return SH_RETRY;
    }
    if (h[KX_C_OVERFLOW]) { kx_table_release(ctx, t); op.t = nullptr; *rc_out = KXPU_E_CAPACITY; return SH_FAIL; }  // unreachable: covered by grow_cap
    t->n_rows = total_rows;
    t->blob_used = total_blob;
    *out = t;
    op.t = nullptr;
    *rc_out = KXPU_OK;
    return SH_DONE;
}

static int32_t shard_run(kxpu_ctx *ctx, const ShardArgs &a, kxpu_table **out) {
    KxExchange *x = ctx->xch;
    ShardOp op;
    op.ctx = ctx; op.x = x; op.a = a;
    for (int attempt = 0; attempt < 16; attempt++) {
        shard_phase1(op);
        shard_phase2(op);
        shard_phase3(op);
        shard_phase4(op);
        int32_t rc = KXPU_OK;
        const int r = shard_complete(op, out, &rc);
        if (r == SH_DONE) return KXPU_OK;
        if (r == SH_FAIL) return rc;
    }
    return KXPU_E_CAPACITY;
}

}  // namespace kxx

using namespace kxx;

void kx_exchange_destroy(kxpu_ctx *ctx) { exchange_free(ctx); }

// ------------------------------------------------------------------ ABI: one process per rank
extern "C" int32_t kxpu_comm_unique_id(uint8_t id_out[KXPU_COMM_ID_BYTES]) {
    if (!id_out) return KXPU_E_INVALID;
    if (!nccl_load()) return KXPU_E_NCCL;
    return g_nccl.get_unique_id(id_out) == 0 ? KXPU_OK : KXPU_E_NCCL;
}

extern "C" int32_t kxpu_comm_init(kxpu_ctx *ctx, int32_t nranks, int32_t rank, const uint8_t id[KXPU_COMM_ID_BYTES]) {
    if (!ctx || !id || nranks < 1 || rank < 0 || rank >= nranks) return KXPU_E_INVALID;
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    if (ctx->multi || ctx->nccl_comm || ctx->xch) return KXPU_E_INVALID;
    if (!nccl_load()) { KX_SET_ERR(ctx, "libnccl.so.2 not found"); return KXPU_E_NCCL; }
    UniqueId uid;
    memcpy(uid.internal, id, 128);
    void *comm = nullptr;
    const int rc = g_nccl.comm_init_rank(&comm, nranks, uid, rank);
    if (rc != 0) {
        KX_SET_ERR(ctx, "ncclCommInitRank: %s", g_nccl.err_string ? g_nccl.err_string(rc) : "error");
        return KXPU_E_NCCL;
    }
    KxExchange *x = new (std::nothrow) KxExchange();
    if (!x) { g_nccl.comm_destroy(comm); return KXPU_E_NOMEM; }
    ctx->nccl_comm = comm;
    ctx->nranks = nranks;
    ctx->rank = rank;
    x->nranks = nranks;
    x->rank = rank;
    ctx->xch = x;
    ipc_setup(ctx, x);
    return KXPU_OK;
}

extern "C" int32_t kxpu_comm_destroy(kxpu_ctx *ctx) {
    if (!ctx) return KXPU_E_INVALID;
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    if (ctx->multi) return KXPU_E_INVALID;
    cudaStreamSynchronize(ctx->stream);
    exchange_free(ctx);
    if (ctx->nccl_comm) {
        g_nccl.comm_destroy(ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    ctx->nranks = 1;
    ctx->rank = 0;
    return KXPU_OK;
}

static int32_t check_shard_args(kxpu_ctx *ctx, const ShardArgs &a, kxpu_table **out) {
    if (!out || (!a.d_text && a.n)) return KXPU_E_INVALID;
    if (a.nq_total) {
        if ((a.nq && !a.d_keys) || a.key_offset + a.nq > a.nq_total) return KXPU_E_INVALID;
        KxExchange *x = ctx->xch;
        if (x && x->p2p && !x->use_nccl && a.nq_total > x->caps.join) {
            KX_SET_ERR(ctx, "sharded join of %zu keys exceeds the exchange capacity of %u", a.nq_total, x->caps.join);
            return KXPU_E_UNSUPPORTED;
        }
        if (x && (!x->p2p || x->use_nccl) && (!a.d_rows_all || a.key_offset != (size_t)x->rank * a.nq || a.nq * (size_t)x->nranks != a.nq_total)) {
            KX_SET_ERR(ctx, "NCCL transport needs equal key slices in rank order and a result buffer");
            return KXPU_E_UNSUPPORTED;
        }
    }
    return KXPU_OK;
}

extern "C" int32_t kxpu_pciids_join_sharded(kxpu_ctx *ctx, const void *d_text_shard, size_t n, uint64_t global_base,
                                            const uint32_t *d_keys, size_t nq, size_t key_offset, size_t nq_total,
                                            int32_t *d_rows_all, kxpu_table **out) {
    if (!ctx) return KXPU_E_INVALID;
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    if (ctx->multi) { KX_SET_ERR(ctx, "this ctx belongs to a kxpu_multi group: use kxpu_multi_pciids_join"); return KXPU_E_INVALID; }
    if (!ctx->xch) { KX_SET_ERR(ctx, "kxpu_comm_init has not been called"); return KXPU_E_NCCL; }
    ShardArgs a{(const uint8_t *)d_text_shard, n, global_base, d_keys, nq, key_offset, nq_total, d_rows_all};
    const int32_t rc = check_shard_args(ctx, a, out);
    if (rc != KXPU_OK) return rc;
    return shard_run(ctx, a, out);
}

extern "C" int32_t kxpu_pciids_load_sharded(kxpu_ctx *ctx, const void *d_text_shard, size_t n, uint64_t global_base,
                                            kxpu_table **out) {
    return kxpu_pciids_join_sharded(ctx, d_text_shard, n, global_base, nullptr, 0, 0, 0, nullptr, out);
}

// ------------------------------------------------------------------ ABI: one process, N GPUs
struct kxpu_multi {
    int n = 0;
    kxpu_ctx *ctx[KX_MAX_RANKS] = {};
};

int32_t kx_ctx_create_on(int32_t ordinal, kxpu_ctx **out);  // api.cu

extern "C" int32_t kxpu_multi_destroy(kxpu_multi *m) {
    if (!m) return KXPU_E_INVALID;
    for (int i = 0; i < m->n; i++) {
        if (!m->ctx[i]) continue;
        cudaSetDevice(m->ctx[i]->device);
        cudaStreamSynchronize(m->ctx[i]->stream);
    }
    for (int i = 0; i < m->n; i++) {
        if (!m->ctx[i]) continue;
        m->ctx[i]->multi = nullptr;
        kxpu_ctx_destroy(m->ctx[i]);
    }
    delete m;
    return KXPU_OK;
}

extern "C" int32_t kxpu_ctx_create_multi(const int32_t *ordinals, int32_t n, kxpu_multi **out) {
    if (!ordinals || !out || n < 1 || n > KX_MAX_RANKS) return KXPU_E_INVALID;
    *out = nullptr;
    kxpu_multi *m = new (std::nothrow) kxpu_multi();
    if (!m) return KXPU_E_NOMEM;
    m->n = n;
    int32_t rc = KXPU_OK;
    for (int i = 0; i < n && rc == KXPU_OK; i++) rc = kx_ctx_create_on(ordinals[i], &m->ctx[i]);
    // every pair of distinct devices needs peer access in both directions (NVSwitch: always there)
    for (int i = 0; i < n && rc == KXPU_OK; i++) {
        cudaSetDevice(m->ctx[i]->device);
        for (int j = 0; j < n && rc == KXPU_OK; j++) {
            if (m->ctx[j]->device == m->ctx[i]->device) continue;
            int can = 0;
            cudaDeviceCanAccessPeer(&can, m->ctx[i]->device, m->ctx[j]->device);
            if (!can) { rc = KXPU_E_NCCL; break; }
            const cudaError_t e = cudaDeviceEnablePeerAccess(m->ctx[j]->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) rc = KXPU_E_CUDA;
            cudaGetLastError();
        }
    }
    for (int i = 0; i < n && rc == KXPU_OK; i++) {
        kxpu_ctx *c = m->ctx[i];
        cudaSetDevice(c->device);
        KxExchange *x = new (std::nothrow) KxExchange();
        if (!x) { rc = KXPU_E_NOMEM; break; }
        x->nranks = n; x->rank = i;
        c->xch = x; c->nranks = n; c->rank = i;
        rc = region_alloc(c, x, kPeerCaps);
    }
    if (rc == KXPU_OK) {
        for (int i = 0; i < n; i++) {
            KxExchange *x = m->ctx[i]->xch;
            for (int j = 0; j < n; j++) x->peer[j] = m->ctx[j]->xch->local;  // direct pointers: one address space
            x->p2p = true;
            x->ipc = false;
            bool distinct = true;
            for (int a = 0; a < n; a++)
                for (int b2 = a + 1; b2 < n; b2++) distinct = distinct && m->ctx[a]->device != m->ctx[b2]->device;
            x->fuse_waits = distinct;
        }
        for (int i = 0; i < n; i++) m->ctx[i]->multi = m;
        *out = m;
        return KXPU_OK;
    }
    kxpu_multi_destroy(m);
    return rc;
}

extern "C" int32_t kxpu_multi_size(kxpu_multi *m) { return m ? m->n : 0; }
extern "C" kxpu_ctx *kxpu_multi_ctx(kxpu_multi *m, int32_t i) { return (m && i >= 0 && i < m->n) ? m->ctx[i] : nullptr; }

extern "C" int32_t kxpu_multi_pciids_join(kxpu_multi *m, const kxpu_shard *shards, size_t nq_total, kxpu_table **tables_out) {
    if (!m || !shards || !tables_out) return KXPU_E_INVALID;
    const int n = m->n;
    // all ranks are driven from this thread, phase by phase: when a rank's wait is enqueued, the push
    // it waits for is already in its peer's stream, so the host never blocks in front of a wait
    for (int i = 0; i < n; i++) m->ctx[i]->mu.lock();
    ShardOp ops[KX_MAX_RANKS];
    int32_t rc = KXPU_OK;
    for (int i = 0; i < n; i++) {
        kxpu_ctx *c = m->ctx[i];
        tables_out[i] = nullptr;
        kx_clear_timings(c);
        ops[i].ctx = c; ops[i].x = c->xch;
        ops[i].a = ShardArgs{(const uint8_t *)shards[i].d_text, shards[i].n, shards[i].global_base, shards[i].d_keys, shards[i].nq,
                            shards[i].key_offset, nq_total, shards[i].d_rows_all};
        cudaSetDevice(c->device);
        const int32_t r = check_shard_args(c, ops[i].a, &tables_out[i]);
        if (r != KXPU_OK && rc == KXPU_OK) rc = r;
    }
    for (int attempt = 0; attempt < 16 && rc == KXPU_OK; attempt++) {
        for (int ph = 1; ph <= 4; ph++) {
            for (int i = 0; i < n; i++) {
                cudaSetDevice(ops[i].ctx->device);
                if (ph == 1) shard_phase1(ops[i]);
                else if (ph == 2) shard_phase2(ops[i]);
                else if (ph == 3) shard_phase3(ops[i]);
                else shard_phase4(ops[i]);
            }
        }
        bool retry = false, done = true;
        for (int i = 0; i < n; i++) {
            cudaSetDevice(ops[i].ctx->device);
            int32_t r = KXPU_OK;
            const int s = shard_complete(ops[i], &tables_out[i], &r);
            if (s == SH_RETRY) { retry = true; done = false; }
            else if (s == SH_FAIL) { if (rc == KXPU_OK) rc = r; done = false; }
        }
        if (rc != KXPU_OK) break;
        if (done) break;
        if (!retry) break;
        for (int i = 0; i < n; i++)  // a retry is collective: ranks that finished hand their table back
            if (tables_out[i]) { cudaSetDevice(ops[i].ctx->device); kx_table_release(ops[i].ctx, tables_out[i]); tables_out[i] = nullptr; }
    }
    if (rc != KXPU_OK)
        for (int i = 0; i < n; i++)
            if (tables_out[i]) { cudaSetDevice(ops[i].ctx->device); kx_table_release(ops[i].ctx, tables_out[i]); tables_out[i] = nullptr; }
    for (int i = n - 1; i >= 0; i--) m->ctx[i]->mu.unlock();
    return rc;
}

// ------------------------------------------------------------------ shard planning (host)
// Smallest offset >= pos at which a top-level line starts (n if none): a line start whose first
// byte is neither '\t' nor '#'.
static size_t next_top_level_start(const uint8_t *text, size_t n, size_t pos) {
    if (pos == 0) return 0;
    if (pos >= n) return n;
    size_t p = pos;
    if (text[p - 1] != '\n') {
        const void *nl = memchr(text + p, '\n', n - p);
        if (!nl) return n;
        p = (size_t)((const uint8_t *)nl - text) + 1;
    }
    while (p < n) {
        if (text[p] != '\t' && text[p] != '#') return p;
        const void *nl = memchr(text + p, '\n', n - p);
        if (!nl) return n;
        p = (size_t)((const uint8_t *)nl - text) + 1;
    }
    return n;
}

extern "C" int32_t kxpu_plan_shards(const uint8_t *text, size_t n, int32_t nranks, uint64_t *cuts_out) {
    if ((!text && n) || nranks < 1 || !cuts_out) return KXPU_E_INVALID;
    cuts_out[0] = 0;
    for (int r = 1; r < nranks; r++) {
        const size_t want = (size_t)((unsigned __int128)n * (unsigned)r / (unsigned)nranks);
        const size_t c = next_top_level_start(text, n, want);
        cuts_out[r] = std::max<uint64_t>(cuts_out[r - 1], c);
    }
    cuts_out[nranks] = n;
    return KXPU_OK;
}
