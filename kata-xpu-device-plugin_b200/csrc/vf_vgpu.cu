// vf_vgpu.cu -- K15: the type join of vGPUs on SR-IOV virtual functions (kxpu_vf_vgpu_types).  include/kxpu.h states
// the rules.
//
// Two launches, one table:
//   - k_vt_lines: one warp per CHUNK bytes of the blob.  Lane l looks at byte base + 32 s + l and decides whether a line
//     starts there (the start of its table, or the byte after a '\n'); the table of a byte is found by walking forward
//     from the chunk's table (one binary search per warp).  Each lane with a line start parses that line on its own and,
//     when the line names a type, inserts its ID into an open-addressing table of {ID, line offset} slots: a slot is
//     claimed by CAS on the ID word and the offset word takes an atomic min.  The blob offset of a line orders lines by
//     table, then by line, so the minimum is the first naming line.  The warp also counts every line start and every
//     naming line.
//   - k_vt_records: one thread per record.  Two 16-byte loads of its kxpu_vfvgpurec, the current type parsed in
//     registers, one probe; a NAMED record re-parses the winning line, builds its key in a 48-byte row of shared memory
//     (kxmdev::type_key, the rule kxpu_classify_mdev uses) and writes it with three 16-byte stores.
// The table starts with SMALL_CAP slots; when more than half of them hold distinct IDs (or a probe run passes
// PROBE_LIMIT) the host runs both launches again with room for every naming line the first run counted.
//
// kxpu_vf_vgpu_drift: one launch, k_vd_drift (records, then groups), parsing through current_type as k_vt_records does.
#include "common.cuh"
#include "mdev.cuh"

namespace kxvt {

constexpr unsigned long long EMPTY = ~0ull;
constexpr uint32_t CHUNK = 2048;        // blob bytes per warp of k_vt_lines
constexpr uint32_t SMALL_CAP = 4096;    // slots of the first run (a real host has a few dozen type IDs)
constexpr uint32_t PROBE_LIMIT = 512;   // first run: a longer probe run flags the table as too small

struct __align__(16) Slot { unsigned long long id, off; };

struct Work {
    const uint8_t *blob;
    const unsigned long long *toff;  // [n_tables + 1]
    uint32_t n_tables;
    unsigned long long lo, hi;       // blob bytes [lo, hi) = [toff[0], toff[n_tables])
    Slot *slots;
    uint32_t mask, limit, stop;      // limit: probe steps (cap on the full run); stop: distinct IDs allowed (cap on the full run)
    unsigned long long *totals;      // 0 lines, 1 naming lines, 2 claims, 3 overflow flag
    const kxpu_vfvgpurec *recs;
    uint32_t n;
    uint4 *keys;
    uint32_t *type_id;
    uint8_t *status;
};

__device__ __forceinline__ bool blank(uint32_t c) { return c == ' ' || c == '\t'; }

// the last table t with toff[t] <= pos (pos in [lo, hi))
__device__ __forceinline__ uint32_t table_of(const Work &W, unsigned long long pos) {
    uint32_t a = 0, b = W.n_tables;  // toff[a] <= pos < toff[b]
    while (b - a > 1) {
        const uint32_t m = (a + b) / 2;
        if (W.toff[m] <= pos) a = m;
        else b = m;
    }
    return a;
}

// The line that starts at p in a table ending at end: true when it names a type; id and the NAME as ten little-endian
// words (bytes past nlen are zero) with its length.
__device__ __forceinline__ bool parse_line(const uint8_t *blob, unsigned long long p, unsigned long long end, uint32_t &id,
                                           uint32_t w[10], uint32_t &nlen) {
    unsigned long long e = p;  // the line's end: its '\n' or the table's end
    while (e < end && blob[e] != '\n') e++;
    if (e > p && blob[e - 1] == '\r') e--;
    while (p < e && blank(blob[p])) p++;
    if (p == e || blob[p] < '1' || blob[p] > '9') return false;
    unsigned long long v = 0;
    uint32_t digits = 0;
    while (p < e && blob[p] >= '0' && blob[p] <= '9') {
        if (++digits > 10) return false;
        v = v * 10 + (blob[p] - '0');
        p++;
    }
    if (v > 0xFFFFFFFFull) return false;
    while (p < e && blank(blob[p])) p++;
    if (p == e || blob[p] != ':') return false;
    p++;
    while (p < e && blank(blob[p])) p++;
    while (e > p && blank(blob[e - 1])) e--;
    if (e == p || e - p > kxmdev::NAME_MAX_BYTES) return false;
    nlen = (uint32_t)(e - p);
#pragma unroll
    for (int k = 0; k < 10; k++) w[k] = 0u;
    for (uint32_t k = 0; k < nlen; k++) w[k >> 2] |= (uint32_t)blob[p + k] << (8 * (k & 3));
    id = (uint32_t)v;
    return kxmdev::type_key(w, nlen, [](uint32_t, uint8_t) {}) != 0u;
}

__device__ __forceinline__ void insert(const Work &W, uint32_t id, unsigned long long off) {
    uint32_t s = kx_hash(id) & W.mask;
    for (uint32_t step = 0; step < W.limit; step++, s = (s + 1) & W.mask) {
        unsigned long long v = __ldcg(&W.slots[s].id);
        if (v == EMPTY) {
            v = atomicCAS(&W.slots[s].id, EMPTY, (unsigned long long)id);
            if (v == EMPTY) {  // a new ID: only a won claim counts, so the count is the number of distinct IDs
                v = id;
                if (atomicAdd(&W.totals[2], 1ull) >= W.stop) atomicOr(&W.totals[3], 1ull);  // half full: run again
            }
        }
        if (v == id) {
            if (off < __ldcg(&W.slots[s].off)) atomicMin(&W.slots[s].off, off);
            return;
        }
    }
    atomicOr(&W.totals[3], 1ull);
}

__global__ void __launch_bounds__(256) k_vt_lines(const Work W) {
    const uint32_t lane = threadIdx.x & 31u;
    const unsigned long long base = W.lo + ((unsigned long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5)) * CHUNK;
    if (base >= W.hi) return;
    const unsigned long long end = min(base + CHUNK, W.hi);
    uint32_t t = table_of(W, base);
    uint32_t lines = 0, named = 0;
    for (unsigned long long s = base; s < end; s += 32) {
        const unsigned long long pos = s + lane;
        uint32_t mt = t;
        bool start = false;
        if (pos < end) {
            while (W.toff[mt + 1] <= pos) mt++;
            start = pos == W.toff[mt] || W.blob[pos - 1] == '\n';
        }
        t = __shfl_sync(0xffffffffu, mt, 31);  // lane 31 holds the furthest table (an inactive lane keeps the last one)
        uint32_t id = 0, w[10], nlen = 0;
        const bool names = start && parse_line(W.blob, pos, W.toff[mt + 1], id, w, nlen);
        if (names) insert(W, id, pos);
        lines += __popc(__ballot_sync(0xffffffffu, start));
        named += __popc(__ballot_sync(0xffffffffu, names));
    }
    if (lane == 0) {
        atomicAdd(&W.totals[0], (unsigned long long)lines);
        atomicAdd(&W.totals[1], (unsigned long long)named);
    }
}

// The current-type rule (include/kxpu.h) on one kxpu_vfvgpurec: cw = cur_txt as four words, len = cur_len, fl = flags.
// Returns the type, with ok set when the read did not fail and cur_txt[0..len), with at most one trailing '\n' removed,
// is a canonical decimal below 2^32.  The caller tests KXPU_VT_READ.  k_vt_records and k_vd_drift both parse through
// it, so the type join and the drift check cannot read one text two ways.
__device__ __forceinline__ unsigned long long current_type(const uint32_t cw[4], uint32_t len, uint32_t fl, bool &ok) {
    uint32_t l = len;
    ok = !(fl & KXPU_VT_CUR_ERR) && len <= 16u;
    if (ok && l && kxmdev::byte_at(cw, l - 1) == '\n') l--;
    ok &= l > 0 && l <= 10u && !(l > 1 && kxmdev::byte_at(cw, 0) == '0');
    unsigned long long v = 0;
#pragma unroll
    for (uint32_t k = 0; k < 16; k++) {
        const uint32_t d = kxmdev::byte_at(cw, k) - '0';
        if (k < l) {
            ok &= d <= 9u;
            v = v * 10 + d;
        }
    }
    ok &= v <= 0xFFFFFFFFull;
    return v;
}

__global__ void __launch_bounds__(256) k_vt_records(const Work W) {
    __shared__ __align__(16) uint8_t skey[256][48];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W.n) return;
    const uint4 *rp = reinterpret_cast<const uint4 *>(W.recs + i);
    const uint4 q0 = rp[0], q1 = rp[1];  // cur_txt[16]; cur_len, flags, reserved
    const uint32_t len = q1.x & 0xffu, fl = (q1.x >> 8) & 0xffu;
    uint8_t *row = skey[threadIdx.x];
    uint4 *row4 = reinterpret_cast<uint4 *>(row);
    row4[0] = row4[1] = row4[2] = make_uint4(0u, 0u, 0u, 0u);
    uint32_t st = KXPU_VT_NONE, tid = 0;
    if (fl & KXPU_VT_READ) {
        const uint32_t cw[4] = {q0.x, q0.y, q0.z, q0.w};
        bool ok;
        const unsigned long long v = current_type(cw, len, fl, ok);
        if (!ok) st = KXPU_VT_BAD;
        else if (v != 0) {
            tid = (uint32_t)v;
            st = KXPU_VT_UNNAMED;
            uint32_t s = kx_hash(tid) & W.mask;
            for (uint32_t step = 0; step <= W.mask; step++, s = (s + 1) & W.mask) {
                const unsigned long long id = W.slots[s].id;
                if (id == EMPTY) break;
                if (id == tid) {
                    const unsigned long long off = W.slots[s].off;
                    uint32_t pid, w[10], nlen;
                    parse_line(W.blob, off, W.toff[table_of(W, off) + 1], pid, w, nlen);
                    row[47] = (uint8_t)kxmdev::type_key(w, nlen, [&](uint32_t p, uint8_t c) { row[p] = c; });
                    st = KXPU_VT_NAMED;
                    break;
                }
            }
        }
    }
    uint4 *kp = W.keys + 3 * (size_t)i;
    kp[0] = row4[0]; kp[1] = row4[1]; kp[2] = row4[2];
    W.type_id[i] = tid;
    W.status[i] = (uint8_t)st;
}

// kxpu_vf_vgpu_drift: the status of record i against the walk's type was, and the type read back in now
__device__ __forceinline__ uint32_t drift_of(const kxpu_vfvgpurec *recs, uint32_t i, uint32_t was, uint32_t &now) {
    const uint4 *rp = reinterpret_cast<const uint4 *>(recs + i);
    const uint4 q0 = rp[0], q1 = rp[1];
    if (!((q1.x >> 8) & KXPU_VT_READ)) {
        now = was;
        return KXPU_VD_SAME;
    }
    const uint32_t cw[4] = {q0.x, q0.y, q0.z, q0.w};
    bool ok;
    const unsigned long long v = current_type(cw, q1.x & 0xffu, (q1.x >> 8) & 0xffu, ok);
    if (!ok) {
        now = 0;
        return KXPU_VD_BAD;
    }
    now = (uint32_t)v;
    return now == was ? KXPU_VD_SAME : now == 0 ? KXPU_VD_CLEARED : KXPU_VD_CHANGED;
}

// One launch: CTAs [0, rec_ctas) give one thread per record; the rest give one warp per group, whose lanes re-parse
// their members (a member is one 32-byte record) and fold the drifted positions with a warp min.  Parsing a member
// again costs less than a second launch that waits for the records.
__global__ void __launch_bounds__(256) k_vd_drift(const kxpu_vfvgpurec *__restrict__ recs, const uint32_t *__restrict__ was,
                                                  uint32_t n, uint32_t rec_ctas, const uint32_t *__restrict__ goff,
                                                  const uint32_t *__restrict__ gmem, uint32_t n_groups,
                                                  uint32_t *__restrict__ type_now, uint8_t *__restrict__ status,
                                                  uint32_t *__restrict__ first, uint32_t *__restrict__ err) {
    if (blockIdx.x < rec_ctas) {
        const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n) return;
        uint32_t now;
        status[i] = (uint8_t)drift_of(recs, i, was[i], now);
        type_now[i] = now;
        return;
    }
    const uint32_t o = (blockIdx.x - rec_ctas) * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    if (o >= n_groups) return;  // warp-uniform
    const uint32_t a = goff[o], b = goff[o + 1];
    uint32_t best = KXPU_VD_STEADY;
    bool bad = false;
    for (uint32_t m = a + lane; m < b; m += 32u) {  // every member is range-checked; parsing stops at a lane's first drift
        const uint32_t i = gmem[m];
        if (i >= n) { bad = true; continue; }
        uint32_t now;
        if (best == KXPU_VD_STEADY && drift_of(recs, i, was[i], now) != KXPU_VD_SAME) best = m - a;
    }
    best = __reduce_min_sync(0xffffffffu, best);
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) {
        first[o] = best;
        if (bad) atomicOr(err, 1u);
    }
}

}  // namespace kxvt

using namespace kxvt;

extern "C" int32_t kxpu_vf_vgpu_types(kxpu_ctx *ctx, const kxpu_vfvgpurec *recs_vt, size_t n, const uint8_t *blob,
                                      const uint64_t *table_off, size_t n_tables, kxpu_vgpukey *keys_out, uint32_t *type_id,
                                      uint8_t *status) {
    static_assert(sizeof(kxpu_vfvgpurec) == 32 && offsetof(kxpu_vfvgpurec, cur_len) == 16, "kxpu_vfvgpurec layout");
    static_assert(sizeof(kxpu_vgpukey) == 48 && offsetof(kxpu_vgpukey, len) == 47, "kxpu_vgpukey layout");
    if (!ctx || (n && (!recs_vt || !keys_out || !type_id || !status)) || !table_off) return KXPU_E_INVALID;
    if (n >= (1ull << 30)) return KXPU_E_UNSUPPORTED;
    if (table_off[n_tables] >= (1ull << 40)) return KXPU_E_UNSUPPORTED;  // a line's offset is packed in 40 bits
    for (size_t t = 0; t < n_tables; t++)
        if (table_off[t + 1] < table_off[t]) { KX_SET_ERR(ctx, "vf_vgpu_types: table %zu: offsets decrease", t); return KXPU_E_INVALID; }
    const unsigned long long lo = table_off[0], hi = table_off[n_tables];
    if (hi > lo && !blob) return KXPU_E_INVALID;
    if (n == 0) return KXPU_OK;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    cudaStream_t st = ctx->stream;
    const size_t bytes = hi - lo;
    // the blob is copied from toff[0] on and addressed as if it started at 0: the device offsets are table_off - lo
    std::vector<unsigned long long> toff(n_tables + 1);
    for (size_t t = 0; t <= n_tables; t++) toff[t] = table_off[t] - lo;
    unsigned long long full = 0;  // 0: the first run; else the slot count of the full run
    for (;;) {
        const unsigned long long cap = full ? full : SMALL_CAP;
        size_t off = 0;
        auto take = [&](size_t b) { size_t o = off; off = (off + b + 255) / 256 * 256; return o; };
        const size_t o_blob = take(bytes), o_toff = take((n_tables + 1) * 8), o_slots = take(cap * sizeof(Slot));
        const size_t o_tot = take(32), o_recs = take(n * sizeof(kxpu_vfvgpurec)), o_keys = take(n * 48);
        const size_t o_tid = take(n * 4), o_st = take(n);
        KxScratch sc(ctx);
        uint8_t *b = nullptr;
        KX_CUDA(ctx, sc.alloc((void **)&b, off));
        if (bytes) cudaMemcpyAsync(b + o_blob, blob + lo, bytes, cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(b + o_toff, toff.data(), (n_tables + 1) * 8, cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(b + o_recs, recs_vt, n * sizeof(kxpu_vfvgpurec), cudaMemcpyHostToDevice, st);
        // KXPU_T_CLASSIFY spans the table resets and launches of every run: from the first run's reset to the last launch
        if (!full && ctx->stage_timing) cudaEventRecord(ctx->ev[2 * KXPU_T_CLASSIFY], st);
        cudaMemsetAsync(b + o_slots, 0xFF, cap * sizeof(Slot), st);
        cudaMemsetAsync(b + o_tot, 0, 32, st);
        Work W;
        W.blob = b + o_blob; W.toff = (const unsigned long long *)(b + o_toff); W.n_tables = (uint32_t)n_tables;
        W.lo = 0; W.hi = bytes;
        W.slots = (Slot *)(b + o_slots); W.mask = (uint32_t)(cap - 1);
        W.limit = full ? (uint32_t)cap : PROBE_LIMIT;
        W.stop = full ? (uint32_t)cap : SMALL_CAP / 2;
        W.totals = (unsigned long long *)(b + o_tot);
        W.recs = (const kxpu_vfvgpurec *)(b + o_recs); W.n = (uint32_t)n;
        W.keys = (uint4 *)(b + o_keys); W.type_id = (uint32_t *)(b + o_tid); W.status = b + o_st;
        if (bytes) {
            const unsigned long long warps = (bytes + CHUNK - 1) / CHUNK;
            k_vt_lines<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(W);
            ctx->launches++;
        }
        k_vt_records<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W);
        ctx->launches++;
        if (ctx->stage_timing) {
            cudaEventRecord(ctx->ev[2 * KXPU_T_CLASSIFY + 1], st);
            ctx->ev_used[KXPU_T_CLASSIFY] = true;
        }
        unsigned long long *h = reinterpret_cast<unsigned long long *>(ctx->h_ctl);
        cudaMemcpyAsync(h, W.totals, 32, cudaMemcpyDeviceToHost, st);
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { KX_SET_ERR(ctx, "vf_vgpu_types failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
        if (h[0] >= (1ull << 30)) { KX_SET_ERR(ctx, "vf_vgpu_types: %llu lines (limit 2^30)", h[0]); return KXPU_E_UNSUPPORTED; }
        if (h[3]) {
            if (full) { KX_SET_ERR(ctx, "vf_vgpu_types: type table overflow"); return KXPU_E_CAPACITY; }
            full = SMALL_CAP;
            while (full < 2 * h[1]) full <<= 1;
            continue;
        }
        cudaMemcpyAsync(keys_out, W.keys, n * 48, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(type_id, W.type_id, n * 4, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(status, W.status, n, cudaMemcpyDeviceToHost, st);
        e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { KX_SET_ERR(ctx, "vf_vgpu_types D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
        return KXPU_OK;
    }
}

extern "C" int32_t kxpu_vf_vgpu_drift(kxpu_ctx *ctx, const kxpu_vfvgpurec *recs_vt, const uint32_t *type_was, size_t n,
                                      const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                      uint32_t *type_now, uint8_t *status_now, uint32_t *group_first) {
    if (!ctx || (n && (!recs_vt || !type_was || !type_now || !status_now)) || !group_off || (n_groups && !group_first))
        return KXPU_E_INVALID;
    if (n >= (1ull << 28) || n_groups >= (1ull << 28)) return KXPU_E_UNSUPPORTED;
    for (size_t g = 0; g < n_groups; g++)
        if (group_off[g + 1] < group_off[g]) { KX_SET_ERR(ctx, "vf_vgpu_drift: group %zu: offsets decrease", g); return KXPU_E_INVALID; }
    const size_t nm = group_off[n_groups];
    if (nm && !group_members) return KXPU_E_INVALID;
    if (n == 0 && n_groups == 0) return KXPU_OK;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    const size_t G = n_groups;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_recs = take(n * sizeof(kxpu_vfvgpurec)), o_was = take(n * 4), o_goff = take((G + 1) * 4);
    const size_t o_gmem = take(nm * 4), o_now = take(n * 4), o_st = take(n), o_first = take(G * 4), o_err = take(16);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_recs, recs_vt, n * sizeof(kxpu_vfvgpurec)); up(o_was, type_was, n * 4);
    up(o_goff, group_off, (G + 1) * 4); up(o_gmem, group_members, nm * 4);
    cudaMemsetAsync(b + o_err, 0, 16, st);
    uint32_t *d_err = (uint32_t *)(b + o_err);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        const size_t rec_ctas = (n + 255) / 256, grp_ctas = (G + 7) / 8;
        k_vd_drift<<<(unsigned)(rec_ctas + grp_ctas), 256, 0, st>>>(
            (const kxpu_vfvgpurec *)(b + o_recs), (const uint32_t *)(b + o_was), (uint32_t)n, (uint32_t)rec_ctas,
            (const uint32_t *)(b + o_goff), (const uint32_t *)(b + o_gmem), (uint32_t)G, (uint32_t *)(b + o_now),
            b + o_st, (uint32_t *)(b + o_first), d_err);
        KX_LAUNCHED(ctx);
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, d_err, 4, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "vf_vgpu_drift failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) { KX_SET_ERR(ctx, "vf_vgpu_drift: a group member index is >= n"); return KXPU_E_INVALID; }
    if (n) {
        cudaMemcpyAsync(type_now, b + o_now, n * 4, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(status_now, b + o_st, n, cudaMemcpyDeviceToHost, st);
    }
    if (G) cudaMemcpyAsync(group_first, b + o_first, G * 4, cudaMemcpyDeviceToHost, st);
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "vf_vgpu_drift D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}
