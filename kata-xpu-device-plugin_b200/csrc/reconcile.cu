// reconcile.cu -- K9: index reconciliation of a rediscovery (kxpu_reconcile).
//
// A rediscovery walks sysfs again and must give every surviving function the CDI index it already has, and every other
// one an index that was never handed out (include/kxpu.h defines the rule).  That is a keyed join of the previous
// snapshot against the new walk plus an ordered count of the entries that did not survive:
//   - k_rc_insert: one thread per entry of prev ++ cur.  It validates the key (non-empty, NUL padded) and, for prev, the
//     index, then inserts the key into one open-addressing table of 16-byte slots { hash << 32 | owner entry, prev
//     entry, cur entry } sized up front to >= 2 (n_prev + n_cur), so there is no growth retry.  A hash hit compares
//     the 40 key bytes with the owner's record (byte for byte, as k_intern does); the entry then claims its list's
//     field of the slot by CAS, and a field that is already claimed is a duplicate within that list.
//   - k_rc_probe: cur entries in tiles of RC_TILE, RC_ITEMS consecutive entries per thread.  Each entry reads its
//     slot's prev field, compares group / klass / tag, writes the states and the kept index, and the non-kept count of
//     the tile goes through the decoupled look-back of scan.cuh (block_excl + lookback), which gives every fresh entry
//     next_index + (non-kept entries before it) in the same kernel.
// Launches: two memsets (table, states / counters) | insert | probe + scan.
#include <algorithm>

#include "common.cuh"
#include "scan.cuh"

namespace kxrc {

constexpr uint32_t EMPTY32 = 0xFFFFFFFFu;
constexpr unsigned long long EMPTY64 = 0xFFFFFFFFFFFFFFFFull;

struct __align__(16) RSlot { unsigned long long tag; uint32_t prev, cur; };  // hash << 32 | owner; entry of each list

constexpr int RC_THREADS = kxscan::SCAN_THREADS;  // block_excl works on SCAN_THREADS threads
constexpr int RC_ITEMS = 4;
constexpr int RC_TILE = RC_THREADS * RC_ITEMS;

// ctl[] (device): 0 error bits, 1 kept, 2 changed
constexpr uint32_t ERR_KEY = 1u, ERR_DUP_PREV = 2u, ERR_DUP_CUR = 4u, ERR_INDEX = 8u;

struct Rc {
    const uint4 *prev, *cur;  // 64-byte records: four uint4 each
    uint32_t n_prev, n_cur;
    unsigned long long next_index;
    RSlot *tab;
    uint32_t cap, shift;
    uint32_t *cslot;          // [n_cur] slot of cur[i] (EMPTY32: its key was invalid)
    unsigned long long *idx;  // [n_cur]
    uint8_t *cstate, *pstate;
    uint32_t *ctl;
    unsigned long long *state;
    uint32_t epoch;
};

__device__ __forceinline__ bool key_eq(const uint4 &a, const uint4 &b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }

// non-empty, and no non-NUL byte after the first NUL, over the 40 key bytes
__device__ __forceinline__ bool key_ok(const uint32_t (&w)[10]) {
    bool seen_nul = false, ok = (w[0] & 0xffu) != 0u;
#pragma unroll
    for (int k = 0; k < 10; k++) {
#pragma unroll
        for (int b = 0; b < 4; b++) {
            const bool nul = ((w[k] >> (8 * b)) & 0xffu) == 0u;
            ok &= nul || !seen_nul;
            seen_nul |= nul;
        }
    }
    return ok;
}

__global__ void __launch_bounds__(256) k_rc_insert(const Rc R) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= R.n_prev + R.n_cur) return;
    const bool is_prev = t < R.n_prev;
    const uint32_t e = is_prev ? t : t - R.n_prev;
    const uint4 *rp = (is_prev ? R.prev : R.cur) + 4 * (size_t)e;
    const uint4 k0 = rp[0], k1 = rp[1], k2 = rp[2];
    const uint32_t w[10] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w, k2.x, k2.y};
    if (is_prev) {
        const uint4 q3 = rp[3];
        const unsigned long long index = ((unsigned long long)q3.w << 32) | q3.z;
        if (index >= R.next_index) atomicOr(&R.ctl[0], ERR_INDEX);
    }
    if (!key_ok(w)) {
        atomicOr(&R.ctl[0], ERR_KEY);
        if (!is_prev) R.cslot[e] = EMPTY32;
        return;
    }
    unsigned long long hv = 0x9E3779B97F4A7C15ull;
#pragma unroll
    for (int k = 0; k < 10; k++) { hv = (hv ^ w[k]) * 0xff51afd7ed558ccdull; hv ^= hv >> 29; }
    const uint32_t h = (uint32_t)(hv >> 32);
    const unsigned long long tag = ((unsigned long long)h << 32) | t;
    uint32_t slot = h >> R.shift;
    for (uint32_t step = 0; step < R.cap; step++) {  // the table is at most half full: a free slot is always reached
        unsigned long long s = __ldcg(&R.tab[slot].tag);
        if (s == EMPTY64) {
            s = atomicCAS(&R.tab[slot].tag, EMPTY64, tag);
            if (s == EMPTY64) s = tag;
        }
        if ((uint32_t)(s >> 32) == h) {
            const uint32_t o = (uint32_t)s;
            const uint4 *op = (o < R.n_prev ? R.prev + 4 * (size_t)o : R.cur + 4 * (size_t)(o - R.n_prev));
            const uint4 o2 = op[2];
            if (key_eq(op[0], k0) && key_eq(op[1], k1) && o2.x == k2.x && o2.y == k2.y) {
                if (atomicCAS(is_prev ? &R.tab[slot].prev : &R.tab[slot].cur, EMPTY32, e) != EMPTY32)
                    atomicOr(&R.ctl[0], is_prev ? ERR_DUP_PREV : ERR_DUP_CUR);
                if (!is_prev) R.cslot[e] = slot;
                return;
            }
        }
        slot = (slot + 1) & (R.cap - 1);
    }
    if (!is_prev) R.cslot[e] = EMPTY32;
}

__global__ void __launch_bounds__(RC_THREADS) k_rc_probe(const Rc R) {
    __shared__ unsigned long long s_excl;
    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    const uint32_t base = blockIdx.x * RC_TILE + tid * RC_ITEMS;  // blocked: RC_ITEMS consecutive entries per thread
    uint32_t slot[RC_ITEMS], pj[RC_ITEMS];
#pragma unroll
    for (int k = 0; k < RC_ITEMS; k++) slot[k] = base + k < R.n_cur ? R.cslot[base + k] : EMPTY32;
#pragma unroll
    for (int k = 0; k < RC_ITEMS; k++) pj[k] = slot[k] != EMPTY32 ? __ldcg(&R.tab[slot[k]].prev) : EMPTY32;
    uint32_t st[RC_ITEMS];
    unsigned long long kept_idx[RC_ITEMS];
    uint32_t nonkept = 0, kept = 0, changed = 0;
#pragma unroll
    for (int k = 0; k < RC_ITEMS; k++) {
        st[k] = KXPU_RC_NEW;
        kept_idx[k] = 0;
        if (pj[k] != EMPTY32) {
            const uint4 c2 = R.cur[4 * (size_t)(base + k) + 2], c3 = R.cur[4 * (size_t)(base + k) + 3];
            const uint4 p2 = R.prev[4 * (size_t)pj[k] + 2], p3 = R.prev[4 * (size_t)pj[k] + 3];
            // bytes 40..55: iommu_group, klass, tag
            const bool same = c2.z == p2.z && c2.w == p2.w && c3.x == p3.x && c3.y == p3.y;
            st[k] = same ? KXPU_RC_KEPT : KXPU_RC_CHANGED;
            kept_idx[k] = ((unsigned long long)p3.w << 32) | p3.z;
            R.pstate[pj[k]] = (uint8_t)st[k];
        }
        if (base + k < R.n_cur) {
            nonkept += st[k] != KXPU_RC_KEPT;
            kept += st[k] == KXPU_RC_KEPT;
            changed += st[k] == KXPU_RC_CHANGED;
        }
    }
    uint32_t tot;
    const uint32_t ex = kxscan::block_excl(nonkept, &tot);
    if (tid < 32) {
        const unsigned long long e = kxscan::lookback(R.state, blockIdx.x, tot, R.epoch);
        if (tid == 0) s_excl = e;
    }
    // kept / changed: one atomic per warp
    kept = __reduce_add_sync(0xffffffffu, kept);
    changed = __reduce_add_sync(0xffffffffu, changed);
    if (lane == 0) {
        if (kept) atomicAdd(&R.ctl[1], kept);
        if (changed) atomicAdd(&R.ctl[2], changed);
    }
    __syncthreads();
    unsigned long long run = R.next_index + s_excl + ex;
#pragma unroll
    for (int k = 0; k < RC_ITEMS; k++) {
        if (base + k >= R.n_cur) break;
        R.cstate[base + k] = (uint8_t)st[k];
        if (st[k] == KXPU_RC_KEPT) R.idx[base + k] = kept_idx[k];
        else R.idx[base + k] = run++;
    }
}

}  // namespace kxrc

using namespace kxrc;

extern "C" int32_t kxpu_reconcile(kxpu_ctx *ctx, const kxpu_snaprec *prev, size_t n_prev, uint64_t next_index,
                                  const kxpu_snaprec *cur, size_t n_cur, uint64_t *index_out, uint8_t *cur_state,
                                  uint8_t *prev_state, kxpu_reconcile_counts *counts) {
    static_assert(sizeof(kxpu_snaprec) == 64 && offsetof(kxpu_snaprec, iommu_group) == 40 && offsetof(kxpu_snaprec, tag) == 48 &&
                      offsetof(kxpu_snaprec, index) == 56,
                  "kxpu_snaprec layout");
    if (!ctx || (n_prev && !prev) || (n_cur && (!cur || !index_out))) return KXPU_E_INVALID;
    if (n_prev + n_cur > (1ull << 30) || n_prev > (1ull << 30) || n_cur > (1ull << 30)) return KXPU_E_UNSUPPORTED;
    if (next_index + (uint64_t)n_cur < next_index) {
        KX_SET_ERR(ctx, "reconcile: next_index + n_cur overflows");
        return KXPU_E_INVALID;
    }
    const uint32_t NP = (uint32_t)n_prev, NC = (uint32_t)n_cur, NT = NP + NC;
    if (NT == 0) {
        if (counts) { memset(counts, 0, sizeof *counts); counts->next_index_out = next_index; }
        return KXPU_OK;
    }
    uint32_t cap = 1024;
    while (cap < 2 * NT) cap <<= 1;
    uint32_t lg = 0;
    while ((1u << lg) < cap) lg++;
    const uint32_t tiles = (NC + RC_TILE - 1) / RC_TILE;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_tab = take((size_t)cap * sizeof(RSlot));
    const size_t o_pstate = take(n_prev), o_ctl = take(16);  // memset together: states to RETIRED, then the counters
    const size_t o_prev = take(n_prev * 64), o_cur = take(n_cur * 64);
    const size_t o_cslot = take(n_cur * 4), o_idx = take(n_cur * 8), o_cstate = take(n_cur);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    unsigned long long *state = nullptr;
    if (tiles) {
        state = kx_scan_state(ctx, tiles);
        if (!state) return KXPU_E_NOMEM;
    }
    cudaStream_t s = ctx->stream;
    Rc R;
    R.prev = (const uint4 *)(b + o_prev); R.cur = (const uint4 *)(b + o_cur);
    R.n_prev = NP; R.n_cur = NC; R.next_index = next_index;
    R.tab = (RSlot *)(b + o_tab); R.cap = cap; R.shift = 32 - lg;
    R.cslot = (uint32_t *)(b + o_cslot); R.idx = (unsigned long long *)(b + o_idx);
    R.cstate = b + o_cstate; R.pstate = b + o_pstate; R.ctl = (uint32_t *)(b + o_ctl);
    R.state = state; R.epoch = tiles ? kx_next_epoch(ctx) : 0u;
    if (n_prev) cudaMemcpyAsync(b + o_prev, prev, n_prev * 64, cudaMemcpyHostToDevice, s);
    if (n_cur) cudaMemcpyAsync(b + o_cur, cur, n_cur * 64, cudaMemcpyHostToDevice, s);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        cudaMemsetAsync(b + o_tab, 0xFF, (size_t)cap * sizeof(RSlot), s);
        if (n_prev) cudaMemsetAsync(b + o_pstate, KXPU_RC_RETIRED, n_prev, s);
        cudaMemsetAsync(b + o_ctl, 0, 16, s);
        k_rc_insert<<<(NT + 255) / 256, 256, 0, s>>>(R);
        ctx->launches++;
        if (tiles) {
            k_rc_probe<<<tiles, RC_THREADS, 0, s>>>(R);
            ctx->launches++;
        }
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, R.ctl, 16, cudaMemcpyDeviceToHost, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "reconcile failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) {
        KX_SET_ERR(ctx, "reconcile:%s%s%s%s", (h[0] & ERR_KEY) ? " an empty or badly padded key;" : "",
                   (h[0] & ERR_DUP_PREV) ? " a duplicate key in prev;" : "", (h[0] & ERR_DUP_CUR) ? " a duplicate key in cur;" : "",
                   (h[0] & ERR_INDEX) ? " a prev index >= next_index;" : "");
        return KXPU_E_INVALID;
    }
    const uint64_t kept = h[1], changed = h[2];
    if (n_cur) {
        cudaMemcpyAsync(index_out, R.idx, n_cur * 8, cudaMemcpyDeviceToHost, s);
        if (cur_state) cudaMemcpyAsync(cur_state, R.cstate, n_cur, cudaMemcpyDeviceToHost, s);
    }
    if (n_prev && prev_state) cudaMemcpyAsync(prev_state, R.pstate, n_prev, cudaMemcpyDeviceToHost, s);
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "reconcile D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (counts) {
        counts->n_kept = kept;
        counts->n_changed = changed;
        counts->n_new = n_cur - kept - changed;
        counts->n_retired = n_prev - kept - changed;
        counts->next_index_out = next_index + (n_cur - kept);
    }
    return KXPU_OK;
}
