// scan.cuh -- exclusive prefix sum over uint32, ONE kernel: per-tile reduce + decoupled look-back
// over tile status words + per-item downsweep ("single-pass scan").  Used where output sizes are
// data dependent (name gather, Allocate names, ListAndWatch bytes, busIndex, radix-sort digit bases).
//
// Tile status word (u64): [63:40] call epoch, [39:38] 1 = aggregate / 2 = inclusive prefix,
// [37:0] value.  The words live in a per-ctx buffer that is zeroed when it is allocated or grown
// (kx_scan_state, api.cu) and then only written by these look-backs with increasing epochs: a word
// whose epoch is not the current call's counts as "not published yet", so nothing is cleared between
// calls.  When the 24-bit epoch wraps (kx_next_epoch), the whole buffer is zeroed again.  Both zeroings
// are cudaMemsetAsync on the ctx stream, so they land before the next look-back on that stream reads a
// word.  KXPU_SCAN_EPOCH_LIMIT (2 .. 2^24, read at context creation) moves the wrap down to that limit,
// so that tests can run it often; results do not depend on it.  Tiles are taken in blockIdx order,
// which the hardware dispatches in order (the same assumption CUB's scan makes).
#pragma once
#include "common.cuh"

namespace kxscan {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;                        // per thread
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;  // 4096 items per block

constexpr unsigned long long ST_AGG = 1ull << 38, ST_PFX = 2ull << 38, ST_FLAGS = 3ull << 38, ST_VAL = (1ull << 38) - 1;
constexpr int ST_EPOCH_SHIFT = 40;

__device__ __forceinline__ uint32_t warp_incl(uint32_t v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, v, d);
        if (kx_lane() >= (uint32_t)d) v += y;
    }
    return v;
}

// block-wide exclusive scan of one value per thread (SCAN_THREADS threads); returns exclusive prefix, total in *tot
__device__ __forceinline__ uint32_t block_excl(uint32_t v, uint32_t *tot) {
    __shared__ uint32_t wsum[SCAN_THREADS / 32];
    __shared__ uint32_t total;
    uint32_t incl = warp_incl(v);
    uint32_t w = threadIdx.x >> 5;
    if (kx_lane() == 31) wsum[w] = incl;
    __syncthreads();
    if (w == 0) {
        uint32_t x = kx_lane() < SCAN_THREADS / 32 ? wsum[kx_lane()] : 0;
        uint32_t xi = warp_incl(x);
        if (kx_lane() < SCAN_THREADS / 32) wsum[kx_lane()] = xi - x;
        if (kx_lane() == SCAN_THREADS / 32 - 1) total = xi;
    }
    __syncthreads();
    uint32_t r = wsum[w] + incl - v;
    *tot = total;
    __syncthreads();
    return r;
}

__device__ __forceinline__ unsigned long long ld_state(const unsigned long long *p) {
    return *reinterpret_cast<const volatile unsigned long long *>(p);
}

// Publish this tile's aggregate and return its exclusive prefix (sum of the aggregates of all tiles
// in front of it).  Called by the first warp of the CTA (all 32 lanes); the look-back reads 32
// predecessors per step.  epoch: kx_next_epoch(ctx), 24 bits.
__device__ __forceinline__ unsigned long long lookback(unsigned long long *state, uint32_t tile, unsigned long long aggregate,
                                                       uint32_t epoch) {
    const uint32_t lane = kx_lane();
    const unsigned long long tag = (unsigned long long)(epoch & 0xffffffu) << ST_EPOCH_SHIFT;
    if (lane == 0) {
        *reinterpret_cast<volatile unsigned long long *>(&state[tile]) = tag | (tile == 0 ? ST_PFX : ST_AGG) | (aggregate & ST_VAL);
        kx_fence_gpu();
    }
    unsigned long long excl = 0;
    long long j0 = (long long)tile - 1;  // lane 0 looks at j0, lane 1 at j0 - 1, ...
    while (j0 >= 0) {
        const long long j = j0 - lane;
        unsigned long long v = 0;
        bool ready = true;
        if (j >= 0) {
            v = ld_state(&state[j]);
            ready = (v >> ST_EPOCH_SHIFT) == (tag >> ST_EPOCH_SHIFT) && (v & ST_FLAGS) != 0;
        }
        const uint32_t not_ready = __ballot_sync(0xffffffffu, !ready);
        const uint32_t pfx = __ballot_sync(0xffffffffu, j >= 0 && ready && (v & ST_FLAGS) == ST_PFX);
        // usable window: lanes in front of the first not-ready lane, up to (and including) the first prefix
        const uint32_t first_nr = not_ready ? (uint32_t)__ffs((int)not_ready) - 1u : 32u;
        const uint32_t first_pf = pfx ? (uint32_t)__ffs((int)pfx) - 1u : 32u;
        const uint32_t take = first_pf < first_nr ? first_pf + 1u : first_nr;  // lanes [0, take)
        unsigned long long part = (lane < take && j >= 0) ? (v & ST_VAL) : 0ull;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) part += __shfl_down_sync(0xffffffffu, part, d);
        excl += __shfl_sync(0xffffffffu, part, 0);
        if (first_pf < first_nr) break;  // reached an inclusive prefix
        j0 -= take;                      // take == 0: the nearest predecessor is not there yet -- look again
        if (take == 0) __nanosleep(20);
    }
    if (lane == 0 && tile != 0) {
        *reinterpret_cast<volatile unsigned long long *>(&state[tile]) = tag | ST_PFX | ((excl + aggregate) & ST_VAL);
        kx_fence_gpu();
    }
    return excl;
}

// out[i] = sum of in[0..i); total (optional) = sum of everything.  One launch.
template <typename OutT>
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(const uint32_t *__restrict__ in, size_t n, OutT *__restrict__ out,
                                                            unsigned long long *state, uint32_t epoch,
                                                            unsigned long long *total_out) {
    __shared__ unsigned long long s_excl;
    // blocked arrangement so that each thread owns SCAN_ITEMS consecutive items
    const size_t base = (size_t)blockIdx.x * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint32_t s = 0;
    if (base + SCAN_ITEMS <= n && (reinterpret_cast<uintptr_t>(in + base) & 15u) == 0) {
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; k += 4) {
            const uint4 q = *reinterpret_cast<const uint4 *>(in + base + k);
            v[k] = q.x; v[k + 1] = q.y; v[k + 2] = q.z; v[k + 3] = q.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < SCAN_ITEMS; k++) v[k] = base + k < n ? in[base + k] : 0u;
    }
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) s += v[k];
    uint32_t tot;
    const uint32_t ex = block_excl(s, &tot);
    if (threadIdx.x < 32) {
        const unsigned long long e = lookback(state, blockIdx.x, tot, epoch);
        if (threadIdx.x == 0) {
            s_excl = e;
            if (total_out && blockIdx.x == gridDim.x - 1) *total_out = e + tot;
        }
    }
    __syncthreads();
    unsigned long long run = s_excl + ex;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) {
        if (base + k < n) out[base + k] = (OutT)run;
        run += v[k];
    }
}

// d_total: optional u64 (device).  KXPU_E_NOMEM (ctx->err set, nothing enqueued, d_out untouched) when
// the status words could not be allocated; kx_scan_state has already cleared the CUDA error, so a later
// stream sync does not report it: the caller must return this status.
template <typename OutT>
static inline int32_t exclusive_scan(kxpu_ctx *ctx, const uint32_t *d_in, size_t n, OutT *d_out, unsigned long long *d_total) {
    size_t nb = (n + SCAN_TILE - 1) / SCAN_TILE;
    if (nb == 0) nb = 1;
    unsigned long long *state = kx_scan_state(ctx, nb);
    if (!state) return KXPU_E_NOMEM;
    scan_kernel<OutT><<<(unsigned)nb, SCAN_THREADS, 0, ctx->stream>>>(d_in, n, d_out, state, kx_next_epoch(ctx), d_total);
    ctx->launches += 1;
    return KXPU_OK;
}

}  // namespace kxscan
