// topology.cu -- K8: GetPreferredAllocation over the NUMA masks of the plugin's devices (kxpu_preferred_allocation).
//
// The reference answers nil, nil (generic_device_plugin.go:378-386); include/kxpu.h defines the rule.  Per request,
// with home(d) = lowest set bit of dev_numa[d] (64 when the mask is 0), U = the homes < 64 of the must-include devices
// and c[k] = the number of candidates (available minus must-include) with home k, the bins are ordered by the key
//   (group, -c[k], k),  group 0 = k in U, 1 = other k < 64, 2 = k = 64,
// and the answer is the must-include positions in request order followed by the first r candidates in (bin order,
// position) order.  A candidate's place is therefore base[bin] + (its rank by position inside the bin), base = the
// exclusive prefix of c over the bins in that order.
//
// Two shapes:
//   - k_pref_warp: one warp per request of at most 256 available positions (kubelet's requests are 8-16 devices).
//     The request lives in shared memory; validation, the 65-bin histogram, the bin order and the ranks are all
//     done by the warp with pairwise comparisons (256^2 / 32 steps at most).  One launch for all such requests.
//   - a larger request: k_big_mark marks the available / must-include positions in a per-device word (duplicates and
//     positions past n_devs show up there), k_big_hist counts the candidates per bin, k_big_scatter walks the device
//     positions in 4096-position tiles, ranks the candidates of each bin inside the tile (warp match + per-warp
//     counters, as the classify radix sort does), takes the bin's offset over the tiles in front from a decoupled
//     look-back over per-(tile, bin) status words and scatters the first r.  Walking the positions rather than the
//     request's list is what makes the rank "ascending position" without a sort.
#include <algorithm>

#include "common.cuh"
#include "scan.cuh"

namespace kxtopo {

constexpr uint32_t BINS = KXPU_MAX_NUMA_NODES + 1;  // 64 nodes + "unknown"
constexpr uint32_t WARP_MAX = 256;                  // available positions a warp request can hold
constexpr int PW_WARPS = 8;

__device__ __forceinline__ uint32_t home_of(unsigned long long mask) { return mask ? (uint32_t)__ffsll((long long)mask) - 1u : 64u; }

// order key of bin k (smaller first): group in bits 40-41, ~c in bits 8-39, k in bits 0-7
__device__ __forceinline__ unsigned long long bin_key(uint32_t k, uint32_t c, unsigned long long U) {
    const unsigned long long grp = k == 64u ? 2ull : (((U >> k) & 1ull) ? 0ull : 1ull);
    return (grp << 40) | ((unsigned long long)(0xFFFFFFFFu - c) << 8) | k;
}

struct Req {
    const unsigned long long *dev_numa;
    uint32_t n_devs, n_req;
    const uint32_t *avail_off, *avail, *must_off, *must, *size, *out_off;
    uint32_t *out;
    uint32_t *err;  // [0] = 1 on an invalid request, [1] = lowest invalid request
};

__device__ __forceinline__ void flag_bad(const Req &R, uint32_t q) {
    atomicOr(&R.err[0], 1u);
    atomicMin(&R.err[1], q);
}

// one warp per request with at most WARP_MAX available positions (larger ones are skipped: the big path takes them)
__global__ void __launch_bounds__(PW_WARPS * 32) k_pref_warp(const Req R) {
    __shared__ uint32_t sp[PW_WARPS][WARP_MAX];      // available positions
    __shared__ uint32_t smu[PW_WARPS][WARP_MAX];     // must-include positions
    __shared__ uint8_t sh[PW_WARPS][WARP_MAX];       // home of each available position
    __shared__ uint8_t sf[PW_WARPS][WARP_MAX];       // 1: that available position is also must-include
    __shared__ uint32_t cnt[PW_WARPS][BINS];
    __shared__ unsigned long long bk[PW_WARPS][BINS];
    __shared__ uint32_t base[PW_WARPS][BINS];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * PW_WARPS + w;
    if (q >= R.n_req) return;
    const uint32_t a0 = R.avail_off[q], na = R.avail_off[q + 1] - a0;
    if (na > WARP_MAX) return;
    const uint32_t m0 = R.must_off[q], nm = R.must_off[q + 1] - m0;  // nm <= size <= na (checked by the host)
    const uint32_t o0 = R.out_off[q], r = R.size[q] - nm;
    bool bad = false;
    for (uint32_t j = lane; j < na; j += 32) {
        const uint32_t p = R.avail[a0 + j];
        const bool in = p < R.n_devs;
        bad |= !in;
        sp[w][j] = p;
        sh[w][j] = (uint8_t)(in ? home_of(R.dev_numa[p]) : 64u);
        sf[w][j] = 0;
    }
    for (uint32_t j = lane; j < nm; j += 32) {
        const uint32_t p = R.must[m0 + j];
        smu[w][j] = p;
        R.out[o0 + j] = p;  // must-include first, in request order
    }
    for (uint32_t k = lane; k < BINS; k += 32) cnt[w][k] = 0u;
    __syncwarp();
    // duplicates inside available / inside must-include, must-include within available, U
    unsigned long long U = 0;
    for (uint32_t j = lane; j < na; j += 32)
        for (uint32_t t = 0; t < j; t++) bad |= sp[w][t] == sp[w][j];
    for (uint32_t j = lane; j < nm; j += 32) {
        const uint32_t p = smu[w][j];
        for (uint32_t t = 0; t < j; t++) bad |= smu[w][t] == p;
        uint32_t at = na;
        for (uint32_t t = 0; t < na; t++) at = sp[w][t] == p ? t : at;
        if (at == na) { bad = true; continue; }
        sf[w][at] = 1;
        const uint32_t h = sh[w][at];
        if (h < 64u) U |= 1ull << h;
    }
    const uint32_t ulo = __reduce_or_sync(0xffffffffu, (uint32_t)U), uhi = __reduce_or_sync(0xffffffffu, (uint32_t)(U >> 32));
    U = ((unsigned long long)uhi << 32) | ulo;
    __syncwarp();
    for (uint32_t j = lane; j < na; j += 32)
        if (!sf[w][j]) atomicAdd(&cnt[w][sh[w][j]], 1u);
    __syncwarp();
    for (uint32_t k = lane; k < BINS; k += 32) bk[w][k] = bin_key(k, cnt[w][k], U);
    __syncwarp();
    for (uint32_t k = lane; k < BINS; k += 32) {
        uint32_t b = 0;
        for (uint32_t t = 0; t < BINS; t++) b += bk[w][t] < bk[w][k] ? cnt[w][t] : 0u;
        base[w][k] = b;
    }
    __syncwarp();
    for (uint32_t j = lane; j < na; j += 32) {
        if (sf[w][j]) continue;
        const uint32_t p = sp[w][j], h = sh[w][j];
        uint32_t rk = base[w][h];
        for (uint32_t t = 0; t < na; t++) rk += (!sf[w][t] && sh[w][t] == h && sp[w][t] < p) ? 1u : 0u;
        if (rk < r) R.out[o0 + nm + rk] = p;
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) flag_bad(R, q);
}

// ---------------------------------------------------------------- one large request
struct Big {
    Req R;
    uint32_t q;
    uint32_t *mark;             // [n_devs] bit 0: available, bit 1: must-include (zeroed per request)
    uint32_t *hist;             // [BINS] candidates per bin (zeroed per request)
    unsigned long long *U;      // homes < 64 of the must-include devices (zeroed per request)
    unsigned long long *state;  // [tiles][BINS] look-back status words
    uint32_t epoch;
};

__global__ void __launch_bounds__(256) k_big_mark(const Big B) {
    const Req &R = B.R;
    const uint32_t a0 = R.avail_off[B.q], na = R.avail_off[B.q + 1] - a0;
    const uint32_t m0 = R.must_off[B.q], nm = R.must_off[B.q + 1] - m0, o0 = R.out_off[B.q];
    const uint32_t stride = gridDim.x * blockDim.x;
    bool bad = false;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < na + nm; j += stride) {
        const bool isMust = j >= na;
        const uint32_t p = isMust ? R.must[m0 + j - na] : R.avail[a0 + j];
        if (isMust) R.out[o0 + j - na] = p;
        if (p >= R.n_devs) { bad = true; continue; }
        const uint32_t bit = isMust ? 2u : 1u;
        if (atomicOr(&B.mark[p], bit) & bit) bad = true;  // the same position twice in one list
        if (isMust) {
            const uint32_t h = home_of(R.dev_numa[p]);
            if (h < 64u) atomicOr(B.U, 1ull << h);
        }
    }
    if (bad) flag_bad(R, B.q);
}

__global__ void __launch_bounds__(256) k_big_hist(const Big B) {
    __shared__ uint32_t h[BINS];
    const Req &R = B.R;
    for (uint32_t k = threadIdx.x; k < BINS; k += blockDim.x) h[k] = 0u;
    __syncthreads();
    const uint32_t a0 = R.avail_off[B.q], na = R.avail_off[B.q + 1] - a0;
    const uint32_t m0 = R.must_off[B.q], nm = R.must_off[B.q + 1] - m0;
    const uint32_t stride = gridDim.x * blockDim.x;
    bool bad = false;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < na + nm; j += stride) {
        const bool isMust = j >= na;
        const uint32_t p = isMust ? R.must[m0 + j - na] : R.avail[a0 + j];
        if (p >= R.n_devs) continue;  // flagged by k_big_mark
        const uint32_t m = B.mark[p];
        if (isMust) bad |= !(m & 1u);  // must-include but not available
        else if (m == 1u) atomicAdd(&h[home_of(R.dev_numa[p])], 1u);
    }
    if (bad) flag_bad(R, B.q);
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < BINS; k += blockDim.x)
        if (h[k]) atomicAdd(&B.hist[k], h[k]);
}

constexpr int BS_WARPS = 16;
constexpr int BS_THREADS = BS_WARPS * 32;
constexpr int BS_STEPS = 8;
constexpr int BS_TILE = BS_THREADS * BS_STEPS;  // 4096 device positions per CTA

__global__ void __launch_bounds__(BS_THREADS) k_big_scatter(const Big B) {
    __shared__ uint32_t cnt[BS_WARPS][BINS];
    __shared__ unsigned long long bk[BINS];
    __shared__ uint32_t tbase[BINS];
    const Req &R = B.R;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5, tile = blockIdx.x;
    const unsigned long long U = *B.U;
    const uint32_t nm = R.must_off[B.q + 1] - R.must_off[B.q];
    const uint32_t o0 = R.out_off[B.q] + nm, r = R.size[B.q] - nm;
    for (uint32_t k = lane; k < BINS; k += 32) cnt[w][k] = 0u;
    if (tid < BINS) bk[tid] = bin_key(tid, B.hist[tid], U);
    __syncwarp();
    const uint32_t wbase = tile * BS_TILE + w * (BS_TILE / BS_WARPS);
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t pos[BS_STEPS], bin[BS_STEPS], rk[BS_STEPS];
#pragma unroll
    for (int s = 0; s < BS_STEPS; s++) {
        const uint32_t p = wbase + s * 32u + lane;
        const bool cand = p < R.n_devs && B.mark[p] == 1u;
        const uint32_t d = cand ? home_of(R.dev_numa[p]) : BINS;  // BINS: non-candidates only match each other
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        uint32_t prev = 0;
        if (cand) prev = cnt[w][d];
        __syncwarp();
        if (cand && (peers & lt) == 0u) cnt[w][d] = prev + (uint32_t)__popc(peers);
        __syncwarp();
        pos[s] = p;
        bin[s] = d;
        rk[s] = prev + (uint32_t)__popc(peers & lt);
    }
    __syncthreads();
    if (tid < BINS) {
        // this bin: exclusive scan over the warps, tile count, offset of the bin in the answer
        uint32_t tot = 0;
#pragma unroll
        for (int k = 0; k < BS_WARPS; k++) {
            const uint32_t x = cnt[k][tid];
            cnt[k][tid] = tot;
            tot += x;
        }
        uint32_t gbase = 0;
        for (uint32_t t = 0; t < BINS; t++) gbase += bk[t] < bk[tid] ? B.hist[t] : 0u;
        // look-back over the tiles in front, for this bin
        const unsigned long long tag = (unsigned long long)(B.epoch & 0xffffffu) << kxscan::ST_EPOCH_SHIFT;
        unsigned long long *st = B.state + tid;
        *reinterpret_cast<volatile unsigned long long *>(st + (size_t)tile * BINS) = tag | (tile == 0 ? kxscan::ST_PFX : kxscan::ST_AGG) | tot;
        uint32_t excl = 0;
        for (long long j = (long long)tile - 1; j >= 0;) {
            const unsigned long long v = kxscan::ld_state(st + (size_t)j * BINS);
            if ((v >> kxscan::ST_EPOCH_SHIFT) != (tag >> kxscan::ST_EPOCH_SHIFT) || (v & kxscan::ST_FLAGS) == 0) continue;
            excl += (uint32_t)(v & kxscan::ST_VAL);
            if ((v & kxscan::ST_FLAGS) == kxscan::ST_PFX) break;
            j--;
        }
        if (tile != 0) *reinterpret_cast<volatile unsigned long long *>(st + (size_t)tile * BINS) = tag | kxscan::ST_PFX | (unsigned long long)(excl + tot);
        tbase[tid] = gbase + excl;
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < BS_STEPS; s++) {
        if (bin[s] < BINS) {
            const uint32_t at = tbase[bin[s]] + cnt[w][bin[s]] + rk[s];
            if (at < r) R.out[o0 + at] = pos[s];
        }
    }
}

}  // namespace kxtopo

using namespace kxtopo;

extern "C" int32_t kxpu_preferred_allocation(kxpu_ctx *ctx, const uint64_t *dev_numa, size_t n_devs, const uint32_t *avail_off,
                                             const uint32_t *avail, const uint32_t *must_off, const uint32_t *must,
                                             const uint32_t *size, size_t n_req, uint32_t *out, uint32_t *out_off) {
    if (!ctx || !out_off || (n_req && (!avail_off || !must_off || !size)) || (n_devs && !dev_numa)) return KXPU_E_INVALID;
    if (n_devs >= 0x7FFFFFFFull || n_req >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    // the request layout and the two size rules on the host: O(n_req)
    out_off[0] = 0;
    if (n_req && (avail_off[0] != 0 || must_off[0] != 0)) { KX_SET_ERR(ctx, "preferred_allocation: offsets must start at 0"); return KXPU_E_INVALID; }
    std::vector<uint32_t> big;
    unsigned long long tot = 0;
    for (size_t q = 0; q < n_req; q++) {
        if (avail_off[q + 1] < avail_off[q] || must_off[q + 1] < must_off[q]) {
            KX_SET_ERR(ctx, "preferred_allocation: request %zu: offsets decrease", q);
            return KXPU_E_INVALID;
        }
        const uint32_t na = avail_off[q + 1] - avail_off[q], nm = must_off[q + 1] - must_off[q];
        if (size[q] < nm || size[q] > na) {
            KX_SET_ERR(ctx, "preferred_allocation: request %zu: size %u is below |must| = %u or above |available| = %u", q, size[q], nm, na);
            return KXPU_E_INVALID;
        }
        tot += size[q];
        if (tot >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
        out_off[q + 1] = (uint32_t)tot;
        if (na > WARP_MAX) big.push_back((uint32_t)q);
    }
    const size_t na_all = n_req ? avail_off[n_req] : 0, nm_all = n_req ? must_off[n_req] : 0;
    if (na_all >= 0x7FFFFFFFull || nm_all >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (n_req == 0) return KXPU_OK;
    if ((na_all && !avail) || (nm_all && !must) || (tot && !out)) return KXPU_E_INVALID;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_numa = take(n_devs * 8), o_aoff = take((n_req + 1) * 4), o_avail = take(na_all * 4);
    const size_t o_moff = take((n_req + 1) * 4), o_must = take(nm_all * 4), o_size = take(n_req * 4);
    const size_t o_ooff = take((n_req + 1) * 4), o_out = take((size_t)tot * 4), o_err = take(8);
    const size_t o_mark = big.empty() ? 0 : take(n_devs * 4), o_ctl = big.empty() ? 0 : take(BINS * 4 + 8);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_numa, dev_numa, n_devs * 8); up(o_aoff, avail_off, (n_req + 1) * 4); up(o_avail, avail, na_all * 4);
    up(o_moff, must_off, (n_req + 1) * 4); up(o_must, must, nm_all * 4); up(o_size, size, n_req * 4);
    up(o_ooff, out_off, (n_req + 1) * 4);
    const uint32_t err_init[2] = {0u, 0xFFFFFFFFu};
    up(o_err, err_init, 8);
    Req R;
    R.dev_numa = (const unsigned long long *)(b + o_numa); R.n_devs = (uint32_t)n_devs; R.n_req = (uint32_t)n_req;
    R.avail_off = (const uint32_t *)(b + o_aoff); R.avail = (const uint32_t *)(b + o_avail);
    R.must_off = (const uint32_t *)(b + o_moff); R.must = (const uint32_t *)(b + o_must);
    R.size = (const uint32_t *)(b + o_size); R.out_off = (const uint32_t *)(b + o_ooff);
    R.out = (uint32_t *)(b + o_out); R.err = (uint32_t *)(b + o_err);
    if (big.size() < n_req) {
        k_pref_warp<<<(unsigned)((n_req + PW_WARPS - 1) / PW_WARPS), PW_WARPS * 32, 0, st>>>(R);
        ctx->launches++;
    }
    if (!big.empty()) {
        const uint32_t tiles = (uint32_t)((n_devs + BS_TILE - 1) / BS_TILE);
        unsigned long long *state = kx_scan_state(ctx, (size_t)(tiles ? tiles : 1) * BINS);
        if (!state) return KXPU_E_NOMEM;
        for (uint32_t q : big) {
            Big B;
            B.R = R; B.q = q;
            B.mark = (uint32_t *)(b + o_mark); B.hist = (uint32_t *)(b + o_ctl);
            B.U = (unsigned long long *)(b + o_ctl + (BINS * 4 + 7) / 8 * 8);
            B.state = state; B.epoch = kx_next_epoch(ctx);
            cudaMemsetAsync(b + o_mark, 0, n_devs * 4, st);
            cudaMemsetAsync(b + o_ctl, 0, BINS * 4 + 8 + 8, st);
            const uint32_t items = avail_off[q + 1] - avail_off[q] + must_off[q + 1] - must_off[q];
            const unsigned g = std::min<unsigned>((items + 255) / 256, 4u * ctx->sm_count);
            k_big_mark<<<g, 256, 0, st>>>(B);
            k_big_hist<<<g, 256, 0, st>>>(B);
            if (tiles) k_big_scatter<<<tiles, BS_THREADS, 0, st>>>(B);
            ctx->launches += tiles ? 3 : 2;
        }
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, R.err, 8, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "preferred_allocation failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) {
        KX_SET_ERR(ctx, "preferred_allocation: request %u: a position >= n_devs, a duplicate, or a must-include position that is not available", h[1]);
        return KXPU_E_INVALID;
    }
    if (tot) {
        cudaMemcpyAsync(out, R.out, (size_t)tot * 4, cudaMemcpyDeviceToHost, st);
        e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { KX_SET_ERR(ctx, "preferred_allocation D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    }
    return KXPU_OK;
}
