// topology.cu -- K8 / K10: GetPreferredAllocation over the NUMA masks of the plugin's devices
// (kxpu_preferred_allocation) and, with the PCIe forest of the walk, under as few PCIe switches as it can
// (kxpu_preferred_allocation_pcie).
//
// The reference answers nil, nil (generic_device_plugin.go:378-386); include/kxpu.h defines the rule.  Per request,
// with home(d) = lowest set bit of dev_numa[d] (64 when the mask is 0), U = the homes < 64 of the must-include devices
// and c[k] = the number of candidates (available minus must-include) with home k, the NUMA bins are ordered by the key
//   (group, -c[k], k),  group 0 = k in U, 1 = other k < 64, 2 = k = 64,
// and the answer is the must-include positions in request order followed by the first r candidates in (bin order,
// position) order.  A candidate's place is therefore base[bin] + (its rank by position inside the bin), base = the
// exclusive prefix of c over the bins in that order.
//
// The PCIe call is the same rule with two more steps in front: the subtree X the candidates are taken from (a best fit
// over the forest's nodes; all devices when no node qualifies) and an lca level per candidate (the deepest node it
// shares with a must-include device).  A bin is then (level, home), LEVELS * 65 of them, ordered by level first; c[k]
// counts the candidates in X.  The two calls share every kernel through a policy parameter that fixes the number of
// levels: with one level (NumaBins) the keys are K8's and every step of the subtree and the lca compiles away.
//
// Two shapes:
//   - k_pref_warp: one warp per request of at most 256 available positions (kubelet's requests are 8-16 devices).
//     The request lives in shared memory; validation, the node counts, X, the lca levels, the 65 NUMA counts and the
//     ranks are all done by the warp with pairwise comparisons (256^2 / 32 steps per pass at most).  One launch for
//     all such requests.
//   - a larger request: k_big_mark marks the available / must-include positions in a per-device word (duplicates and
//     positions past n_devs show up there) and, for the PCIe policy, counts available and must-include devices up each
//     device's chain with warp-aggregated atomics; k_pick reduces the qualifying nodes to X under the key's
//     comparator (two launches: per CTA, then over the CTAs); k_big_hist counts the candidates per bin, k_big_scatter
//     walks the device positions in 4096-position tiles, ranks the candidates of each bin inside the tile (warp match +
//     per-warp counters, as the classify radix sort does), takes the bin's offset over the tiles in front from a
//     decoupled look-back over per-(tile, bin) status words and scatters the first r.  Walking the positions rather
//     than the request's list is what makes the rank "ascending position" without a sort.
#include <algorithm>

#include "common.cuh"
#include "scan.cuh"

namespace kxtopo {

constexpr uint32_t NUMA_BINS = KXPU_MAX_NUMA_NODES + 1;  // 64 nodes + "unknown"
constexpr uint32_t WARP_MAX = 256;                       // available positions a warp request can hold
constexpr int MAXD = KXPU_PCIE_MAX_DEPTH;
constexpr uint32_t NO_NODE = KXPU_PCIE_NO_NODE;

struct NumaBins {  // kxpu_preferred_allocation: one level
    static constexpr bool PCIE = false;
    static constexpr uint32_t LEVELS = 1;
    static constexpr int WARPS = 8;
};
struct PcieBins {  // kxpu_preferred_allocation_pcie: lca depth 7 .. 0, then "none"
    static constexpr bool PCIE = true;
    static constexpr uint32_t LEVELS = MAXD + 1;
    static constexpr int WARPS = 2;  // the ancestor table takes 8 KB of shared memory per warp
};

__device__ __forceinline__ uint32_t home_of(unsigned long long mask) { return mask ? (uint32_t)__ffsll((long long)mask) - 1u : 64u; }

// order key of NUMA bin k (smaller first): group in bits 40-41, ~c in bits 8-39, k in bits 0-7
__device__ __forceinline__ unsigned long long bin_key(uint32_t k, uint32_t c, unsigned long long U) {
    const unsigned long long grp = k == 64u ? 2ull : (((U >> k) & 1ull) ? 0ull : 1ull);
    return (grp << 40) | ((unsigned long long)(0xFFFFFFFFu - c) << 8) | k;
}
// level in bits 42-45 in front of it
__device__ __forceinline__ unsigned long long level_key(uint32_t lvl, uint32_t k, uint32_t c, unsigned long long U) {
    return ((unsigned long long)lvl << 42) | bin_key(k, c, U);
}

struct Req {
    const unsigned long long *dev_numa;
    uint32_t n_devs, n_req;
    const uint32_t *avail_off, *avail, *must_off, *must, *size, *out_off;
    uint32_t *out;
    uint32_t *err;  // [0] = 1 on an invalid request, [1] = lowest invalid request, [2] = 1 on an invalid forest
    // the forest (PcieBins only)
    const uint32_t *dev_node, *parent;
    const uint8_t *depth;
    uint32_t n_nodes;
};

__device__ __forceinline__ void flag_bad(const Req &R, uint32_t q) {
    atomicOr(&R.err[0], 1u);
    atomicMin(&R.err[1], q);
}

// ancestors of device p's node, anc[t] = the node at depth t for t <= the returned depth (-1: no node, or a forest
// that breaks off -- then k_forest_check has flagged it)
__device__ __forceinline__ int chain_of(const Req &R, uint32_t p, uint32_t *anc) {
    uint32_t v = p < R.n_devs ? R.dev_node[p] : NO_NODE;
    if (v >= R.n_nodes) return -1;
    const int D = R.depth[v];
    if (D >= MAXD) return -1;
    for (int t = D; t >= 0; t--) {
        anc[t] = v;
        if (t == 0) break;
        v = R.parent[v];
        if (v >= R.n_nodes) return -1;
    }
    return D;
}

// the forest rules of kxpu_preferred_allocation_pcie
__global__ void __launch_bounds__(256) k_forest_check(const Req R) {
    const uint32_t stride = gridDim.x * blockDim.x, m = max(R.n_devs, R.n_nodes);
    bool bad = false;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
        if (i < R.n_nodes) {
            const uint32_t p = R.parent[i], d = R.depth[i];
            bad |= d >= (uint32_t)MAXD || (p == NO_NODE ? d != 0u : (p >= i || d != R.depth[p] + 1u));
        }
        if (i < R.n_devs) {
            const uint32_t v = R.dev_node[i];
            bad |= v != NO_NODE && v >= R.n_nodes;
        }
    }
    if (bad) atomicOr(&R.err[2], 1u);
}

// a qualifying node as the warp shape sees it: avail, depth, the avail of its ancestors (anc[t], t < depth), the lowest
// available position in it and its id.  depth -1: none
struct NodeKey {
    uint32_t a, anc[MAXD], mn, node;
    int d;
};
// strictly smaller key (include/kxpu.h: avail, -depth, the ancestors' avail from the parent up, lowest position)
__device__ __forceinline__ bool key_less(const NodeKey &x, const NodeKey &y) {
    if (x.d < 0) return false;
    if (y.d < 0) return true;
    if (x.a != y.a) return x.a < y.a;
    if (x.d != y.d) return x.d > y.d;
    int decided = 0;  // -1: x smaller, 1: y smaller
#pragma unroll
    for (int t = MAXD - 1; t >= 0; t--)
        if (t < x.d && !decided && x.anc[t] != y.anc[t]) decided = x.anc[t] < y.anc[t] ? -1 : 1;
    if (decided) return decided < 0;
    return x.mn < y.mn;
}

// one warp per request with at most WARP_MAX available positions (larger ones are skipped: the big path takes them)
template <class P>
__global__ void __launch_bounds__(P::WARPS * 32) k_pref_warp(const Req R) {
    constexpr int W = P::WARPS;
    constexpr int AW = P::PCIE ? W : 1, AN = P::PCIE ? (int)WARP_MAX : 1;
    __shared__ uint32_t sp[W][WARP_MAX];            // available positions
    __shared__ uint32_t smu[W][WARP_MAX];           // must-include positions
    __shared__ uint8_t sh[W][WARP_MAX];             // home of each available position
    __shared__ uint8_t sf[W][WARP_MAX];             // bit 0: also must-include; bit 1: a candidate (in X)
    __shared__ unsigned long long sk[W][WARP_MAX];  // order key of each candidate's bin
    __shared__ uint32_t cnt[W][NUMA_BINS];
    __shared__ uint32_t sanc[AW][AN][MAXD];         // ancestors of each available position's node
    __shared__ int8_t sdep[AW][AN];                 // depth of that node, -1: none
    __shared__ uint8_t slvl[AW][AN];                // lca level: 7 - lca depth, MAXD = none
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * W + w;
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
        if constexpr (P::PCIE) {
            sdep[w][j] = (int8_t)chain_of(R, p, sanc[w][j]);
            slvl[w][j] = MAXD;
        }
    }
    for (uint32_t j = lane; j < nm; j += 32) {
        const uint32_t p = R.must[m0 + j];
        smu[w][j] = p;
        R.out[o0 + j] = p;  // must-include first, in request order
    }
    for (uint32_t k = lane; k < NUMA_BINS; k += 32) cnt[w][k] = 0u;
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
    // X: the best qualifying node over the chains of the available positions (pairwise: the positions sharing each
    // of my ancestors), and each position's lca level
    int xd = -1;
    uint32_t xnode = NO_NODE;
    if constexpr (P::PCIE) {
        NodeKey best = {};
        best.d = -1;
        const uint32_t want = R.size[q];
        for (uint32_t j = lane; j < na; j += 32) {
            const int D = sdep[w][j];
            if (D < 0) continue;
            uint32_t mine[MAXD], cA[MAXD], cM[MAXD], mn[MAXD];
#pragma unroll
            for (int t = 0; t < MAXD; t++) { mine[t] = t <= D ? sanc[w][j][t] : NO_NODE; cA[t] = 0; cM[t] = 0; mn[t] = 0xFFFFFFFFu; }
            for (uint32_t k = 0; k < na; k++) {
                const int Dk = sdep[w][k];
                int m = -1;
#pragma unroll
                for (int t = 0; t < MAXD; t++)
                    if (t <= D && t <= Dk && sanc[w][k][t] == mine[t]) m = t;
                const uint32_t mk = sf[w][k] & 1u, pk = sp[w][k];
#pragma unroll
                for (int t = 0; t < MAXD; t++)
                    if (t <= m) { cA[t]++; cM[t] += mk; mn[t] = min(mn[t], pk); }
            }
            uint32_t lvl = MAXD;
#pragma unroll
            for (int t = 0; t < MAXD; t++) {
                if (t > D) continue;
                if (cM[t]) lvl = MAXD - 1 - t;
                if (cM[t] == nm && cA[t] >= want) {
                    NodeKey c;
                    c.a = cA[t]; c.d = t; c.mn = mn[t]; c.node = mine[t];
#pragma unroll
                    for (int u = 0; u < MAXD; u++) c.anc[u] = cA[u];
                    if (key_less(c, best)) best = c;
                }
            }
            slvl[w][j] = (uint8_t)lvl;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            NodeKey o;
            o.a = __shfl_xor_sync(0xffffffffu, best.a, off);
            o.d = __shfl_xor_sync(0xffffffffu, best.d, off);
            o.mn = __shfl_xor_sync(0xffffffffu, best.mn, off);
            o.node = __shfl_xor_sync(0xffffffffu, best.node, off);
#pragma unroll
            for (int u = 0; u < MAXD; u++) o.anc[u] = __shfl_xor_sync(0xffffffffu, best.anc[u], off);
            if (key_less(o, best)) best = o;
        }
        xd = best.d;
        xnode = best.node;
        __syncwarp();
    }
    for (uint32_t j = lane; j < na; j += 32) {
        if (sf[w][j]) continue;
        if constexpr (P::PCIE)
            if (xd >= 0 && (sdep[w][j] < xd || sanc[w][j][xd] != xnode)) continue;
        sf[w][j] = 2;
        atomicAdd(&cnt[w][sh[w][j]], 1u);
    }
    __syncwarp();
    for (uint32_t j = lane; j < na; j += 32) {
        if (sf[w][j] != 2) continue;
        const uint32_t h = sh[w][j];
        uint32_t lvl = 0;
        if constexpr (P::PCIE) lvl = slvl[w][j];
        sk[w][j] = level_key(lvl, h, cnt[w][h], U);
    }
    __syncwarp();
    for (uint32_t j = lane; j < na; j += 32) {
        if (sf[w][j] != 2) continue;
        const uint32_t p = sp[w][j];
        const unsigned long long kj = sk[w][j];
        uint32_t rk = 0;
        for (uint32_t t = 0; t < na; t++)
            rk += (sf[w][t] == 2 && (sk[w][t] < kj || (sk[w][t] == kj && sp[w][t] < p))) ? 1u : 0u;
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
    // PcieBins only
    uint32_t *navail, *nmust, *nmin;  // [n_nodes] available / must-include devices in the node, lowest available position
    uint16_t *bin;                    // [n_devs] bin of each candidate, BINS outside X (written by k_big_hist)
    uint32_t *pick;                   // [pick CTAs] best node of each CTA of k_pick
    uint32_t *x;                      // X, NO_NODE: all devices (set to NO_NODE per request)
};

template <class P>
__global__ void __launch_bounds__(256) k_big_mark(const Big B) {
    const Req &R = B.R;
    const uint32_t a0 = R.avail_off[B.q], na = R.avail_off[B.q + 1] - a0;
    const uint32_t m0 = R.must_off[B.q], nm = R.must_off[B.q + 1] - m0, o0 = R.out_off[B.q];
    const uint32_t stride = gridDim.x * blockDim.x, lane = threadIdx.x & 31u;
    bool bad = false;
    // warp-uniform trip count: the PCIe counts below aggregate over the whole warp
    for (uint32_t j0 = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; j0 < na + nm; j0 += stride) {
        const uint32_t j = j0 + lane;
        const bool active = j < na + nm, isMust = j >= na;
        uint32_t p = 0xFFFFFFFFu;
        if (active) {
            p = isMust ? R.must[m0 + j - na] : R.avail[a0 + j];
            if (isMust) R.out[o0 + j - na] = p;
            if (p >= R.n_devs) {
                bad = true;
            } else {
                const uint32_t bit = isMust ? 2u : 1u;
                if (atomicOr(&B.mark[p], bit) & bit) bad = true;  // the same position twice in one list
                if (isMust) {
                    const uint32_t h = home_of(R.dev_numa[p]);
                    if (h < 64u) atomicOr(B.U, 1ull << h);
                }
            }
        }
        if constexpr (P::PCIE) {
            // up the chain by depth, 7 .. 0, so that the lanes under one node meet at every level (the roots take
            // one atomic per warp and kind)
            uint32_t anc[MAXD];
            const int D = active ? chain_of(R, p, anc) : -1;
#pragma unroll
            for (int t = MAXD - 1; t >= 0; t--) {
                const uint32_t v = t <= D ? anc[t] : NO_NODE;
                const uint32_t tag = v == NO_NODE ? NO_NODE : (v | (isMust ? 0x80000000u : 0u));
                const uint32_t peers = __match_any_sync(0xffffffffu, tag);
                if (v == NO_NODE) continue;
                const bool leader = lane == (uint32_t)__ffs((int)peers) - 1u;
                if (isMust) {
                    if (leader) atomicAdd(&B.nmust[v], (uint32_t)__popc(peers));
                } else {
                    const uint32_t lo = __reduce_min_sync(peers, p);
                    if (leader) { atomicAdd(&B.navail[v], (uint32_t)__popc(peers)); atomicMin(&B.nmin[v], lo); }
                }
            }
        }
    }
    if (bad) flag_bad(R, B.q);
}

// strictly smaller key of two nodes from the counts of k_big_mark (NO_NODE: worst)
__device__ __forceinline__ bool node_less(const Big &B, uint32_t u, uint32_t v) {
    if (u == NO_NODE) return false;
    if (v == NO_NODE) return true;
    const uint32_t au = B.navail[u], av = B.navail[v];
    if (au != av) return au < av;
    const uint32_t du = B.R.depth[u], dv = B.R.depth[v];
    if (du != dv) return du > dv;
    uint32_t pu = u, pv = v;
    for (uint32_t t = du; t > 0; t--) {
        pu = B.R.parent[pu];
        pv = B.R.parent[pv];
        if (pu >= B.R.n_nodes || pv >= B.R.n_nodes) break;  // a broken forest (flagged by k_forest_check)
        const uint32_t x = B.navail[pu], y = B.navail[pv];
        if (x != y) return x < y;
    }
    return B.nmin[u] < B.nmin[v];
}

constexpr int PICK_THREADS = 256;

// list == nullptr: the nodes 0 .. count-1; else the nodes list[0 .. count).  out[blockIdx.x] = the smallest qualifying one
__global__ void __launch_bounds__(PICK_THREADS) k_pick(const Big B, const uint32_t *list, uint32_t count, uint32_t *out) {
    __shared__ uint32_t wb[PICK_THREADS / 32];
    const Req &R = B.R;
    const uint32_t nm = R.must_off[B.q + 1] - R.must_off[B.q], want = R.size[B.q];
    uint32_t best = NO_NODE;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
        const uint32_t v = list ? list[i] : i;
        if (v == NO_NODE || B.nmust[v] != nm || B.navail[v] < want) continue;
        if (node_less(B, v, best)) best = v;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const uint32_t o = __shfl_xor_sync(0xffffffffu, best, off);
        if (node_less(B, o, best)) best = o;
    }
    if ((threadIdx.x & 31u) == 0) wb[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t b = wb[0];
        for (int k = 1; k < PICK_THREADS / 32; k++)
            if (node_less(B, wb[k], b)) b = wb[k];
        out[blockIdx.x] = b;
    }
}

template <class P>
__global__ void __launch_bounds__(256) k_big_hist(const Big B) {
    constexpr uint32_t BINS = P::LEVELS * NUMA_BINS;
    __shared__ uint32_t h[BINS];
    const Req &R = B.R;
    for (uint32_t k = threadIdx.x; k < BINS; k += blockDim.x) h[k] = 0u;
    __syncthreads();
    const uint32_t a0 = R.avail_off[B.q], na = R.avail_off[B.q + 1] - a0;
    const uint32_t m0 = R.must_off[B.q], nm = R.must_off[B.q + 1] - m0;
    const uint32_t stride = gridDim.x * blockDim.x;
    uint32_t x = NO_NODE;
    if constexpr (P::PCIE) x = *B.x;
    bool bad = false;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < na + nm; j += stride) {
        const bool isMust = j >= na;
        const uint32_t p = isMust ? R.must[m0 + j - na] : R.avail[a0 + j];
        if (p >= R.n_devs) continue;  // flagged by k_big_mark
        const uint32_t m = B.mark[p];
        if (isMust) { bad |= !(m & 1u); continue; }  // must-include but not available
        if (m != 1u) continue;
        uint32_t b = home_of(R.dev_numa[p]);
        if constexpr (P::PCIE) {
            // in X, and the deepest ancestor holding a must-include device
            uint32_t anc[MAXD];
            const int D = chain_of(R, p, anc);
            bool inX = x == NO_NODE;
            int lca = -1;
#pragma unroll
            for (int t = MAXD - 1; t >= 0; t--) {
                if (t > D) continue;
                inX |= anc[t] == x;
                if (lca < 0 && B.nmust[anc[t]]) lca = t;
            }
            b = inX ? (lca < 0 ? (uint32_t)MAXD : (uint32_t)(MAXD - 1 - lca)) * NUMA_BINS + b : BINS;
            B.bin[p] = (uint16_t)b;
        }
        if (b < BINS) atomicAdd(&h[b], 1u);
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

template <class P>
__global__ void __launch_bounds__(BS_THREADS) k_big_scatter(const Big B) {
    constexpr uint32_t BINS = P::LEVELS * NUMA_BINS;
    __shared__ uint32_t cnt[BS_WARPS][BINS];
    __shared__ unsigned long long bk[BINS];
    __shared__ uint32_t tbase[BINS];
    const Req &R = B.R;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5, tile = blockIdx.x;
    const unsigned long long U = *B.U;
    const uint32_t nm = R.must_off[B.q + 1] - R.must_off[B.q];
    const uint32_t o0 = R.out_off[B.q] + nm, r = R.size[B.q] - nm;
    for (uint32_t k = lane; k < BINS; k += 32) cnt[w][k] = 0u;
    for (uint32_t b = tid; b < BINS; b += BS_THREADS) {
        const uint32_t k = b % NUMA_BINS;
        uint32_t c = 0;  // candidates with home k over all levels
        for (uint32_t l = 0; l < P::LEVELS; l++) c += B.hist[l * NUMA_BINS + k];
        bk[b] = level_key(b / NUMA_BINS, k, c, U);
    }
    __syncwarp();
    const uint32_t wbase = tile * BS_TILE + w * (BS_TILE / BS_WARPS);
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t pos[BS_STEPS], bin[BS_STEPS], rk[BS_STEPS];
#pragma unroll
    for (int s = 0; s < BS_STEPS; s++) {
        const uint32_t p = wbase + s * 32u + lane;
        const bool cand = p < R.n_devs && B.mark[p] == 1u;
        uint32_t d = BINS;  // BINS: non-candidates only match each other
        if (cand) {
            if constexpr (P::PCIE) d = B.bin[p];
            else d = home_of(R.dev_numa[p]);
        }
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        uint32_t prev = 0;
        if (d < BINS) prev = cnt[w][d];
        __syncwarp();
        if (d < BINS && (peers & lt) == 0u) cnt[w][d] = prev + (uint32_t)__popc(peers);
        __syncwarp();
        pos[s] = p;
        bin[s] = d;
        rk[s] = prev + (uint32_t)__popc(peers & lt);
    }
    __syncthreads();
    // per bin: exclusive scan over the warps and the tile count; publish every aggregate of this thread before the
    // first look-back, so that a thread holding two bins never keeps a later tile waiting on its second
    // (between the two loops tbase[b] holds the tile count: each bin belongs to one thread)
    const unsigned long long tag = (unsigned long long)(B.epoch & 0xffffffu) << kxscan::ST_EPOCH_SHIFT;
    for (uint32_t b = tid; b < BINS; b += BS_THREADS) {
        uint32_t t = 0;
#pragma unroll
        for (int k = 0; k < BS_WARPS; k++) {
            const uint32_t x = cnt[k][b];
            cnt[k][b] = t;
            t += x;
        }
        tbase[b] = t;
        *reinterpret_cast<volatile unsigned long long *>(B.state + (size_t)tile * BINS + b) =
            tag | (tile == 0 ? kxscan::ST_PFX : kxscan::ST_AGG) | t;
    }
    for (uint32_t b = tid; b < BINS; b += BS_THREADS) {
        const uint32_t tot = tbase[b];
        uint32_t gbase = 0;  // offset of the bin in the answer
        for (uint32_t t = 0; t < BINS; t++) gbase += bk[t] < bk[b] ? B.hist[t] : 0u;
        // look-back over the tiles in front, for this bin
        unsigned long long *st = B.state + b;
        uint32_t excl = 0;
        for (long long j = (long long)tile - 1; j >= 0;) {
            const unsigned long long v = kxscan::ld_state(st + (size_t)j * BINS);
            if ((v >> kxscan::ST_EPOCH_SHIFT) != (tag >> kxscan::ST_EPOCH_SHIFT) || (v & kxscan::ST_FLAGS) == 0) continue;
            excl += (uint32_t)(v & kxscan::ST_VAL);
            if ((v & kxscan::ST_FLAGS) == kxscan::ST_PFX) break;
            j--;
        }
        if (tile != 0) *reinterpret_cast<volatile unsigned long long *>(st + (size_t)tile * BINS) = tag | kxscan::ST_PFX | (unsigned long long)(excl + tot);
        tbase[b] = gbase + excl;
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

// the whole call; dev_node == nullptr for NumaBins
template <class P>
static int32_t preferred_allocation(kxpu_ctx *ctx, const uint64_t *dev_numa, const uint32_t *dev_node, size_t n_devs,
                                    const uint32_t *parent, const uint8_t *depth, size_t n_nodes, const uint32_t *avail_off,
                                    const uint32_t *avail, const uint32_t *must_off, const uint32_t *must, const uint32_t *size,
                                    size_t n_req, uint32_t *out, uint32_t *out_off) {
    constexpr uint32_t BINS = P::LEVELS * NUMA_BINS;
    const char *fn = P::PCIE ? "preferred_allocation_pcie" : "preferred_allocation";
    // the request layout and the two size rules on the host: O(n_req)
    out_off[0] = 0;
    if (n_req && (avail_off[0] != 0 || must_off[0] != 0)) { KX_SET_ERR(ctx, "%s: offsets must start at 0", fn); return KXPU_E_INVALID; }
    std::vector<uint32_t> big;
    unsigned long long tot = 0;
    for (size_t q = 0; q < n_req; q++) {
        if (avail_off[q + 1] < avail_off[q] || must_off[q + 1] < must_off[q]) {
            KX_SET_ERR(ctx, "%s: request %zu: offsets decrease", fn, q);
            return KXPU_E_INVALID;
        }
        const uint32_t na = avail_off[q + 1] - avail_off[q], nm = must_off[q + 1] - must_off[q];
        if (size[q] < nm || size[q] > na) {
            KX_SET_ERR(ctx, "%s: request %zu: size %u is below |must| = %u or above |available| = %u", fn, q, size[q], nm, na);
            return KXPU_E_INVALID;
        }
        tot += size[q];
        if (tot >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
        out_off[q + 1] = (uint32_t)tot;
        if (na > WARP_MAX) big.push_back((uint32_t)q);
    }
    const size_t na_all = n_req ? avail_off[n_req] : 0, nm_all = n_req ? must_off[n_req] : 0;
    if (na_all >= 0x7FFFFFFFull || nm_all >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (n_req == 0 && !P::PCIE) return KXPU_OK;  // the PCIe call still checks its forest
    if ((na_all && !avail) || (nm_all && !must) || (tot && !out)) return KXPU_E_INVALID;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_numa = take(n_devs * 8), o_aoff = take((n_req + 1) * 4), o_avail = take(na_all * 4);
    const size_t o_moff = take((n_req + 1) * 4), o_must = take(nm_all * 4), o_size = take(n_req * 4);
    const size_t o_ooff = take((n_req + 1) * 4), o_out = take((size_t)tot * 4), o_err = take(16);
    const size_t o_mark = big.empty() ? 0 : take(n_devs * 4), o_ctl = big.empty() ? 0 : take(BINS * 4 + 8);
    const size_t o_node = P::PCIE ? take(n_devs * 4) : 0, o_parent = P::PCIE ? take(n_nodes * 4) : 0;
    const size_t o_depth = P::PCIE ? take(n_nodes) : 0;
    const unsigned pick_ctas = (unsigned)std::min<size_t>((n_nodes + PICK_THREADS - 1) / PICK_THREADS, 2u * (unsigned)ctx->sm_count);
    const bool big_pcie = P::PCIE && !big.empty();
    const size_t o_counts = big_pcie ? take(n_nodes * 12) : 0, o_bin = big_pcie ? take(n_devs * 2) : 0;
    const size_t o_pick = big_pcie ? take((size_t)pick_ctas * 4 + 4) : 0;
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_numa, dev_numa, n_devs * 8);
    if (n_req) {
        up(o_aoff, avail_off, (n_req + 1) * 4); up(o_avail, avail, na_all * 4);
        up(o_moff, must_off, (n_req + 1) * 4); up(o_must, must, nm_all * 4); up(o_size, size, n_req * 4);
        up(o_ooff, out_off, (n_req + 1) * 4);
    }
    const uint32_t err_init[4] = {0u, 0xFFFFFFFFu, 0u, 0u};
    up(o_err, err_init, 16);
    Req R;
    R.dev_numa = (const unsigned long long *)(b + o_numa); R.n_devs = (uint32_t)n_devs; R.n_req = (uint32_t)n_req;
    R.avail_off = (const uint32_t *)(b + o_aoff); R.avail = (const uint32_t *)(b + o_avail);
    R.must_off = (const uint32_t *)(b + o_moff); R.must = (const uint32_t *)(b + o_must);
    R.size = (const uint32_t *)(b + o_size); R.out_off = (const uint32_t *)(b + o_ooff);
    R.out = (uint32_t *)(b + o_out); R.err = (uint32_t *)(b + o_err);
    R.dev_node = nullptr; R.parent = nullptr; R.depth = nullptr; R.n_nodes = 0;
    if constexpr (P::PCIE) {
        up(o_node, dev_node, n_devs * 4); up(o_parent, parent, n_nodes * 4); up(o_depth, depth, n_nodes);
        R.dev_node = (const uint32_t *)(b + o_node); R.parent = (const uint32_t *)(b + o_parent);
        R.depth = (const uint8_t *)(b + o_depth); R.n_nodes = (uint32_t)n_nodes;
        const size_t m = std::max(n_devs, n_nodes);
        if (m) {
            k_forest_check<<<(unsigned)std::min<size_t>((m + 255) / 256, 4u * (unsigned)ctx->sm_count), 256, 0, st>>>(R);
            ctx->launches++;
        }
    }
    if (big.size() < n_req) {
        k_pref_warp<P><<<(unsigned)((n_req + P::WARPS - 1) / P::WARPS), P::WARPS * 32, 0, st>>>(R);
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
            B.navail = (uint32_t *)(b + o_counts); B.nmust = B.navail + n_nodes; B.nmin = B.nmust + n_nodes;
            B.bin = (uint16_t *)(b + o_bin); B.x = (uint32_t *)(b + o_pick); B.pick = B.x + 1;
            cudaMemsetAsync(b + o_mark, 0, n_devs * 4, st);
            cudaMemsetAsync(b + o_ctl, 0, BINS * 4 + 8 + 8, st);
            if (big_pcie) {
                cudaMemsetAsync(b + o_counts, 0, n_nodes * 8, st);
                cudaMemsetAsync(b + o_counts + n_nodes * 8, 0xFF, n_nodes * 4, st);
                cudaMemsetAsync(b + o_pick, 0xFF, 4, st);
            }
            const uint32_t items = avail_off[q + 1] - avail_off[q] + must_off[q + 1] - must_off[q];
            const unsigned g = std::min<unsigned>((items + 255) / 256, 4u * ctx->sm_count);
            k_big_mark<P><<<g, 256, 0, st>>>(B);
            ctx->launches++;
            if (big_pcie && pick_ctas) {
                k_pick<<<pick_ctas, PICK_THREADS, 0, st>>>(B, nullptr, (uint32_t)n_nodes, B.pick);
                k_pick<<<1, PICK_THREADS, 0, st>>>(B, B.pick, pick_ctas, B.x);
                ctx->launches += 2;
            }
            k_big_hist<P><<<g, 256, 0, st>>>(B);
            if (tiles) k_big_scatter<P><<<tiles, BS_THREADS, 0, st>>>(B);
            ctx->launches += tiles ? 2 : 1;
        }
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, R.err, 16, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s failed: %s", fn, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[2]) {
        KX_SET_ERR(ctx, "%s: invalid forest: a device node >= n_nodes, a parent not below its child, or a depth that is not the parent's + 1 (0 for a root) or is >= %d", fn, MAXD);
        return KXPU_E_INVALID;
    }
    if (h[0]) {
        KX_SET_ERR(ctx, "%s: request %u: a position >= n_devs, a duplicate, or a must-include position that is not available", fn, h[1]);
        return KXPU_E_INVALID;
    }
    if (tot) {
        cudaMemcpyAsync(out, R.out, (size_t)tot * 4, cudaMemcpyDeviceToHost, st);
        e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s D2H failed: %s", fn, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    }
    return KXPU_OK;
}

}  // namespace kxtopo

using namespace kxtopo;

extern "C" int32_t kxpu_preferred_allocation(kxpu_ctx *ctx, const uint64_t *dev_numa, size_t n_devs, const uint32_t *avail_off,
                                             const uint32_t *avail, const uint32_t *must_off, const uint32_t *must,
                                             const uint32_t *size, size_t n_req, uint32_t *out, uint32_t *out_off) {
    if (!ctx || !out_off || (n_req && (!avail_off || !must_off || !size)) || (n_devs && !dev_numa)) return KXPU_E_INVALID;
    if (n_devs >= 0x7FFFFFFFull || n_req >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    return preferred_allocation<NumaBins>(ctx, dev_numa, nullptr, n_devs, nullptr, nullptr, 0, avail_off, avail, must_off,
                                          must, size, n_req, out, out_off);
}

extern "C" int32_t kxpu_preferred_allocation_pcie(kxpu_ctx *ctx, const uint64_t *dev_numa, const uint32_t *dev_node,
                                                  size_t n_devs, const uint32_t *parent, const uint8_t *depth, size_t n_nodes,
                                                  const uint32_t *avail_off, const uint32_t *avail, const uint32_t *must_off,
                                                  const uint32_t *must, const uint32_t *size, size_t n_req, uint32_t *out,
                                                  uint32_t *out_off) {
    if (!ctx || !out_off || (n_req && (!avail_off || !must_off || !size)) || (n_devs && !dev_numa)) return KXPU_E_INVALID;
    if (n_nodes && (!parent || !depth)) return KXPU_E_INVALID;
    if (n_devs >= 0x7FFFFFFFull || n_req >= 0x7FFFFFFFull || n_nodes >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (!dev_node)
        return preferred_allocation<NumaBins>(ctx, dev_numa, nullptr, n_devs, nullptr, nullptr, 0, avail_off, avail, must_off,
                                              must, size, n_req, out, out_off);
    return preferred_allocation<PcieBins>(ctx, dev_numa, dev_node, n_devs, parent, depth, n_nodes, avail_off, avail, must_off,
                                          must, size, n_req, out, out_off);
}
