// reset.cu -- K16: can VFIO reset every member of each group between tenants (kxpu_reset_check).  include/kxpu.h states
// the rule.
//
// Five launches, one table keyed by the parent bridges:
//   - kx_pcie_parse: kxpu_pcie_tree's path parse gives every record's chain (node keys, root first).
//   - k_rs_parse: one thread per record.  Five 16-byte vector loads of its kxpu_resetrec; reset_method is cut into pieces
//     at ' ' in registers and each piece compared with the seven names, into methods[i].  When the last key of its chain
//     is a function (a bridge), the key is inserted into an open-addressing table of u64 slots (CAS on an empty slot).
//     The table has at least two slots per record, so a probe sequence always ends.
//   - k_rs_fold: one thread per record with a chain.  For every function key of its chain found in the table it lowers
//     the slot's `bad` word to its index when it is not class-bound (atomic min), else folds (iommu_group << 32 | index)
//     into the slot's `lo` (atomic min) and (iommu_group << 32 | ~index) into its `hi` (atomic max): the lowest and
//     highest group under the bridge, each with the lowest index that carries it.
//   - k_rs_verdict: one thread per record reads its parent's slot into set_verdict[i].
//   - k_rs_group: one thread per group member finds its group ordinal by binary search over group_off and lowers
//     group_reset[o] (all ones from a memset) to its index with an atomic min when it has no reset; a member index >= n
//     sets the error word instead.
#include "common.cuh"

namespace kxreset {

constexpr unsigned long long EMPTY = ~0ull;  // a host-bridge key, so never a bridge's
constexpr unsigned long long HOST_BRIDGE = 1ull << 63;
constexpr uint32_t NONE = ~0u;
constexpr int MAXD = KXPU_PCIE_MAX_DEPTH;

struct Drivers {
    unsigned long long d0[KXPU_MAX_RULES], d1[KXPU_MAX_RULES], m0[KXPU_MAX_RULES], m1[KXPU_MAX_RULES];
    uint32_t n;
};

struct Work {
    const kxpu_devrec *recs;
    const kxpu_resetrec *rrs;
    uint32_t n, allow;
    const unsigned long long *chain;  // [n * MAXD]
    const uint8_t *clen;              // [n]
    unsigned long long *keys;         // [mask + 1] the table: a bridge's key
    uint32_t *bad;                    //   the lowest record below it that is not class-bound, or NONE
    unsigned long long *lo, *hi;      //   the lowest / highest (group, index) pair below it
    uint32_t mask;
    uint8_t *methods;
    uint32_t *set_verdict;
    const uint32_t *goff, *gmem;
    uint32_t G, m0, m1;  // members [m0, m1) = [goff[0], goff[G])
    uint32_t *group_reset;
    uint32_t *err;       // [0] = 1: a member index >= n
};

struct Name {
    unsigned long long lo, hi;
    uint32_t len, bit;
};
__host__ __device__ constexpr Name name(const char *s, uint32_t bit) {
    Name r{0, 0, 0, bit};
    for (uint32_t k = 0; s[k]; k++, r.len++) {
        if (k < 8) r.lo |= (unsigned long long)(uint8_t)s[k] << (8 * k);
        else r.hi |= (unsigned long long)(uint8_t)s[k] << (8 * (k - 8));
    }
    return r;
}

// the bit of the piece whose first 16 bytes are lo / hi (little-endian) and whose length is len; 0 for any other piece
__device__ __forceinline__ uint32_t name_bit(unsigned long long lo, unsigned long long hi, uint32_t len) {
    constexpr Name N[7] = {name("flr", KXPU_RM_FLR),         name("af_flr", KXPU_RM_AF_FLR),
                           name("pm", KXPU_RM_PM),           name("bus", KXPU_RM_BUS),
                           name("cxl_bus", KXPU_RM_CXL_BUS), name("device_specific", KXPU_RM_DEVICE_SPECIFIC),
                           name("acpi", KXPU_RM_ACPI)};
    uint32_t b = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) b |= (len == N[k].len && lo == N[k].lo && hi == N[k].hi) ? N[k].bit : 0u;
    return b;
}

// reset_method's rule over the record's 64 text bytes (w, little-endian words), its length and flags
__device__ __forceinline__ uint32_t parse_methods(const uint32_t (&w)[16], uint32_t len, uint32_t flags) {
    if ((flags & KXPU_RS_READ_ERR) || len > KXPU_RESET_FILE_MAX) return 0;
    if (flags & KXPU_RS_ABSENT) return (flags & KXPU_RS_LEGACY) ? KXPU_RM_UNNAMED : 0u;
    uint32_t m = 0, tl = 0;
    unsigned long long lo = 0, hi = 0;
#pragma unroll
    for (uint32_t k = 0; k <= KXPU_RESET_FILE_MAX; k++) {  // constant indices: the text stays in registers
        const uint32_t c = k < KXPU_RESET_FILE_MAX ? (w[k >> 2] >> (8 * (k & 3))) & 0xffu : 0u;
        const bool end = k >= len || (k + 1 == len && c == '\n');
        if (end || c == ' ') {
            m |= name_bit(lo, hi, tl);
            lo = hi = 0;
            tl = 0;
            if (end) break;
        } else {
            if (tl < 8) lo |= (unsigned long long)c << (8 * tl);
            else if (tl < 16) hi |= (unsigned long long)c << (8 * (tl - 8));
            tl++;
        }
    }
    return m;
}

__device__ __forceinline__ uint32_t slot_of(unsigned long long key, uint32_t mask) {
    return (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 32) & mask;
}

// the slot holding key, or NONE
__device__ __forceinline__ uint32_t find(const Work &W, unsigned long long key) {
    for (uint32_t s = slot_of(key, W.mask);; s = (s + 1) & W.mask) {
        const unsigned long long v = __ldcg(W.keys + s);
        if (v == key) return s;
        if (v == EMPTY) return NONE;
    }
}

__global__ void __launch_bounds__(256) k_rs_parse(const Work W) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W.n) return;
    const uint4 *rp = reinterpret_cast<const uint4 *>(W.rrs + i);
    uint32_t w[16];
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const uint4 v = rp[q];
        w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
    }
    const uint4 t = rp[4];  // len, flags, reserved
    W.methods[i] = (uint8_t)parse_methods(w, t.x & 0xffu, (t.x >> 8) & 0xffu);
    const uint32_t l = W.clen[i];
    if (!l) return;
    const unsigned long long key = W.chain[(size_t)i * MAXD + l - 1];
    if (key & HOST_BRIDGE) return;
    for (uint32_t s = slot_of(key, W.mask);; s = (s + 1) & W.mask) {
        unsigned long long v = __ldcg(W.keys + s);
        if (v == EMPTY) {
            v = atomicCAS(W.keys + s, EMPTY, key);
            if (v == EMPTY) return;
        }
        if (v == key) return;
    }
}

__global__ void __launch_bounds__(256) k_rs_fold(const Work W, const __grid_constant__ Drivers D) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= W.n) return;
    const uint32_t l = W.clen[j];
    if (!l) return;
    const uint4 *rp = reinterpret_cast<const uint4 *>(W.recs + j);
    const uint4 q2 = rp[2], q3 = rp[3];  // driver; iommu_group, lengths, flags
    const unsigned long long drv0 = (unsigned long long)q2.y << 32 | q2.x, drv1 = (unsigned long long)q2.w << 32 | q2.z;
    bool match = false;
#pragma unroll
    for (uint32_t r = 0; r < KXPU_MAX_RULES; r++)  // constant indices: the table stays in the parameter bank
        match |= r < D.n && (drv0 & D.m0[r]) == D.d0[r] && (drv1 & D.m1[r]) == D.d1[r];
    const bool bound = match && !(((q3.y >> 16) & 0xffu) & (KXPU_REC_DRIVER_ERR | KXPU_REC_IOMMU_ERR | KXPU_REC_IS_DIR));
    const unsigned long long g = (unsigned long long)q3.x << 32;
    for (uint32_t t = 0; t < l; t++) {
        const unsigned long long key = W.chain[(size_t)j * MAXD + t];
        if (key & HOST_BRIDGE) continue;
        const uint32_t s = find(W, key);
        if (s == NONE) continue;
        if (!bound) {
            atomicMin(W.bad + s, j);
        } else {
            atomicMin(W.lo + s, g | j);
            atomicMax(W.hi + s, g | (NONE - j));
        }
    }
}

__global__ void __launch_bounds__(256) k_rs_verdict(const Work W) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W.n) return;
    const uint32_t l = W.clen[i];
    uint32_t v = KXPU_RESET_NO_PATH;
    if (l) {
        const unsigned long long key = W.chain[(size_t)i * MAXD + l - 1];
        const uint32_t s = (key & HOST_BRIDGE) ? NONE : find(W, key);  // i inserted its parent: s is found
        if (s == NONE) {
            v = KXPU_RESET_ROOT_BUS;
        } else if ((v = __ldcg(W.bad + s)) == NONE) {
            const unsigned long long lo = __ldcg(W.lo + s), hi = __ldcg(W.hi + s);
            if (lo >> 32 == hi >> 32) v = KXPU_RESET_SET_OK;
            else if (W.recs[i].iommu_group != (uint32_t)(lo >> 32)) v = (uint32_t)lo;
            else v = NONE - (uint32_t)hi;
        }
    }
    W.set_verdict[i] = v;
}

__global__ void __launch_bounds__(256) k_rs_group(const Work W) {
    const uint32_t m = W.m0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= W.m1) return;
    const uint32_t i = W.gmem[m];
    if (i >= W.n) {
        atomicOr(W.err, 1u);
        return;
    }
    const uint32_t meth = W.methods[i];
    const bool fn = (meth & W.allow) || ((meth & KXPU_RM_UNNAMED) && W.allow == KXPU_RM_ALL);
    if (fn || W.set_verdict[i] == KXPU_RESET_SET_OK) return;
    uint32_t lo = 0, hi = W.G;  // the last o with goff[o] <= m: the group holding position m
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (W.goff[mid] <= m) lo = mid;
        else hi = mid;
    }
    atomicMin(W.group_reset + lo, i);
}

}  // namespace kxreset

using namespace kxreset;

extern "C" int32_t kxpu_reset_check(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                                    const kxpu_pcipath *paths, const kxpu_resetrec *rrs, size_t n, uint32_t allow,
                                    const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                    uint8_t *methods, uint32_t *set_verdict, uint32_t *group_reset) {
    static_assert(sizeof(kxpu_resetrec) == 80 && offsetof(kxpu_resetrec, len) == 64 && offsetof(kxpu_resetrec, flags) == 65,
                  "kxpu_resetrec layout");
    if (!ctx || (n && (!recs || !paths || !rrs || !methods || !set_verdict)) || !group_off || (n_groups && !group_reset) ||
        !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES)
        return KXPU_E_INVALID;
    if (n >= (1ull << 28) || n_groups >= (1ull << 28)) return KXPU_E_UNSUPPORTED;  // kxpu_pcie_tree's parse limit
    Drivers D;
    memset(&D, 0, sizeof D);
    {
        unsigned long long drv[KXPU_MAX_RULES][4];
        const int32_t rc = kx_rule_drivers(ctx, rules, n_rules, drv);
        if (rc != KXPU_OK) return rc;
        for (size_t r = 0; r < n_rules; r++) {
            D.d0[r] = drv[r][0]; D.d1[r] = drv[r][1]; D.m0[r] = drv[r][2]; D.m1[r] = drv[r][3];
        }
        D.n = (uint32_t)n_rules;
    }
    if (allow & ~KXPU_RM_ALL) { KX_SET_ERR(ctx, "reset_check: allow 0x%x has bits outside KXPU_RM_ALL", allow); return KXPU_E_INVALID; }
    for (size_t g = 0; g < n_groups; g++)
        if (group_off[g + 1] < group_off[g]) { KX_SET_ERR(ctx, "reset_check: group %zu: offsets decrease", g); return KXPU_E_INVALID; }
    const size_t m0 = group_off[0], m1 = group_off[n_groups];
    if (m1 > m0 && !group_members) return KXPU_E_INVALID;
    if (n == 0 && n_groups == 0) return KXPU_OK;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    size_t cap = 1024;
    while (cap < 2 * n) cap <<= 1;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_recs = take(n * sizeof(kxpu_devrec)), o_paths = take(n * sizeof(kxpu_pcipath));
    const size_t o_rrs = take(n * sizeof(kxpu_resetrec)), o_goff = take((n_groups + 1) * 4), o_gmem = take(m1 * 4);
    const size_t o_chain = take(n * MAXD * 8), o_clen = take(n), o_keys = take(cap * 8), o_bad = take(cap * 4);
    const size_t o_lo = take(cap * 8), o_hi = take(cap * 8), o_meth = take(n), o_set = take(n * 4);
    const size_t o_gr = take(n_groups * 4), o_err = take(4);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_recs, recs, n * sizeof(kxpu_devrec)); up(o_paths, paths, n * sizeof(kxpu_pcipath));
    up(o_rrs, rrs, n * sizeof(kxpu_resetrec)); up(o_goff, group_off, (n_groups + 1) * 4);
    if (m1 > m0) up(o_gmem + m0 * 4, group_members + m0, (m1 - m0) * 4);
    cudaMemsetAsync(b + o_keys, 0xFF, cap * 8, st);
    cudaMemsetAsync(b + o_bad, 0xFF, cap * 4, st);
    cudaMemsetAsync(b + o_lo, 0xFF, cap * 8, st);
    cudaMemsetAsync(b + o_hi, 0, cap * 8, st);
    if (n_groups) cudaMemsetAsync(b + o_gr, 0xFF, n_groups * 4, st);
    cudaMemsetAsync(b + o_err, 0, 4, st);
    Work W;
    W.recs = (const kxpu_devrec *)(b + o_recs); W.rrs = (const kxpu_resetrec *)(b + o_rrs);
    W.n = (uint32_t)n; W.allow = allow;
    W.chain = (const unsigned long long *)(b + o_chain); W.clen = b + o_clen;
    W.keys = (unsigned long long *)(b + o_keys); W.bad = (uint32_t *)(b + o_bad);
    W.lo = (unsigned long long *)(b + o_lo); W.hi = (unsigned long long *)(b + o_hi); W.mask = (uint32_t)(cap - 1);
    W.methods = b + o_meth; W.set_verdict = (uint32_t *)(b + o_set);
    W.goff = (const uint32_t *)(b + o_goff); W.gmem = (const uint32_t *)(b + o_gmem);
    W.G = (uint32_t)n_groups; W.m0 = (uint32_t)m0; W.m1 = (uint32_t)m1;
    W.group_reset = (uint32_t *)(b + o_gr); W.err = (uint32_t *)(b + o_err);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        if (n) {
            const unsigned g = (unsigned)((n + 255) / 256);
            kx_pcie_parse(st, W.recs, (const kxpu_pcipath *)(b + o_paths), W.n, (unsigned long long *)(b + o_chain), b + o_clen);
            k_rs_parse<<<g, 256, 0, st>>>(W);
            k_rs_fold<<<g, 256, 0, st>>>(W, D);
            k_rs_verdict<<<g, 256, 0, st>>>(W);
            ctx->launches += 4;
        }
        if (m1 > m0) {
            k_rs_group<<<(unsigned)((m1 - m0 + 255) / 256), 256, 0, st>>>(W);
            ctx->launches++;
        }
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, W.err, 4, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "reset_check failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) { KX_SET_ERR(ctx, "reset_check: a group member index is >= n"); return KXPU_E_INVALID; }
    if (n) {
        cudaMemcpyAsync(methods, W.methods, n, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(set_verdict, W.set_verdict, n * 4, cudaMemcpyDeviceToHost, st);
    }
    if (n_groups) cudaMemcpyAsync(group_reset, W.group_reset, n_groups * 4, cudaMemcpyDeviceToHost, st);
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "reset_check D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}
