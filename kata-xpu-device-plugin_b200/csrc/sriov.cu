// sriov.cu -- K14: the SR-IOV verdict of a walk (kxpu_sriov).  include/kxpu.h states the rules.
//
// Three launches, one table:
//   - k_sr_insert: one thread per record.  Two 16-byte vector loads of its kxpu_sriovrec and one of its bdf; it parses
//     sriov_numvfs into numvfs[i], stores the packed key of its physfn (or NONE) in pf_of[i] for the probe, and inserts
//     its own bdf key, when canonical, into an open-addressing table of u64 slots key << 32 | index.  A slot is claimed by
//     CAS; a slot holding the same key takes an atomic min of the whole word, which leaves the lowest index because the
//     high halves are equal.  The table has at least two slots per record, so a probe sequence always ends.
//   - k_sr_probe: one thread per record looks its physfn key up (pf_of[i] = the lowest index, NO_PF for none or itself)
//     and decides whether the record blocks its group: a VF whose PF is bound to a rule's driver, or numvfs > 0.
//   - k_sr_fold: one thread per group member finds its group ordinal by binary search over group_off and lowers
//     group_sriov[o] (all ones from a memset) to its index with an atomic min when it blocks; a member index >= n sets
//     the error word instead.
// kxpu_mdev_pf runs the same table with k_sr_insert<true> (one thread per PCI record, its bdf only) and k_sr_probe<true>
// (one thread per mdev, the physfn of its side record; no verdict); the <false> instantiations are kxpu_sriov's kernels.
#include "common.cuh"

namespace kxsriov {

constexpr unsigned long long EMPTY = ~0ull;
constexpr uint32_t NONE = ~0u;
constexpr uint32_t NO_PF = KXPU_NO_PF;

// the rule drivers as kx_rule_drivers returns them
struct Drivers {
    unsigned long long d0[KXPU_MAX_RULES], d1[KXPU_MAX_RULES], m0[KXPU_MAX_RULES], m1[KXPU_MAX_RULES];
    uint32_t n;
};

struct Work {
    const kxpu_devrec *recs;
    const kxpu_sriovrec *srs;
    uint32_t n;
    unsigned long long *slots;
    uint32_t mask;
    uint32_t *pf_of, *numvfs;
    uint8_t *blocks;             // [n] 1: the record blocks its group
    const uint32_t *goff, *gmem;
    uint32_t G, m0, m1;          // members [m0, m1) = [goff[0], goff[G])
    uint32_t *group_sriov;
    uint32_t *err;               // [0] = 1: a member index >= n
};

// kxpu_mdev_pf's probe side: the mdevs whose side records Work::srs are (pf_of has nm entries).  A parameter of its own,
// after Work and Drivers, so kxpu_sriov's kernels keep their parameter layout
struct MdevSide {
    const kxpu_mdevrec *mrecs;
    uint32_t nm;
};

__device__ __forceinline__ int hexv(uint32_t c) {
    return (c >= '0' && c <= '9') ? (int)(c - '0') : (c >= 'a' && c <= 'f') ? (int)(c - 'a' + 10) : -1;
}

// a 16-byte NUL-padded field holding a canonical lowercase "dddd:bb:dd.f" up to its first NUL -> domain << 16 | bus << 8 |
// dev << 3 | fn, else NONE (the key never reaches NONE: it has 29 bits)
__device__ __forceinline__ uint32_t bdf_key(const uint4 &q) {
    const uint8_t *t = reinterpret_cast<const uint8_t *>(&q);
    if (t[12] != 0 || t[4] != ':' || t[7] != ':' || t[10] != '.') return NONE;
    int h[8];
    const int at[8] = {0, 1, 2, 3, 5, 6, 8, 9};  // domain, bus, device digits
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 8; k++) {
        h[k] = hexv(t[at[k]]);
        ok &= h[k] >= 0;
    }
    const uint32_t fn = (uint32_t)t[11] - '0';
    const int dev = h[6] << 4 | h[7];
    if (!ok || fn > 7u || dev > 0x1f) return NONE;
    return (uint32_t)(h[0] << 12 | h[1] << 8 | h[2] << 4 | h[3]) << 16 | (uint32_t)(h[4] << 4 | h[5]) << 8 | (uint32_t)dev << 3 | fn;
}

// sriov_numvfs (the 8 bytes little-endian in txt): at most one trailing '\n', then a canonical decimal 0..65535; anything
// else 0.  Bytes are shifted out of the word, so the record stays in registers.
__device__ __forceinline__ uint32_t parse_numvfs(unsigned long long txt, uint32_t len, uint32_t flags) {
    if ((flags & KXPU_SR_NUMVFS_ERR) || len > 8u) return 0;
    if (len && ((txt >> (8 * (len - 1))) & 0xffu) == '\n') len--;
    if (len == 0 || len > 5u || (len > 1 && (txt & 0xffu) == '0')) return 0;
    uint32_t v = 0;
    for (uint32_t k = 0; k < len; k++) {
        const uint32_t d = (uint32_t)((txt >> (8 * k)) & 0xffu) - '0';
        if (d > 9u) return 0;
        v = v * 10u + d;
    }
    return v <= 65535u ? v : 0;
}

__device__ __forceinline__ uint32_t slot_of(uint32_t key, uint32_t mask) { return kx_hash(key) & mask; }

// the key of physfn (s0: its 16 bytes; flags: the side record's) for a probe, NONE when it cannot match
__device__ __forceinline__ uint32_t physfn_key(const uint4 &s0, uint32_t flags) {
    return (flags & KXPU_SR_PHYSFN_ERR) ? NONE : bdf_key(s0);
}

// MP (kxpu_mdev_pf): the PCI records' bdfs only; their side records are the mdevs', read by the probe
template <bool MP>
__global__ void __launch_bounds__(256) k_sr_insert(const Work W) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W.n) return;
    uint4 s0, s1;  // physfn[16]; numvfs_txt[8], numvfs_len, flags, reserved
    if constexpr (!MP) {
        const uint4 *sp = reinterpret_cast<const uint4 *>(W.srs + i);
        s0 = sp[0];
        s1 = sp[1];
    }
    const uint4 b0 = reinterpret_cast<const uint4 *>(W.recs + i)[0];  // bdf[16]
    if constexpr (!MP) {
        const uint32_t len = s1.z & 0xffu, flags = (s1.z >> 8) & 0xffu;
        W.numvfs[i] = parse_numvfs((unsigned long long)s1.y << 32 | s1.x, len, flags);
        W.pf_of[i] = physfn_key(s0, flags);
    }
    const uint32_t key = bdf_key(b0);
    if (key == NONE) return;
    const unsigned long long mine = (unsigned long long)key << 32 | i;
    for (uint32_t s = slot_of(key, W.mask);; s = (s + 1) & W.mask) {
        unsigned long long v = __ldcg(W.slots + s);
        if (v == EMPTY) {
            v = atomicCAS(W.slots + s, EMPTY, mine);
            if (v == EMPTY) return;
        }
        if ((uint32_t)(v >> 32) == key) {
            if (mine < v) atomicMin(W.slots + s, mine);
            return;
        }
    }
}

// MP (kxpu_mdev_pf): thread i is mdev i; its key comes from its side record, a physfn equal to its parent never matches,
// and there is no verdict
template <bool MP>
__global__ void __launch_bounds__(256) k_sr_probe(const Work W, const __grid_constant__ Drivers D, const MdevSide M) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t key;
    if constexpr (MP) {
        if (i >= M.nm) return;
        const uint4 *sp = reinterpret_cast<const uint4 *>(W.srs + i);
        key = physfn_key(sp[0], (sp[1].z >> 8) & 0xffu);
        // parent: bytes 36..51 of the mdev record, 4-byte aligned
        const uint32_t *pw = reinterpret_cast<const uint32_t *>(reinterpret_cast<const uint8_t *>(M.mrecs + i) + 36);
        const uint4 par = make_uint4(pw[0], pw[1], pw[2], pw[3]);
        if (key != NONE && bdf_key(par) == key) key = NONE;
    } else {
        if (i >= W.n) return;
        key = W.pf_of[i];
    }
    uint32_t p = NO_PF;
    if (key != NONE) {
        for (uint32_t s = slot_of(key, W.mask);; s = (s + 1) & W.mask) {
            const unsigned long long v = __ldcg(W.slots + s);
            if (v == EMPTY) break;
            if ((uint32_t)(v >> 32) == key) {
                p = (uint32_t)v;
                break;
            }
        }
        if (!MP && p == i) p = NO_PF;
    }
    W.pf_of[i] = p;
    if constexpr (MP) return;
    bool blocks = W.numvfs[i] > 0;
    if (p != NO_PF) {  // the PF's driver (bytes 32..47) and flags (byte 54)
        const uint4 *rp = reinterpret_cast<const uint4 *>(W.recs + p);
        const uint4 q2 = rp[2], q3 = rp[3];
        const unsigned long long drv0 = (unsigned long long)q2.y << 32 | q2.x, drv1 = (unsigned long long)q2.w << 32 | q2.z;
        bool match = false;
#pragma unroll
        for (uint32_t r = 0; r < KXPU_MAX_RULES; r++)  // constant indices: the table stays in the parameter bank
            match |= r < D.n && (drv0 & D.m0[r]) == D.d0[r] && (drv1 & D.m1[r]) == D.d1[r];
        blocks |= match && !(((q3.y >> 16) & 0xffu) & KXPU_REC_DRIVER_ERR);
    }
    W.blocks[i] = blocks;
}

__global__ void __launch_bounds__(256) k_sr_fold(const Work W) {
    const uint32_t m = W.m0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= W.m1) return;
    const uint32_t i = W.gmem[m];
    if (i >= W.n) {
        atomicOr(W.err, 1u);
        return;
    }
    if (!W.blocks[i]) return;
    uint32_t lo = 0, hi = W.G;  // the last o with goff[o] <= m: the group holding position m
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (W.goff[mid] <= m) lo = mid;
        else hi = mid;
    }
    atomicMin(W.group_sriov + lo, i);
}

}  // namespace kxsriov

using namespace kxsriov;

extern "C" int32_t kxpu_sriov(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                              const kxpu_sriovrec *srs, size_t n, const uint32_t *group_ids, const uint32_t *group_off,
                              const uint32_t *group_members, size_t n_groups, uint32_t *pf_of, uint32_t *numvfs,
                              uint32_t *group_sriov) {
    static_assert(sizeof(kxpu_sriovrec) == 32 && offsetof(kxpu_sriovrec, numvfs_len) == 24, "kxpu_sriovrec layout");
    (void)group_ids;  // the group ordinals are positions in the CSR
    if (!ctx || (n && (!recs || !srs || !pf_of || !numvfs)) || !group_off || (n_groups && !group_sriov) || !rules ||
        n_rules == 0 || n_rules > KXPU_MAX_RULES)
        return KXPU_E_INVALID;
    if (n >= (1ull << 30) || n_groups >= (1ull << 30)) return KXPU_E_UNSUPPORTED;  // the table's 2n slots fit 2^31
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
    for (size_t g = 0; g < n_groups; g++)
        if (group_off[g + 1] < group_off[g]) { KX_SET_ERR(ctx, "sriov: group %zu: offsets decrease", g); return KXPU_E_INVALID; }
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
    const size_t o_recs = take(n * sizeof(kxpu_devrec)), o_srs = take(n * sizeof(kxpu_sriovrec));
    const size_t o_goff = take((n_groups + 1) * 4), o_gmem = take(m1 * 4), o_slots = take((size_t)cap * 8);
    const size_t o_pf = take(n * 4), o_nv = take(n * 4), o_blk = take(n), o_gs = take(n_groups * 4), o_err = take(4);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_recs, recs, n * sizeof(kxpu_devrec)); up(o_srs, srs, n * sizeof(kxpu_sriovrec));
    up(o_goff, group_off, (n_groups + 1) * 4);
    if (m1 > m0) up(o_gmem + m0 * 4, group_members + m0, (m1 - m0) * 4);
    cudaMemsetAsync(b + o_slots, 0xFF, (size_t)cap * 8, st);
    if (n_groups) cudaMemsetAsync(b + o_gs, 0xFF, n_groups * 4, st);
    cudaMemsetAsync(b + o_err, 0, 4, st);
    Work W;
    W.recs = (const kxpu_devrec *)(b + o_recs); W.srs = (const kxpu_sriovrec *)(b + o_srs); W.n = (uint32_t)n;
    W.slots = (unsigned long long *)(b + o_slots); W.mask = (uint32_t)(cap - 1);
    W.pf_of = (uint32_t *)(b + o_pf); W.numvfs = (uint32_t *)(b + o_nv); W.blocks = b + o_blk;
    W.goff = (const uint32_t *)(b + o_goff); W.gmem = (const uint32_t *)(b + o_gmem);
    W.G = (uint32_t)n_groups; W.m0 = (uint32_t)m0; W.m1 = (uint32_t)m1;
    W.group_sriov = (uint32_t *)(b + o_gs); W.err = (uint32_t *)(b + o_err);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        if (n) {
            const unsigned g = (unsigned)((n + 255) / 256);
            k_sr_insert<false><<<g, 256, 0, st>>>(W);
            k_sr_probe<false><<<g, 256, 0, st>>>(W, D, MdevSide{nullptr, 0});
            ctx->launches += 2;
        }
        if (m1 > m0) {
            k_sr_fold<<<(unsigned)((m1 - m0 + 255) / 256), 256, 0, st>>>(W);
            ctx->launches++;
        }
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, W.err, 4, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "sriov failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) { KX_SET_ERR(ctx, "sriov: a group member index is >= n"); return KXPU_E_INVALID; }
    if (n) {
        cudaMemcpyAsync(pf_of, W.pf_of, n * 4, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(numvfs, W.numvfs, n * 4, cudaMemcpyDeviceToHost, st);
    }
    if (n_groups) cudaMemcpyAsync(group_sriov, W.group_sriov, n_groups * 4, cudaMemcpyDeviceToHost, st);
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "sriov D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}

extern "C" int32_t kxpu_mdev_pf(kxpu_ctx *ctx, const kxpu_devrec *recs, size_t n_recs, const kxpu_mdevrec *mrecs,
                                const kxpu_sriovrec *msrs, size_t n_mdevs, uint32_t *pf_of) {
    static_assert(offsetof(kxpu_mdevrec, parent) == 36 && sizeof(kxpu_mdevrec) % 16 == 0, "kxpu_mdevrec layout");
    if (!ctx || (n_recs && !recs) || (n_mdevs && (!mrecs || !msrs || !pf_of))) return KXPU_E_INVALID;
    if (n_recs >= (1ull << 30) || n_mdevs >= (1ull << 30)) return KXPU_E_UNSUPPORTED;  // as kxpu_sriov's table
    if (n_mdevs == 0) return KXPU_OK;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    size_t cap = 1024;
    while (cap < 2 * n_recs) cap <<= 1;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_recs = take(n_recs * sizeof(kxpu_devrec)), o_mrecs = take(n_mdevs * sizeof(kxpu_mdevrec));
    const size_t o_srs = take(n_mdevs * sizeof(kxpu_sriovrec)), o_slots = take((size_t)cap * 8), o_pf = take(n_mdevs * 4);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_recs, recs, n_recs * sizeof(kxpu_devrec));
    up(o_mrecs, mrecs, n_mdevs * sizeof(kxpu_mdevrec));
    up(o_srs, msrs, n_mdevs * sizeof(kxpu_sriovrec));
    cudaMemsetAsync(b + o_slots, 0xFF, (size_t)cap * 8, st);
    Work W;
    memset(&W, 0, sizeof W);
    W.recs = (const kxpu_devrec *)(b + o_recs); W.srs = (const kxpu_sriovrec *)(b + o_srs); W.n = (uint32_t)n_recs;
    W.slots = (unsigned long long *)(b + o_slots); W.mask = (uint32_t)(cap - 1);
    W.pf_of = (uint32_t *)(b + o_pf);
    const MdevSide M{(const kxpu_mdevrec *)(b + o_mrecs), (uint32_t)n_mdevs};
    Drivers D;
    memset(&D, 0, sizeof D);  // not read: the mdev probe gives no verdict
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        if (n_recs) {
            k_sr_insert<true><<<(unsigned)((n_recs + 255) / 256), 256, 0, st>>>(W);
            ctx->launches++;
        }
        k_sr_probe<true><<<(unsigned)((n_mdevs + 255) / 256), 256, 0, st>>>(W, D, M);
        ctx->launches++;
    }
    cudaMemcpyAsync(pf_of, W.pf_of, n_mdevs * 4, cudaMemcpyDeviceToHost, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "mdev_pf failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}
