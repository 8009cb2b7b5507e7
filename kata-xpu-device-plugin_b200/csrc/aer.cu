// aer.cu -- K12: PCIe AER health (kxpu_aer_health).  include/kxpu.h states the file format and the fold.
//
// Two kernels:
//   - k_aer_files: one warp per file.  The count is the LAST line that begins with the prefix, so the warp walks the
//     file backward in 32-byte windows.  Lane l of a window looks at byte q = hi - 32 + l: q starts a line when it is
//     the file's first byte or follows a '\n'.  A starting lane compares the prefix and parses the number after it on
//     its own (at most 20 + 20 bytes); a ballot of the matches picks the highest one, and the first window with a match
//     ends the walk.  A sysfs AER file ends with its TOTAL line, so the walk usually reads one or two windows.
//   - k_aer_groups: one warp per group ORs its members' bits (members strided over the lanes, a warp OR at the end).
#include "common.cuh"

namespace kxaer {

constexpr int THREADS = 256, WARPS = THREADS / 32;
constexpr unsigned long long UNKNOWN = ~0ull;
constexpr uint32_t ERR_RANGE = 1u, ERR_MEMBER = 2u;

__constant__ char PFX_FATAL[] = "TOTAL_ERR_FATAL ";
__constant__ char PFX_NONFATAL[] = "TOTAL_ERR_NONFATAL ";

// the line at t[q ..) (q a line start, len the file's length): *match when it begins with pfx; its count, or UNKNOWN
__device__ __forceinline__ unsigned long long parse_line(const uint8_t *t, uint32_t q, uint32_t len, const char *pfx,
                                                        uint32_t pl, bool *match) {
    *match = false;
    if (len - q < pl) return UNKNOWN;
    for (uint32_t k = 0; k < pl; k++)
        if (t[q + k] != (uint8_t)pfx[k]) return UNKNOWN;
    *match = true;
    unsigned long long v = 0;
    uint32_t nd = 0, p = q + pl;
    for (; p < len && t[p] != '\n'; p++, nd++) {
        const uint32_t d = (uint32_t)t[p] - '0';
        if (d > 9u || nd == 20u) return UNKNOWN;                    // not a digit ('\r' included), or a 21st digit
        if (v > (UNKNOWN - d) / 10ull) return UNKNOWN;              // above 2^64 - 1
        v = v * 10ull + d;
    }
    if (nd == 0u || (nd > 1u && t[q + pl] == '0') || v == UNKNOWN) return UNKNOWN;  // empty, a leading zero, 2^64 - 1
    return v;
}

__global__ void __launch_bounds__(THREADS) k_aer_files(const uint8_t *__restrict__ text, unsigned long long text_len,
                                                       const unsigned long long *__restrict__ file_off,
                                                       const uint32_t *__restrict__ file_len, uint32_t n_files,
                                                       unsigned long long *__restrict__ totals, uint32_t *__restrict__ err) {
    const uint32_t f = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    if (f >= n_files) return;
    const unsigned long long off = file_off[f];
    const uint32_t len = file_len[f];
    if (off > text_len || len > text_len - off) {
        if (lane == 0) atomicOr(err, ERR_RANGE);
        return;
    }
    unsigned long long result = UNKNOWN;
    if (len != 0u && len <= (uint32_t)KXPU_AER_FILE_MAX) {
        const uint8_t *t = text + off;
        const bool fatal = (f & 1u) == 0u;
        const char *pfx = fatal ? PFX_FATAL : PFX_NONFATAL;
        const uint32_t pl = fatal ? 16u : 19u;
        for (int hi = (int)len; hi > 0; hi -= 32) {
            const int q = hi - 32 + (int)lane;
            bool match = false;
            unsigned long long v = UNKNOWN;
            if (q >= 0 && (q == 0 || t[q - 1] == '\n')) v = parse_line(t, (uint32_t)q, len, pfx, pl, &match);
            const uint32_t hits = __ballot_sync(0xffffffffu, match);
            if (hits) {
                result = __shfl_sync(0xffffffffu, v, 31 - __clz(hits));
                break;
            }
        }
    }
    if (lane == 0) totals[f] = result;
}

__global__ void __launch_bounds__(THREADS) k_aer_groups(const unsigned long long *__restrict__ totals, uint32_t n,
                                                        const uint32_t *__restrict__ goff, const uint32_t *__restrict__ gmem,
                                                        uint32_t n_groups, unsigned long long fatal_limit,
                                                        unsigned long long nonfatal_limit, uint8_t *__restrict__ group_aer,
                                                        uint32_t *__restrict__ err) {
    const uint32_t o = blockIdx.x * WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    if (o >= n_groups) return;
    uint32_t bits = 0;
    bool bad = false;
    for (uint32_t m = goff[o] + lane; m < goff[o + 1]; m += 32u) {
        const uint32_t i = gmem[m];
        if (i >= n) { bad = true; continue; }
        const unsigned long long tf = totals[2ull * i], tn = totals[2ull * i + 1];
        if (tf == UNKNOWN || tn == UNKNOWN) bits |= KXPU_AER_UNKNOWN;
        if (tf != UNKNOWN && tf > fatal_limit) bits |= KXPU_AER_FATAL;
        if (tn != UNKNOWN && tn > nonfatal_limit) bits |= KXPU_AER_NONFATAL;
    }
    bits = __reduce_or_sync(0xffffffffu, bits);
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) {
        group_aer[o] = (uint8_t)bits;
        if (bad) atomicOr(err, ERR_MEMBER);
    }
}

}  // namespace kxaer

using namespace kxaer;

extern "C" int32_t kxpu_aer_health(kxpu_ctx *ctx, const uint8_t *text, size_t text_len, const uint64_t *file_off,
                                   const uint32_t *file_len, size_t n, uint64_t fatal_limit, uint64_t nonfatal_limit,
                                   const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                   uint64_t *totals, uint8_t *group_aer) {
    if (!ctx || (text_len && !text) || (n && (!file_off || !file_len)) || !group_off || (n_groups && !group_aer))
        return KXPU_E_INVALID;
    if (n >= (1ull << 28) || n_groups >= (1ull << 28)) return KXPU_E_UNSUPPORTED;
    for (size_t g = 0; g < n_groups; g++)
        if (group_off[g + 1] < group_off[g]) { KX_SET_ERR(ctx, "aer_health: group %zu: offsets decrease", g); return KXPU_E_INVALID; }
    const size_t nm = group_off[n_groups];
    if (nm && !group_members) return KXPU_E_INVALID;
    if (n == 0 && n_groups == 0) return KXPU_OK;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    const size_t NF = 2 * n, G = n_groups;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_text = take(text_len), o_foff = take(NF * 8), o_flen = take(NF * 4), o_tot = take(NF * 8);
    const size_t o_goff = take((G + 1) * 4), o_gmem = take(nm * 4), o_gaer = take(G), o_err = take(16);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_text, text, text_len); up(o_foff, file_off, NF * 8); up(o_flen, file_len, NF * 4);
    up(o_goff, group_off, (G + 1) * 4); up(o_gmem, group_members, nm * 4);
    cudaMemsetAsync(b + o_err, 0, 16, st);
    uint32_t *d_err = (uint32_t *)(b + o_err);
    unsigned long long *d_tot = (unsigned long long *)(b + o_tot);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        if (NF) {
            k_aer_files<<<(unsigned)((NF + WARPS - 1) / WARPS), THREADS, 0, st>>>(
                b + o_text, (unsigned long long)text_len, (const unsigned long long *)(b + o_foff),
                (const uint32_t *)(b + o_flen), (uint32_t)NF, d_tot, d_err);
            KX_LAUNCHED(ctx);
        }
        if (G) {
            k_aer_groups<<<(unsigned)((G + WARPS - 1) / WARPS), THREADS, 0, st>>>(
                d_tot, (uint32_t)n, (const uint32_t *)(b + o_goff), (const uint32_t *)(b + o_gmem), (uint32_t)G,
                (unsigned long long)fatal_limit, (unsigned long long)nonfatal_limit, b + o_gaer, d_err);
            KX_LAUNCHED(ctx);
        }
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, d_err, 4, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "aer_health failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) {
        KX_SET_ERR(ctx, "aer_health:%s%s", (h[0] & ERR_RANGE) ? " a file range lies outside text_len;" : "",
                   (h[0] & ERR_MEMBER) ? " a group member index is >= n;" : "");
        return KXPU_E_INVALID;
    }
    if (totals && NF) cudaMemcpyAsync(totals, d_tot, NF * 8, cudaMemcpyDeviceToHost, st);
    if (G) cudaMemcpyAsync(group_aer, b + o_gaer, G, cudaMemcpyDeviceToHost, st);
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "aer_health D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}
