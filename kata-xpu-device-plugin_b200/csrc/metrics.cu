// metrics.cu -- K17 Prometheus metrics: kxpu_metrics_devices (include/kxpu.h states the document).
//
// The shape of the other emitters: a size pass, the single-pass exclusive scan (scan.cuh) over the 3n sample lengths in
// family-major order, so that every sample's offset is its family's base plus its prefix, and a write pass.  Both passes
// give each device one warp.  A device's bytes are dominated by its label strings, and a reason's detail is anything from
// empty to KXPU_METRICS_STRING_MAX bytes: the lanes take 32 consecutive bytes of a string per step, each decides the
// output of its own byte from the bytes around it (UTF-8 repair and escaping need at most three bytes of context either
// way), and a warp prefix sum of the widths places the bytes.  So a long detail costs 32 times fewer steps than in one
// thread, and there is one code path, with no split between short and long devices to keep equal.
#include "common.cuh"
#include "emit.cuh"
#include "scan.cuh"

namespace kxmet {

using kxemit::dec_len;
using kxemit::dec_write;

constexpr int WARPS = 8;  // devices per CTA
constexpr int THREADS = 32 * WARPS;
constexpr unsigned FULL = 0xffffffffu;

// the kinds' names: offsets and lengths into KXPU_METRICS_REASONS
struct Names {
    uint8_t off[KXPU_MR_COUNT];
    uint8_t len[KXPU_MR_COUNT];
};
constexpr Names names_of(const char *s) {
    Names t{};
    uint32_t k = 0, start = 0, i = 0;
    for (; s[i]; i++)
        if (s[i] == ',') { t.off[k] = (uint8_t)start; t.len[k] = (uint8_t)(i - start); k++; start = i + 1; }
    t.off[k] = (uint8_t)start;
    t.len[k] = (uint8_t)(i - start);
    return t;
}
constexpr uint32_t count_names(const char *s) {
    uint32_t k = 1;
    for (uint32_t i = 0; s[i]; i++) k += s[i] == ',';
    return k;
}
static_assert(count_names(KXPU_METRICS_REASONS) == KXPU_MR_COUNT, "one name per kind");
// The literals are copied lane by lane, each lane a different byte: in global memory (read through the read-only
// cache) a warp's 32 bytes are one request, where the constant cache would serve 32 different addresses one by one.
// c_nt is read at one address per warp, so it stays in constant memory.
__device__ const char c_names[] = KXPU_METRICS_REASONS;
__constant__ Names c_nt = names_of(KXPU_METRICS_REASONS);

#define KX_LIT(name, text)                    \
    __device__ const char name[] = text;      \
    constexpr uint32_t name##_LEN = sizeof(text) - 1;
KX_LIT(L_P1, "kata_xpu_device_healthy{resource=\"")
KX_LIT(L_P2, "kata_xpu_device_unhealthy_reason{resource=\"")
KX_LIT(L_P3, "kata_xpu_pcie_aer_errors{resource=\"")
KX_LIT(L_MD, "\",device=\"")
KX_LIT(L_MA, "\",address=\"")
KX_LIT(L_VAL, "\"} ")
KX_LIT(L_RK, "\",reason=\"")
KX_LIT(L_RD, "\",detail=\"")
KX_LIT(L_RE, "\"} 1\n")
KX_LIT(L_SEV, "\",severity=\"")
KX_LIT(L_FATAL, "fatal")
KX_LIT(L_NONFATAL, "nonfatal")
KX_LIT(L_H1, KXPU_METRICS_HEALTHY_HEAD)
KX_LIT(L_H2, KXPU_METRICS_REASON_HEAD)
KX_LIT(L_H3, KXPU_METRICS_AER_HEAD)
#undef KX_LIT

// ------------------------------------------------------------------ UTF-8 repair and label escaping, per byte
__device__ __forceinline__ bool is_cont(uint32_t c) { return (c & 0xC0u) == 0x80u; }
// continuation bytes a lead byte asks for; 0: not a lead (ASCII, a continuation byte, C0, C1, F5..FF)
__device__ __forceinline__ uint32_t lead_need(uint32_t c) {
    return c < 0xC2u ? 0u : c < 0xE0u ? 1u : c < 0xF0u ? 2u : c < 0xF5u ? 3u : 0u;
}
// the k-th byte (1-based) after `lead` continues its sequence: the second byte's range depends on the lead (no overlong
// form, no surrogate, nothing above U+10FFFF), every later byte is 80..BF
__device__ __forceinline__ bool cont_ok(uint32_t lead, uint32_t k, uint32_t c) {
    if (k == 1) {
        if (lead == 0xE0u) return c >= 0xA0u && c <= 0xBFu;
        if (lead == 0xEDu) return c >= 0x80u && c <= 0x9Fu;
        if (lead == 0xF0u) return c >= 0x90u && c <= 0xBFu;
        if (lead == 0xF4u) return c >= 0x80u && c <= 0x8Fu;
    }
    return is_cont(c);
}
// how many bytes after the lead at q continue its sequence, at most need
__device__ __forceinline__ uint32_t run_of(const uint8_t *s, uint32_t len, uint32_t q, uint32_t lead, uint32_t need) {
    uint32_t k = 0;
    while (k < need && q + 1u + k < len && cont_ok(lead, k + 1u, s[q + 1u + k])) k++;
    return k;
}
// The output width of byte p of s[0, len).  Decoding from the start, a step begins at a byte that is no continuation
// byte, or at a continuation byte the step in front of it did not take; a step takes its lead and the bytes that continue
// it (a maximal subpart when it stops short).  So a continuation byte belongs to the nearest non-continuation byte at
// most three bytes in front when that lead's run reaches it, and starts a step of its own otherwise.  A step's first byte
// carries the whole output: a complete sequence is copied, anything else is one U+FFFD; the bytes it took carry 0.
__device__ __forceinline__ uint32_t esc_width(const uint8_t *s, uint32_t len, uint32_t p) {
    const uint32_t c = s[p];
    if (c < 0x80u) return (c == '\\' || c == '"' || c == '\n') ? 2u : 1u;
    if (is_cont(c)) {
        for (uint32_t d = 1; d <= 3u && d <= p; d++) {
            const uint32_t q = s[p - d];
            if (is_cont(q)) continue;
            const uint32_t need = lead_need(q);
            return need >= d && run_of(s, len, p - d, q, need) >= d ? 0u : 3u;
        }
        return 3u;
    }
    const uint32_t need = lead_need(c);
    return need && run_of(s, len, p, c, need) == need ? need + 1u : 3u;
}
// writes byte p's output (width w, from esc_width) to d
__device__ __forceinline__ void esc_put(const uint8_t *s, uint32_t len, uint32_t p, uint32_t w, uint8_t *d) {
    if (w == 0u) return;
    const uint32_t c = s[p];
    if (c < 0x80u) {
        if (w == 2u) { d[0] = '\\'; d[1] = c == '\n' ? (uint8_t)'n' : (uint8_t)c; }
        else d[0] = (uint8_t)c;
        return;
    }
    const uint32_t need = lead_need(c);
    if (need && w == need + 1u && run_of(s, len, p, c, need) == need) {
        for (uint32_t k = 0; k <= need; k++) d[k] = s[p + k];
        return;
    }
    d[0] = 0xEFu; d[1] = 0xBFu; d[2] = 0xBDu;
}

// ------------------------------------------------------------------ warp helpers (all 32 lanes, uniform arguments)
__device__ __forceinline__ uint32_t warp_width(const uint8_t *s, uint32_t len) {
    uint32_t w = 0;
    for (uint32_t b = 0; b < len; b += 32u) {
        const uint32_t p = b + kx_lane();
        if (p < len) w += esc_width(s, len, p);
    }
    return __reduce_add_sync(FULL, w);
}
__device__ __forceinline__ uint8_t *warp_put(const uint8_t *s, uint32_t len, uint8_t *d) {
    for (uint32_t b = 0; b < len; b += 32u) {
        const uint32_t p = b + kx_lane();
        const uint32_t w = p < len ? esc_width(s, len, p) : 0u;
        const uint32_t incl = kxscan::warp_incl(w);
        esc_put(s, len, p, w, d + incl - w);
        d += __shfl_sync(FULL, incl, 31);
    }
    return d;
}
__device__ __forceinline__ uint8_t *warp_lit(const char *lit, uint32_t len, uint8_t *d) {
    for (uint32_t k = kx_lane(); k < len; k += 32u) d[k] = (uint8_t)__ldg(lit + k);
    return d + len;
}
__device__ __forceinline__ uint8_t *warp_dec(unsigned long long v, uint8_t *d) {
    const uint32_t l = dec_len(v);
    if (kx_lane() == 0) dec_write(v, l, d);
    return d + l;
}

__device__ __forceinline__ kxpu_metricdev load_dev(const kxpu_metricdev *p) {
    static_assert(sizeof(kxpu_metricdev) == 64, "four 16-byte loads");
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    union { uint4 v[4]; kxpu_metricdev d; } u;
#pragma unroll
    for (int k = 0; k < 4; k++) u.v[k] = __ldg(q + k);
    return u.d;
}

// the bytes every sample of a device shares: resource, device and address labels between the name and the family's tail
__device__ __forceinline__ uint32_t common_len(const kxpu_metricdev &dv, const uint8_t *str) {
    return warp_width(str + dv.resource_off, dv.resource_len) + L_MD_LEN + dec_len(dv.group) + L_MA_LEN +
           warp_width(str + dv.address_off, dv.address_len);
}
__device__ __forceinline__ uint8_t *put_common(const char *name, uint32_t name_len, const kxpu_metricdev &dv,
                                               const uint8_t *str, uint8_t *d) {
    d = warp_lit(name, name_len, d);
    d = warp_put(str + dv.resource_off, dv.resource_len, d);
    d = warp_lit(L_MD, L_MD_LEN, d);
    d = warp_dec(dv.group, d);
    d = warp_lit(L_MA, L_MA_LEN, d);
    return warp_put(str + dv.address_off, dv.address_len, d);
}
__device__ __forceinline__ uint32_t aer_len(uint32_t common, uint32_t sev_len, unsigned long long v) {
    return L_P3_LEN + common + L_SEV_LEN + sev_len + L_VAL_LEN + dec_len(v) + 1u;
}

// lens[f * n + i]: the bytes of device i's samples in family f; fam[f] += the family's total
__global__ void __launch_bounds__(THREADS) k_met_len(const kxpu_metricdev *__restrict__ devs, uint32_t n,
                                                     const uint8_t *__restrict__ str, const kxpu_metricreason *__restrict__ rs,
                                                     uint32_t *__restrict__ lens, unsigned long long *__restrict__ fam) {
    __shared__ unsigned long long s_fam[3];
    if (threadIdx.x < 3) s_fam[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t i = blockIdx.x * WARPS + (threadIdx.x >> 5);
    if (i < n) {
        const kxpu_metricdev dv = load_dev(devs + i);
        const uint32_t common = common_len(dv, str);
        const uint32_t l1 = L_P1_LEN + common + L_VAL_LEN + 2u;  // "0\n" or "1\n"
        uint32_t l2 = 0;
        for (uint32_t r = 0; r < dv.reason_count; r++) {
            const kxpu_metricreason e = rs[dv.reason_off + r];
            l2 += L_P2_LEN + common + L_RK_LEN + c_nt.len[e.kind] + L_RD_LEN + warp_width(str + e.detail_off, e.detail_len) +
                  L_RE_LEN;
        }
        uint32_t l3 = 0;
        if (dv.aer_fatal != KXPU_METRICS_NO_VALUE) l3 += aer_len(common, L_FATAL_LEN, dv.aer_fatal);
        if (dv.aer_nonfatal != KXPU_METRICS_NO_VALUE) l3 += aer_len(common, L_NONFATAL_LEN, dv.aer_nonfatal);
        if (kx_lane() == 0) {
            lens[i] = l1;
            lens[n + i] = l2;
            lens[2u * n + i] = l3;
            atomicAdd(&s_fam[0], (unsigned long long)l1);
            if (l2) atomicAdd(&s_fam[1], (unsigned long long)l2);
            if (l3) atomicAdd(&s_fam[2], (unsigned long long)l3);
        }
    }
    __syncthreads();
    if (threadIdx.x < 3 && s_fam[threadIdx.x]) atomicAdd(&fam[threadIdx.x], s_fam[threadIdx.x]);
}

struct WriteParams {
    const kxpu_metricdev *devs;
    const uint8_t *str;
    const kxpu_metricreason *rs;
    const unsigned long long *offs;  // the scan of lens: 3n exclusive prefixes
    uint8_t *out;
    uint32_t n;
    uint32_t head_on;                // bit f: family f has samples, and its header is written at head_at[f]
    unsigned long long shift[3];     // family f's samples sit at offs[f * n + i] + shift[f]: the headers in front of them
    unsigned long long head_at[3];
};

__global__ void __launch_bounds__(THREADS) k_met_write(const __grid_constant__ WriteParams P) {
    const uint32_t w = threadIdx.x >> 5;
    if (blockIdx.x == 0 && w < 3 && (P.head_on >> w & 1u)) {
        const char *h = w == 0 ? L_H1 : w == 1 ? L_H2 : L_H3;
        const uint32_t hl = w == 0 ? L_H1_LEN : w == 1 ? L_H2_LEN : L_H3_LEN;
        warp_lit(h, hl, P.out + P.head_at[w]);
    }
    const uint32_t i = blockIdx.x * WARPS + w;
    if (i >= P.n) return;
    const kxpu_metricdev dv = load_dev(P.devs + i);
    uint8_t *d = put_common(L_P1, L_P1_LEN, dv, P.str, P.out + P.offs[i] + P.shift[0]);
    d = warp_lit(L_VAL, L_VAL_LEN, d);
    if (kx_lane() == 0) { d[0] = dv.healthy ? '1' : '0'; d[1] = '\n'; }
    if (dv.reason_count) {
        d = P.out + P.offs[P.n + i] + P.shift[1];
        for (uint32_t r = 0; r < dv.reason_count; r++) {
            const kxpu_metricreason e = P.rs[dv.reason_off + r];
            d = put_common(L_P2, L_P2_LEN, dv, P.str, d);
            d = warp_lit(L_RK, L_RK_LEN, d);
            d = warp_lit(c_names + c_nt.off[e.kind], c_nt.len[e.kind], d);
            d = warp_lit(L_RD, L_RD_LEN, d);
            d = warp_put(P.str + e.detail_off, e.detail_len, d);
            d = warp_lit(L_RE, L_RE_LEN, d);
        }
    }
    const bool fatal = dv.aer_fatal != KXPU_METRICS_NO_VALUE, nonfatal = dv.aer_nonfatal != KXPU_METRICS_NO_VALUE;
    if (fatal || nonfatal) {
        d = P.out + P.offs[2u * P.n + i] + P.shift[2];
        for (int k = 0; k < 2; k++) {
            if (!(k ? nonfatal : fatal)) continue;
            d = put_common(L_P3, L_P3_LEN, dv, P.str, d);
            d = warp_lit(L_SEV, L_SEV_LEN, d);
            d = k ? warp_lit(L_NONFATAL, L_NONFATAL_LEN, d) : warp_lit(L_FATAL, L_FATAL_LEN, d);
            d = warp_lit(L_VAL, L_VAL_LEN, d);
            d = warp_dec(k ? dv.aer_nonfatal : dv.aer_fatal, d);
            if (kx_lane() == 0) *d = '\n';
            d += 1;
        }
    }
}

}  // namespace kxmet

using namespace kxmet;

// the host's argument checks of kxpu_metrics_devices (include/kxpu.h), in device order; KXPU_OK when all hold
static int32_t metrics_check(kxpu_ctx *ctx, const kxpu_metricdev *devs, size_t n, size_t strings_len,
                             const kxpu_metricreason *reasons, size_t n_reasons) {
    auto range = [&](const char *what, size_t i, uint64_t off, uint64_t len) {
        if (off > strings_len || len > strings_len - off) {
            KX_SET_ERR(ctx, "metrics_devices: device %zu: the %s range [%llu, +%llu) is not inside strings", i, what,
                       (unsigned long long)off, (unsigned long long)len);
            return KXPU_E_INVALID;
        }
        if (len > KXPU_METRICS_STRING_MAX) {
            KX_SET_ERR(ctx, "metrics_devices: device %zu: the %s is longer than %u bytes", i, what, KXPU_METRICS_STRING_MAX);
            return KXPU_E_UNSUPPORTED;
        }
        return KXPU_OK;
    };
    for (size_t i = 0; i < n; i++) {
        const kxpu_metricdev &d = devs[i];
        int32_t rc = range("resource", i, d.resource_off, d.resource_len);
        if (rc == KXPU_OK) rc = range("address", i, d.address_off, d.address_len);
        if (rc != KXPU_OK) return rc;
        if (d.healthy > 1u) {
            KX_SET_ERR(ctx, "metrics_devices: device %zu: healthy is %u, not 0 or 1", i, d.healthy);
            return KXPU_E_INVALID;
        }
        if (d.reason_off > n_reasons || d.reason_count > n_reasons - d.reason_off) {
            KX_SET_ERR(ctx, "metrics_devices: device %zu: its reasons are not inside the %zu entries", i, n_reasons);
            return KXPU_E_INVALID;
        }
        for (uint32_t r = 0; r < d.reason_count; r++) {
            const kxpu_metricreason &e = reasons[d.reason_off + r];
            if (e.kind >= KXPU_MR_COUNT || (r && e.kind <= reasons[d.reason_off + r - 1].kind)) {
                KX_SET_ERR(ctx, "metrics_devices: device %zu: reason %u has kind %u, not a kind above the one before", i, r,
                           e.kind);
                return KXPU_E_INVALID;
            }
            rc = range("detail", i, e.detail_off, e.detail_len);
            if (rc != KXPU_OK) return rc;
        }
    }
    return KXPU_OK;
}

extern "C" int32_t kxpu_metrics_devices(kxpu_ctx *ctx, const kxpu_metricdev *devs, size_t n, const uint8_t *strings,
                                        size_t strings_len, const kxpu_metricreason *reasons, size_t n_reasons, uint8_t *out,
                                        size_t cap, size_t *len) {
    if (!ctx || !len || (n && !devs) || (strings_len && !strings) || (n_reasons && !reasons)) return KXPU_E_INVALID;
    if (n >= (1ull << 28)) {
        KX_SET_ERR(ctx, "metrics_devices: n = %zu is not below 2^28", n);
        return KXPU_E_UNSUPPORTED;
    }
    int32_t rc = metrics_check(ctx, devs, n, strings_len, reasons, n_reasons);
    if (rc != KXPU_OK) return rc;
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    if (n == 0) { *len = 0; return KXPU_OK; }
    const uint32_t N = (uint32_t)n, blocks = (N + WARPS - 1) / WARPS;
    KxScratch sc(ctx);
    kxpu_metricdev *d_devs = nullptr;
    kxpu_metricreason *d_rs = nullptr;
    uint8_t *d_str = nullptr;
    uint32_t *d_lens = nullptr;
    unsigned long long *d_fam = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&d_devs, n * sizeof(kxpu_metricdev)));
    KX_CUDA(ctx, sc.alloc((void **)&d_rs, n_reasons * sizeof(kxpu_metricreason)));
    KX_CUDA(ctx, sc.alloc((void **)&d_str, strings_len));
    KX_CUDA(ctx, sc.alloc((void **)&d_lens, 3 * n * sizeof(uint32_t)));
    KX_CUDA(ctx, sc.alloc((void **)&d_fam, 3 * sizeof(unsigned long long)));
    cudaStream_t st = ctx->stream;
    KX_CUDA(ctx, cudaMemcpyAsync(d_devs, devs, n * sizeof(kxpu_metricdev), cudaMemcpyHostToDevice, st));
    if (n_reasons) KX_CUDA(ctx, cudaMemcpyAsync(d_rs, reasons, n_reasons * sizeof(kxpu_metricreason), cudaMemcpyHostToDevice, st));
    if (strings_len) KX_CUDA(ctx, cudaMemcpyAsync(d_str, strings, strings_len, cudaMemcpyHostToDevice, st));
    KX_CUDA(ctx, cudaMemsetAsync(d_fam, 0, 3 * sizeof(unsigned long long), st));
    KxTimer timer(ctx, KXPU_T_EMIT);
    k_met_len<<<blocks, THREADS, 0, st>>>(d_devs, N, d_str, d_rs, d_lens, d_fam);
    KX_LAUNCHED(ctx);
    unsigned long long fam[3] = {0, 0, 0};
    KX_CUDA(ctx, cudaMemcpyAsync(fam, d_fam, sizeof fam, cudaMemcpyDeviceToHost, st));
    KX_CUDA(ctx, cudaStreamSynchronize(st));
    const unsigned long long head_len[3] = {L_H1_LEN, L_H2_LEN, L_H3_LEN};
    WriteParams P{};
    unsigned long long total = 0, heads = 0;  // the document: each present family's header, then its samples
    for (int f = 0; f < 3; f++) {
        if (fam[f]) {
            P.head_on |= 1u << f;
            P.head_at[f] = total;
            heads += head_len[f];
            total += head_len[f];
        }
        P.shift[f] = heads;
        total += fam[f];
    }
    if (total >= (1ull << 40)) {
        KX_SET_ERR(ctx, "metrics_devices: the document would be %llu bytes, not below 2^40", total);
        return KXPU_E_UNSUPPORTED;
    }
    *len = (size_t)total;
    if (!out || cap < total) return total ? KXPU_E_NOSPACE : KXPU_OK;
    if (total > kxscan::ST_VAL) {
        KX_SET_ERR(ctx, "metrics_devices: a document of %llu bytes cannot be staged in device memory", total);
        return KXPU_E_NOMEM;
    }
    unsigned long long *d_offs = nullptr;
    uint8_t *d_out = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&d_offs, 3 * n * sizeof(unsigned long long)));
    KX_CUDA(ctx, sc.alloc((void **)&d_out, total));
    rc = kxscan::exclusive_scan<unsigned long long>(ctx, d_lens, 3 * n, d_offs, nullptr);
    if (rc != KXPU_OK) return rc;
    P.devs = d_devs;
    P.str = d_str;
    P.rs = d_rs;
    P.offs = d_offs;
    P.out = d_out;
    P.n = N;
    k_met_write<<<blocks, THREADS, 0, st>>>(P);
    KX_LAUNCHED(ctx);
    timer.stop();
    KX_CUDA(ctx, cudaMemcpyAsync(out, d_out, total, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        KX_SET_ERR(ctx, "metrics_devices failed: %s", cudaGetErrorString(e));
        return KXPU_E_CUDA;
    }
    return KXPU_OK;
}
