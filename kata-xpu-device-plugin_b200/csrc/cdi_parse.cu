// cdi_parse.cu -- K13: kxpu_cdi_parse[_mdev|_cdev|_mdev_cdev|_vf_vgpu[_cdev]], the inverse of the CDI spec emitter (emit.cu, K6).
//
// A call accepts a document exactly when the emitter, given the records it decodes, writes the same bytes.  It runs in
// two steps:
//   - decode: one kernel over the document in byte tiles.  A device starts right after a '\n' that is followed by the
//     format's literal 0 ("  - name: \"" / "    {\n      \"name\": \""); nothing else in either document matches it.  A
//     CTA stages its tile (and a halo that holds the longest fragment) in shared memory, finds the starts with one ballot
//     per warp and row of 256 positions, scans the 256 row-warp counts, gets the tile's first record slot from the
//     decoupled look-back (scan.cuh) and decodes each of its devices from shared memory into its slot.  The decode is
//     lenient: every field is read at the offset a well-formed fragment puts it, digits wrap instead of overflowing, and
//     every read stops at the staged window, so a damaged document only decodes to records that fail the next step.
//   - verify: the decoded records go through the emitter's own kernel into device scratch, and a vectorised compare
//     holds that output against the uploaded document (lengths first).  The grammar lives in the emitter alone.
#include <string>

#include "cdi.cuh"
#include "common.cuh"
#include "scan.cuh"

namespace kxparse {

constexpr int PT = 8192;         // document bytes per CTA
constexpr int PARSE_THREADS = 256;
constexpr int ROWS = PT / PARSE_THREADS;  // positions per thread, one row of 256 consecutive positions each
constexpr int LEAD = 16;         // bytes staged in front of the tile: the '\n' before a start at the tile's first byte
constexpr int PAT_MAX = 32;
constexpr int LAYOUT_PCI = KX_CDI_PCI, LAYOUT_MDEV = KX_CDI_MDEV, LAYOUT_CDEV = KX_CDI_CDEV,
              LAYOUT_MDEV_CDEV = KX_CDI_MDEV_CDEV, LAYOUT_TYPED = KX_CDI_TYPED, LAYOUT_TYPED_CDEV = KX_CDI_TYPED_CDEV;
template <int LAYOUT> constexpr bool is_typed_layout = LAYOUT == LAYOUT_TYPED || LAYOUT == LAYOUT_TYPED_CDEV;
// bytes staged past the tile: >= the layout's longest fragment plus the start pattern, in whole 16-byte words
template <int LAYOUT> constexpr int HALO = is_typed_layout<LAYOUT> ? 576 : LAYOUT == LAYOUT_MDEV_CDEV ? 528 : 512;
constexpr int HALO_MAX = HALO<LAYOUT_TYPED>;  // the host pads every document for the largest halo
static_assert(HALO<LAYOUT_PCI> >= KX_CDI_FRAG_MAX + PAT_MAX, "a fragment that starts in the tile must end inside the window");
static_assert(HALO<LAYOUT_MDEV_CDEV> >= KX_CDI_FRAG_MAX_MDEV_CDEV + PAT_MAX && HALO<LAYOUT_MDEV_CDEV> % 16 == 0,
              "a fragment that starts in the tile must end inside the window");
static_assert(HALO<LAYOUT_TYPED> >= KX_CDI_FRAG_MAX_TYPED + PAT_MAX && HALO<LAYOUT_TYPED> % 16 == 0,
              "a fragment that starts in the tile must end inside the window");
static_assert(HALO_MAX >= HALO<LAYOUT_PCI> && HALO_MAX >= HALO<LAYOUT_MDEV_CDEV>, "the host padding must cover every layout's window");
template <int LAYOUT> constexpr int WIN = LEAD + PT + HALO<LAYOUT>;

struct ParseParams {
    const uint8_t *doc;           // padded with zeros to a whole tile plus HALO_MAX + LEAD bytes
    unsigned long long len;
    void *recs;                   // kxpu_cdidev[cap], kxpu_mdevcdi[cap] or kxpu_mdevcdev[cap]
    unsigned long long cap;       // records beyond it are counted, not written
    unsigned long long *state;    // tile status words (scan.cuh look-back)
    uint32_t epoch;
    unsigned long long *count;    // written by the last tile: the number of starts
    uint32_t pat_len;             // '\n' + literal 0
    uint32_t l1, l2, l3, lm;      // literal 1, literal 2, literal 3 (with the kind), literal 4 (mdev: the annotation's
                                  // opening, cdev: the node literal)
    uint8_t pat[PAT_MAX];
    uint32_t l9;                  // mdev cdev: the literal after the uuid, which ends in the node literal; the typed
                                  // layouts: the literal between the type ID and the key
    uint32_t l10;                 // the typed layouts: the literal after the key (the node literal)
};

template <int LAYOUT>
struct ParseSmem {
    alignas(16) uint8_t win[WIN<LAYOUT>];
    uint32_t mask[ROWS * (PARSE_THREADS / 32)];  // row-major: mask[row * 8 + warp] = the warp's ballot in that row
    uint32_t base[ROWS * (PARSE_THREADS / 32)];  // exclusive count of starts in front of that row-warp inside the tile
    unsigned long long tile_base;
};

__device__ __forceinline__ bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

template <int FMT, int LAYOUT>
__global__ void __launch_bounds__(PARSE_THREADS) k_cdi_decode(const __grid_constant__ ParseParams P) {
    constexpr int HALO_L = HALO<LAYOUT>, WIN_L = WIN<LAYOUT>;
    __shared__ ParseSmem<LAYOUT> S;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    const unsigned long long t0 = (unsigned long long)blockIdx.x * PT;
    // ---- stage [t0 - LEAD, t0 + PT + HALO): the buffer is padded, so only the front of tile 0 needs a guard
    {
        const uint4 *src = reinterpret_cast<const uint4 *>(P.doc + t0) - 1;
        uint4 *dst = reinterpret_cast<uint4 *>(S.win);
        for (uint32_t k = tid; k < (uint32_t)(WIN_L / 16); k += PARSE_THREADS)
            dst[k] = (blockIdx.x == 0 && k == 0) ? make_uint4(0, 0, 0, 0) : src[k];
    }
    __syncthreads();
    // bytes at or past the document's end read as 0 (the padding is zero and the window ends with the halo)
    const unsigned long long rest = P.len - t0;  // > 0: every tile holds a byte of the document
    const uint32_t wend = (uint32_t)(LEAD + (rest < (unsigned long long)(PT + HALO_L) ? rest : (unsigned long long)(PT + HALO_L)));
    auto at = [&](uint32_t q) -> uint8_t { return q < wend ? S.win[q] : (uint8_t)0; };
    // ---- starts: row r holds positions t0 + r * 256 + tid
    for (uint32_t r = 0; r < (uint32_t)ROWS; r++) {
        const uint32_t q = LEAD + r * PARSE_THREADS + tid;  // window offset of the position
        bool hit = q < wend && at(q - 1) == '\n';
        for (uint32_t k = 1; hit && k < P.pat_len; k++) hit = at(q - 1 + k) == P.pat[k];
        const uint32_t m = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) S.mask[r * (PARSE_THREADS / 32) + w] = m;
    }
    __syncthreads();
    // ---- slots: the 256 row-warp counts scanned in position order (thread t holds row t / 8, warp t % 8)
    uint32_t tot;
    const uint32_t cnt = __popc(S.mask[tid]);
    const uint32_t ex = kxscan::block_excl(cnt, &tot);
    S.base[tid] = ex;
    if (w == 0) {
        const unsigned long long excl = kxscan::lookback(P.state, blockIdx.x, tot, P.epoch);
        if (lane == 0) {
            S.tile_base = excl;
            if (blockIdx.x == gridDim.x - 1) *P.count = excl + tot;
        }
    }
    __syncthreads();
    // ---- decode: thread t takes the starts of row-warp t, in position order
    uint32_t m = S.mask[tid];
    unsigned long long slot = S.tile_base + S.base[tid];
    const uint32_t r = tid / (PARSE_THREADS / 32), ww = tid % (PARSE_THREADS / 32);
    for (; m; m &= m - 1u, slot++) {
        const uint32_t l = (uint32_t)__ffs((int)m) - 1u;
        uint32_t q = LEAD + r * PARSE_THREADS + ww * 32u + l + P.pat_len - 1u;  // after literal 0
        unsigned long long index = 0;
        const uint32_t name_at = q;
        for (uint32_t k = 0; k < 20u && is_digit(at(q)); k++, q++) index = index * 10ull + (at(q) - '0');
        const uint32_t name_end = q;
        q += P.l1;
        const bool quoted = FMT == KXPU_FMT_YAML && at(q) == '"';
        if (quoted) q++;
        uint8_t bdf[16] = {0};
        for (uint32_t k = 0; k < 16u; k++, q++) {
            const uint8_t c = at(q);
            if (c == '"' || c == '\n' || c == 0) break;
            bdf[k] = c;
        }
        if (quoted) q++;
        q += P.l2;
        uint32_t group = 0;
        for (uint32_t k = 0; k < 10u && is_digit(at(q)); k++, q++) group = group * 10u + (at(q) - '0');
        if (slot >= P.cap) continue;
        if constexpr (is_typed_layout<LAYOUT>) {  // the type ID follows the name's second copy and literal 4, then literal 9,
                                                  // the key up to its closing quote, literal 10 and (typed cdev) N
            q += P.l3 + (name_end - name_at) + P.lm;
            uint32_t type_id = 0;
            for (uint32_t k = 0; k < 10u && is_digit(at(q)); k++, q++) type_id = type_id * 10u + (at(q) - '0');
            q += P.l9;
            uint32_t kw[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, kl = 0;  // the key, packed as it sits in the record
            bool open = true;
#pragma unroll
            for (uint32_t k = 0; k < 40u; k++) {
                const uint8_t c = open ? at(q + k) : (uint8_t)0;
                open = open && c != '"' && c != '\n' && c != 0;
                if (open) { kw[k >> 2] |= (uint32_t)c << (8u * (k & 3u)); kl++; }
            }
            q += kl;
            uint32_t node = 0;
            if constexpr (LAYOUT == LAYOUT_TYPED_CDEV) {
                q += P.l10;
                for (uint32_t k = 0; k < 10u && is_digit(at(q)); k++, q++) node = node * 10u + (at(q) - '0');
            }
            uint32_t bw[4];
            memcpy(bw, bdf, 16);
            uint4 *o = reinterpret_cast<uint4 *>(static_cast<kxpu_vfvgpucdi *>(P.recs) + slot);
            o[0] = make_uint4(bw[0], bw[1], bw[2], bw[3]);
            o[1] = make_uint4(group, node, (uint32_t)index, (uint32_t)(index >> 32));
            o[2] = make_uint4(type_id, kl, kw[0], kw[1]);  // key_len, reserved[3] = 0
            o[3] = make_uint4(kw[2], kw[3], kw[4], kw[5]);
            o[4] = make_uint4(kw[6], kw[7], kw[8], kw[9]);
        } else if (LAYOUT == LAYOUT_PCI) {
            kxpu_cdidev d;
            memcpy(d.bdf, bdf, 16);
            d.iommu_group = group;
            d.vfio_cdev = 0;
            d.index = index;
            static_cast<kxpu_cdidev *>(P.recs)[slot] = d;
        } else if constexpr (LAYOUT == LAYOUT_CDEV) {  // N follows the name's second copy and the node literal
            q += P.l3 + (name_end - name_at) + P.lm;  // the second copy is as long as the first in a valid fragment
            uint32_t node = 0;
            for (uint32_t k = 0; k < 10u && is_digit(at(q)); k++, q++) node = node * 10u + (at(q) - '0');
            kxpu_cdidev d;
            memcpy(d.bdf, bdf, 16);
            d.iommu_group = group;
            d.vfio_cdev = node;
            d.index = index;
            static_cast<kxpu_cdidev *>(P.recs)[slot] = d;
        } else {  // the uuid follows the name's second copy: "<kind>=<index>" and the mdev annotation's opening
            q += P.l3;
            for (uint32_t k = 0; k < 20u && is_digit(at(q)); k++) q++;
            q += P.lm;
            kxpu_mdevcdi d;
            for (uint32_t k = 0; k < 36u; k++) d.uuid[k] = (char)at(q + k);
            d.iommu_group = group;
            memcpy(d.parent, bdf, 16);
            d.index = index;
            if constexpr (LAYOUT == LAYOUT_MDEV_CDEV) {  // N follows the uuid and the literal after it
                q += 36u + P.l9;
                uint32_t node = 0;
                for (uint32_t k = 0; k < 10u && is_digit(at(q)); k++, q++) node = node * 10u + (at(q) - '0');
                kxpu_mdevcdev *c = static_cast<kxpu_mdevcdev *>(P.recs) + slot;
                c->dev = d;
                *reinterpret_cast<uint4 *>(&c->vfio_cdev) = make_uint4(node, 0u, 0u, 0u);  // vfio_cdev, reserved[3]
            } else {
                static_cast<kxpu_mdevcdi *>(P.recs)[slot] = d;
            }
        }
    }
}

// bad = 1 unless *total == len and a[0, len) == b[0, len); a and b are 16-byte aligned
__global__ void __launch_bounds__(256) k_cdi_compare(const uint8_t *a, const uint8_t *b, unsigned long long len,
                                                     const unsigned long long *total, uint32_t *bad) {
    if (*total != len) {
        if (blockIdx.x == 0 && threadIdx.x == 0) *bad = 1u;
        return;
    }
    const unsigned long long n16 = len / 16, stride = (unsigned long long)gridDim.x * blockDim.x;
    const uint4 *a4 = reinterpret_cast<const uint4 *>(a), *b4 = reinterpret_cast<const uint4 *>(b);
    bool diff = false;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
        const uint4 x = a4[i], y = b4[i];
        diff |= ((x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w)) != 0u;
    }
    if (blockIdx.x == 0 && threadIdx.x < len % 16) diff |= a[n16 * 16 + threadIdx.x] != b[n16 * 16 + threadIdx.x];
    if (__syncthreads_or(diff) && threadIdx.x == 0) *bad = 1u;
}

}  // namespace kxparse

using namespace kxparse;

template <int FMT, int LAYOUT>
static void decode_launch(kxpu_ctx *ctx, uint32_t tiles, const ParseParams &P) {
    k_cdi_decode<FMT, LAYOUT><<<tiles, PARSE_THREADS, 0, ctx->stream>>>(P);
}

// LAYOUT_MDEV: out is kxpu_mdevcdi[cap], LAYOUT_MDEV_CDEV: kxpu_mdevcdev[cap], the typed layouts kxpu_vfvgpucdi[cap],
// else kxpu_cdidev[cap]
static int32_t cdi_parse(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len, void *out,
                         size_t cap, size_t *n, int layout, const char *what) {
    const bool mdev = layout == LAYOUT_MDEV || layout == LAYOUT_MDEV_CDEV;
    if (!ctx || !n || !kind || (len && !doc) || (cap && !out) || (format != KXPU_FMT_YAML && format != KXPU_FMT_JSON))
        return KXPU_E_INVALID;
    if (len >= (1ull << 32)) { KX_SET_ERR(ctx, "%s: a document of 2^32 bytes or more", what); return KXPU_E_UNSUPPORTED; }
    if (!kx_cdi_kind_ok(kind)) { KX_SET_ERR(ctx, "%s: kind is not a CDI vendor/class of at most 63 bytes", what); return KXPU_E_UNSUPPORTED; }
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    const bool typed = layout == LAYOUT_TYPED || layout == LAYOUT_TYPED_CDEV;
    std::string part[11];
    for (int k = 0; k < 11; k++) part[k] = kx_cdi_part(format, layout, k, kind);
    if (len == part[8].size() && memcmp(doc, part[8].data(), len) == 0) {  // the zero-device document
        *n = 0;
        return KXPU_OK;
    }
    // the shortest fragment: the literals, one-digit index (twice) and group (twice; cdev: the group and N), a one-byte
    // bdf, the uuid, a one-digit type ID and a one-byte key, and in JSON the separator after the device
    size_t lits = 0;
    for (int k : {0, 1, 2, 3, 4, 5, 9, 10}) lits += part[k].size();
    const size_t frag_min = lits + 5 + (mdev ? 36 : 0) + (typed ? 2 : 0) + (format == KXPU_FMT_JSON ? 1 : 0);
    const size_t fixed = part[6].size() + part[7].size();
    if (len < fixed + frag_min) { KX_SET_ERR(ctx, "%s: not a document the emitter writes", what); return KXPU_E_INVALID; }
    const size_t max_n = (len - fixed) / frag_min;  // no valid document of len bytes holds more devices
    const size_t rec_bytes = layout == LAYOUT_MDEV ? sizeof(kxpu_mdevcdi)
                             : layout == LAYOUT_MDEV_CDEV ? sizeof(kxpu_mdevcdev)
                             : typed ? sizeof(kxpu_vfvgpucdi) : sizeof(kxpu_cdidev);
    const uint32_t tiles = (uint32_t)((len + PT - 1) / PT);
    const size_t padded = (size_t)tiles * PT + HALO_MAX + LEAD;

    ParseParams P;
    memset(&P, 0, sizeof P);
    const std::string pat = "\n" + part[0];
    if (pat.size() > (size_t)PAT_MAX) return KXPU_E_INVALID;  // the literal grew: PAT_MAX must follow
    memcpy(P.pat, pat.data(), pat.size());
    P.pat_len = (uint32_t)pat.size();
    P.l1 = (uint32_t)part[1].size();
    P.l2 = (uint32_t)part[2].size();
    P.l3 = (uint32_t)part[3].size();
    P.lm = (uint32_t)part[4].size();
    P.l9 = (uint32_t)part[9].size();
    P.l10 = (uint32_t)part[10].size();

    KxScratch sc(ctx);
    uint8_t *d_doc = nullptr;
    void *d_recs = nullptr;
    unsigned long long *d_ctl = nullptr;  // [0] count, [1] compare verdict
    KX_CUDA(ctx, sc.alloc((void **)&d_doc, padded));
    KX_CUDA(ctx, sc.alloc(&d_recs, max_n * rec_bytes));
    KX_CUDA(ctx, sc.alloc((void **)&d_ctl, 16));
    cudaMemcpyAsync(d_doc, doc, len, cudaMemcpyHostToDevice, ctx->stream);
    cudaMemsetAsync(d_doc + len, 0, padded - len, ctx->stream);
    cudaMemsetAsync(d_ctl, 0, 16, ctx->stream);
    P.doc = d_doc;
    P.len = len;
    P.recs = d_recs;
    P.cap = max_n;
    P.count = d_ctl;
    P.state = kx_scan_state(ctx, tiles);
    if (!P.state) return KXPU_E_NOMEM;
    P.epoch = kx_next_epoch(ctx);

    KxTimer tm(ctx, KXPU_T_EMIT);  // decode, the re-emit and the compare, with the one host read of the count between
    if (layout == LAYOUT_TYPED) {
        if (format == KXPU_FMT_YAML) decode_launch<KXPU_FMT_YAML, LAYOUT_TYPED>(ctx, tiles, P);
        else decode_launch<KXPU_FMT_JSON, LAYOUT_TYPED>(ctx, tiles, P);
    } else if (layout == LAYOUT_TYPED_CDEV) {
        if (format == KXPU_FMT_YAML) decode_launch<KXPU_FMT_YAML, LAYOUT_TYPED_CDEV>(ctx, tiles, P);
        else decode_launch<KXPU_FMT_JSON, LAYOUT_TYPED_CDEV>(ctx, tiles, P);
    } else if (layout == LAYOUT_MDEV_CDEV) {
        if (format == KXPU_FMT_YAML) decode_launch<KXPU_FMT_YAML, LAYOUT_MDEV_CDEV>(ctx, tiles, P);
        else decode_launch<KXPU_FMT_JSON, LAYOUT_MDEV_CDEV>(ctx, tiles, P);
    } else if (mdev) {
        if (format == KXPU_FMT_YAML) decode_launch<KXPU_FMT_YAML, LAYOUT_MDEV>(ctx, tiles, P);
        else decode_launch<KXPU_FMT_JSON, LAYOUT_MDEV>(ctx, tiles, P);
    } else if (layout == LAYOUT_CDEV) {
        if (format == KXPU_FMT_YAML) decode_launch<KXPU_FMT_YAML, LAYOUT_CDEV>(ctx, tiles, P);
        else decode_launch<KXPU_FMT_JSON, LAYOUT_CDEV>(ctx, tiles, P);
    } else {
        if (format == KXPU_FMT_YAML) decode_launch<KXPU_FMT_YAML, LAYOUT_PCI>(ctx, tiles, P);
        else decode_launch<KXPU_FMT_JSON, LAYOUT_PCI>(ctx, tiles, P);
    }
    KX_LAUNCHED(ctx);
    unsigned long long count = 0;
    cudaMemcpyAsync(&count, d_ctl, 8, cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s decode failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (count == 0 || count > max_n) { KX_SET_ERR(ctx, "%s: not a document the emitter writes", what); return KXPU_E_INVALID; }
    uint8_t *d_emit = nullptr;
    unsigned long long *d_total = nullptr;
    int32_t rc = kx_cdi_emit_enqueue(ctx, format, kind, d_recs, (size_t)count, layout, sc, &d_emit, &d_total, false);
    if (rc != KXPU_OK) return rc;
    k_cdi_compare<<<(unsigned)ctx->sm_count * 4, 256, 0, ctx->stream>>>(d_doc, d_emit, len, d_total,
                                                                         reinterpret_cast<uint32_t *>(d_ctl + 1));
    KX_LAUNCHED(ctx);
    tm.stop();
    unsigned long long h[3] = {0, 0, 0};
    cudaMemcpyAsync(h, d_total, 16, cudaMemcpyDeviceToHost, ctx->stream);
    cudaMemcpyAsync(h + 2, d_ctl + 1, 8, cudaMemcpyDeviceToHost, ctx->stream);
    e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s verify failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[1] || h[2]) {  // a bdf / uuid / type the emitter refuses, or bytes it would not write
        KX_SET_ERR(ctx, "%s: not a document the emitter writes", what);
        return KXPU_E_INVALID;
    }
    *n = (size_t)count;
    if (cap < count) return KXPU_E_NOSPACE;
    cudaMemcpyAsync(out, d_recs, count * rec_bytes, cudaMemcpyDeviceToHost, ctx->stream);
    e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s D2H failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}

extern "C" int32_t kxpu_cdi_parse(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                                  kxpu_cdidev *out, size_t cap, size_t *n) {
    return cdi_parse(ctx, format, kind, doc, len, out, cap, n, LAYOUT_PCI, "cdi_parse");
}

extern "C" int32_t kxpu_cdi_parse_mdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                                       kxpu_mdevcdi *out, size_t cap, size_t *n) {
    return cdi_parse(ctx, format, kind, doc, len, out, cap, n, LAYOUT_MDEV, "cdi_parse_mdev");
}

extern "C" int32_t kxpu_cdi_parse_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                                       kxpu_cdidev *out, size_t cap, size_t *n) {
    return cdi_parse(ctx, format, kind, doc, len, out, cap, n, LAYOUT_CDEV, "cdi_parse_cdev");
}

extern "C" int32_t kxpu_cdi_parse_mdev_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc,
                                            size_t len, kxpu_mdevcdev *out, size_t cap, size_t *n) {
    return cdi_parse(ctx, format, kind, doc, len, out, cap, n, LAYOUT_MDEV_CDEV, "cdi_parse_mdev_cdev");
}

extern "C" int32_t kxpu_cdi_parse_vf_vgpu(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc, size_t len,
                                          kxpu_vfvgpucdi *out, size_t cap, size_t *n) {
    return cdi_parse(ctx, format, kind, doc, len, out, cap, n, LAYOUT_TYPED, "cdi_parse_vf_vgpu");
}

extern "C" int32_t kxpu_cdi_parse_vf_vgpu_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const uint8_t *doc,
                                               size_t len, kxpu_vfvgpucdi *out, size_t cap, size_t *n) {
    return cdi_parse(ctx, format, kind, doc, len, out, cap, n, LAYOUT_TYPED_CDEV, "cdi_parse_vf_vgpu_cdev");
}
