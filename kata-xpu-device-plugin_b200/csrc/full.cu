// full.cu -- SURVEY 8(f) row 4: the rest of the pci.ids model -- subsystem rows
// (vendor, device, subvendor, subdevice) and the class / subclass / prog-if section -- on top of the
// (vendor,device) table.  The reference scans these lines and ignores them (device_plugin.go:
// 229-237); their meaning is the file's own format statement (utils/pci.ids:23-27, :38195-38200),
// restated in the test oracle (full_build) with the reference's matching rules carried one
// level down (raw byte prefixes, first occurrence wins at every level).
//
// Every line is governed by the nearest top-level line in front of it (vendor / class) and, for the
// double-tab lines, by the nearest single-tab line behind that top-level line (device / subclass).
// Both are prefix properties with an associative combine:
//     (top, tab1) . (top', tab1') = top' present ? (top', tab1') : (top, tab1' present ? tab1' : tab1)
// so: pass A, one warp per 2 KiB chunk, every lane summarises its 64 bytes, the warp combines them
// and publishes the chunk's summary (and class_first); passes B and C look back over the chunk
// summaries for the carry, scan the lane summaries inside the warp and walk the lines again --
// B records the winning subclass lines (their class line must be the first of its id), C the
// double-tab rows whose governing single-tab line is the WINNING line of its key ((vendor,device)
// row of the table / subclass line of pass B).  Double-tab rows live in a 64-bit-key hash table
// (atomicMin of the line offset: first occurrence wins).  A "next" row: built for parity and
// reasonable speed (one coalesced read of the text per pass), not tuned like the hot kernel.
#include <algorithm>
#include <new>
#include <vector>

#include "internal.cuh"
#include "parse_common.cuh"

namespace kxfull {

using kxparse::CW;
constexpr int WARPS = 8;
constexpr int STG = CW + 32;  // byte in front of the chunk + chunk + line-head lookahead
constexpr unsigned long long HAS = 1ull << 63;
constexpr unsigned long long OFF_MASK = (1ull << 44) - 1;
// top word:  [63] present, [62:61] 1 vendor (4 hex) / 2 class ("C " + 2 hex) / 0 other, [59:44] id, [43:0] offset
// tab1 word: [63] present, [62] four hex digits follow the tab, [61] at least two do, [59:44] the four-digit value (or the
//            two-digit value << 8): parsed without looking at the governing line, which a lane may not know yet; [43:0] offset
// empty-slot key.  It is also a legal subsystem key (\t\tffff ffff under device ffff of vendor ffff): that key lives
// in the dedicated slot [cap] behind the probed ones, as key 0xffffffff does in the (vendor,device) table
constexpr unsigned long long KEY_EMPTY = ~0ull;

struct HSlot { unsigned long long key, line; };

struct Params {
    const uint8_t *text;
    unsigned long long n;
    uint32_t num_chunks;
    unsigned long long *top_state, *tab_state;  // [num_chunks] chunk summaries
    unsigned long long *class_first;            // [256]
    unsigned long long *sub_line;               // [65536] winning subclass line of (class << 8 | subclass)
    HSlot *hs, *hp;                             // subsystem rows [hcap + 1] / prog-if rows [pcap + 1] (first occurrence: atomicMin of the line)
    uint32_t hcap, hshift, pcap, pshift;
    uint32_t *flags;                            // [0] subsystem table overflow, [1] prog-if table overflow
    KxTableDev tab;                             // the finished (vendor,device) table of the same text
};

struct State { unsigned long long top, tab; };
__device__ __forceinline__ State combine(const State a, const State b) {
    State r;
    if (b.top & HAS) { r = b; return r; }
    r.top = a.top;
    r.tab = (b.tab & HAS) ? b.tab : a.tab;
    return r;
}

__device__ __forceinline__ bool lhex(uint32_t c) { return (c - 0x30u < 10u) || (c - 0x61u < 6u); }
__device__ __forceinline__ uint32_t hv(uint32_t c) { return c <= 0x39u ? c - 0x30u : c - 0x61u + 10u; }
__device__ __forceinline__ bool hex_n(const uint8_t *s, int k, uint32_t &v) {
    v = 0;
    for (int i = 0; i < k; i++) {
        if (!lhex(s[i])) return false;
        v = v * 16u + hv(s[i]);
    }
    return true;
}

// chunk g into buf: buf[0] = byte in front of the chunk ('\n' for the first chunk), buf[1 + p] = text[g*CW + p];
// bytes behind the text read as '\n' (EOF ends the last line)
__device__ __forceinline__ void stage(const Params &P, uint32_t g, uint32_t lane, uint8_t *buf) {
    const long long base = (long long)g * CW - 1;
    for (int i = (int)lane; i < STG; i += 32) {
        const long long q = base + i;
        buf[i] = q < 0 ? (uint8_t)'\n' : ((unsigned long long)q < P.n ? P.text[q] : (uint8_t)'\n');
    }
    __syncwarp();
}

// walk the line starts of my 64 bytes; f(kind, p, state) with kind 0 top / 1 tab1 / 2 tab2, p = chunk-relative offset.
// `s` runs along: a top-level line replaces both words, a single-tab line the tab word.
template <typename F>
__device__ __forceinline__ void walk(const Params &P, uint32_t g, uint32_t lane, const uint8_t *buf, State &s, F f) {
    const unsigned long long cbase = (unsigned long long)g * CW;
    for (uint32_t p = lane * 64u; p < lane * 64u + 64u; p++) {
        if (cbase + p >= P.n) break;
        if (buf[p] != (uint8_t)'\n') continue;  // buf[p] is the byte in front of position p
        const uint8_t *l = buf + 1 + p;
        const uint32_t c0 = l[0];
        if (c0 == (uint32_t)'#' || c0 == (uint32_t)'\n') {
            if (c0 == (uint32_t)'\n') { s.top = HAS | ((cbase + p) & OFF_MASK); s.tab = 0; }  // an empty line is a top-level line
            continue;
        }
        if (c0 == (uint32_t)'\t') {
            if (l[1] == (uint8_t)'\t') { f(2, p, s); continue; }
            uint32_t id = 0, id2 = 0;
            const bool ok4 = hex_n(l + 1, 4, id), ok2 = ok4 || hex_n(l + 1, 2, id2);
            if (!ok4) id = id2 << 8;
            s.tab = HAS | (ok4 ? 1ull << 62 : 0ull) | (ok2 ? 1ull << 61 : 0ull) | ((unsigned long long)id << 44) | ((cbase + p) & OFF_MASK);
            f(1, p, s);
            continue;
        }
        uint32_t id = 0, kind = 0;
        if (c0 == (uint32_t)'C' && l[1] == (uint8_t)' ' && hex_n(l + 2, 2, id)) kind = 2u;
        else if (hex_n(l, 4, id)) kind = 1u;
        else id = 0;
        s.top = HAS | ((unsigned long long)kind << 61) | ((unsigned long long)id << 44) | ((cbase + p) & OFF_MASK);
        s.tab = 0;
        f(0, p, s);
    }
}

// pass A: chunk summaries, class_first
__global__ void __launch_bounds__(WARPS * 32) k_summary(const Params P) {
    __shared__ uint8_t s_buf[WARPS][STG];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t g = blockIdx.x * WARPS + w;
    if (g >= P.num_chunks) return;
    stage(P, g, lane, s_buf[w]);
    State s{0, 0};
    walk(P, g, lane, s_buf[w], s, [&](int kind, uint32_t, const State &st) {
        if (kind == 0 && ((st.top >> 61) & 3ull) == 2ull) atomicMin(&P.class_first[(st.top >> 44) & 0xffull], st.top & OFF_MASK);
    });
    // combine over the lanes, in order
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        State o;
        o.top = __shfl_up_sync(0xffffffffu, s.top, d);
        o.tab = __shfl_up_sync(0xffffffffu, s.tab, d);
        if (lane >= (uint32_t)d) s = combine(o, s);
    }
    if (lane == 31) { P.top_state[g] = s.top; P.tab_state[g] = s.tab; }
}

__device__ __forceinline__ void hash_min(HSlot *hs, uint32_t cap, uint32_t shift, uint32_t *overflow, unsigned long long key, unsigned long long line) {
    if (key == KEY_EMPTY) { atomicMin(&hs[cap].line, line); return; }
    uint32_t slot = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> shift);
    for (uint32_t step = 0; step < 2048u && step < cap; step++) {
        const unsigned long long k = __ldcg(&hs[slot].key);
        if (k == key) { atomicMin(&hs[slot].line, line); return; }
        if (k == KEY_EMPTY) {
            const unsigned long long old = atomicCAS(&hs[slot].key, KEY_EMPTY, key);
            if (old == KEY_EMPTY || old == key) { atomicMin(&hs[slot].line, line); return; }
        }
        slot = (slot + 1u) & (cap - 1u);
    }
    *overflow = 1u;
}
__device__ __forceinline__ unsigned long long hash_get(const HSlot *hs, uint32_t cap, uint32_t shift, unsigned long long key) {
    if (key == KEY_EMPTY) return hs[cap].line;
    uint32_t slot = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> shift);
    for (uint32_t step = 0; step < cap; step++) {
        const unsigned long long k = hs[slot].key;
        if (k == key) return hs[slot].line;
        if (k == KEY_EMPTY) break;
        slot = (slot + 1u) & (cap - 1u);
    }
    return KX_NO_OFF;
}

// the winning line of (vendor, device) in the finished table, or KX_NO_OFF
__device__ __forceinline__ unsigned long long device_line(const KxTableDev &tb, uint32_t key) {
    const uint32_t slot = kxparse::table_find(tb, key);
    if (slot == 0xffffffffu) return KX_NO_OFF;
    const KxSlot &s = tb.slots[slot];
    return (s.row >= 0) ? s.min_line : KX_NO_OFF;
}

// pass B (PASS 1): winning subclass lines; pass C (PASS 2): double-tab rows under winning single-tab lines
template <int PASS>
__global__ void __launch_bounds__(WARPS * 32) k_rows(const Params P) {
    __shared__ uint8_t s_buf[WARPS][STG];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t g = blockIdx.x * WARPS + w;
    if (g >= P.num_chunks) return;
    stage(P, g, lane, s_buf[w]);
    // carry into the chunk: nearest top word in front; the tab word of the nearest chunk that has one, unless a
    // chunk with a top-level line (and no single-tab line behind it) lies in between
    State carry{0, 0};
    {
        bool top_done = false, tab_done = false;
        for (long long q0 = (long long)g - 1; q0 >= 0 && !(top_done && tab_done); q0 -= 32) {
            const long long q = q0 - lane;
            const unsigned long long t = q >= 0 ? P.top_state[q] : 0ull, d = q >= 0 ? P.tab_state[q] : 0ull;
            const uint32_t tm = __ballot_sync(0xffffffffu, (t & HAS) != 0), dm = __ballot_sync(0xffffffffu, (d & HAS) != 0);
            if (!tab_done && (tm | dm)) {
                const uint32_t first = (uint32_t)__ffs((int)(tm | dm)) - 1u;  // nearest chunk with either
                const unsigned long long dd = __shfl_sync(0xffffffffu, d, first);
                carry.tab = (dd & HAS) ? dd : 0ull;
                tab_done = true;
            }
            if (!top_done && tm) {
                carry.top = __shfl_sync(0xffffffffu, t, (uint32_t)__ffs((int)tm) - 1u);
                top_done = true;
            }
        }
    }
    // lane summaries -> state at the start of my 64 bytes
    State mine{0, 0};
    walk(P, g, lane, s_buf[w], mine, [](int, uint32_t, const State &) {});
    State inc = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        State o;
        o.top = __shfl_up_sync(0xffffffffu, inc.top, d);
        o.tab = __shfl_up_sync(0xffffffffu, inc.tab, d);
        if (lane >= (uint32_t)d) inc = combine(o, inc);
    }
    State excl;
    excl.top = __shfl_up_sync(0xffffffffu, inc.top, 1);
    excl.tab = __shfl_up_sync(0xffffffffu, inc.tab, 1);
    if (lane == 0) { excl.top = 0; excl.tab = 0; }
    State s = combine(carry, excl);
    const unsigned long long cbase = (unsigned long long)g * CW;
    const uint8_t *buf = s_buf[w];
    walk(P, g, lane, buf, s, [&](int kind, uint32_t p, const State &st) {
        if (!(st.top & HAS)) return;
        const uint32_t tk = (uint32_t)(st.top >> 61) & 3u, tid = (uint32_t)(st.top >> 44) & 0xffffu;
        const unsigned long long anchor = st.top & OFF_MASK;
        if (PASS == 1) {
            // a subclass line under the FIRST line of its class id
            if (kind == 1 && tk == 2u && (st.tab & (1ull << 61)) && P.class_first[tid & 0xffu] == anchor)
                atomicMin(&P.sub_line[((tid & 0xffu) << 8) | ((uint32_t)(st.tab >> 52) & 0xffu)], cbase + p);
            return;
        }
        if (kind != 2 || !(st.tab & HAS)) return;
        const uint32_t did = (uint32_t)(st.tab >> 44) & 0xffffu;
        const unsigned long long tab_off = st.tab & OFF_MASK;
        const uint8_t *l = buf + 1 + p;
        uint32_t a, b;
        if (tk == 1u) {
            // subsystem line: the vendor line is the first of its id and the device line is the winning one
            if (!(st.tab & (1ull << 62)) || P.tab.vendor_first[tid] != anchor || device_line(P.tab, (tid << 16) | did) != tab_off) return;
            if (!hex_n(l + 2, 4, a) || l[6] != (uint8_t)' ' || !hex_n(l + 7, 4, b)) return;
            hash_min(P.hs, P.hcap, P.hshift, P.flags, ((unsigned long long)tid << 48) | ((unsigned long long)did << 32) | ((unsigned long long)a << 16) | b, cbase + p);
        } else if (tk == 2u) {
            const uint32_t c = tid & 0xffu, sc = (did >> 8) & 0xffu;
            if (!(st.tab & (1ull << 61)) || P.class_first[c] != anchor || P.sub_line[(c << 8) | sc] != tab_off) return;
            if (!hex_n(l + 2, 2, a)) return;
            hash_min(P.hp, P.pcap, P.pshift, P.flags + 1, (3ull << 24) | ((unsigned long long)c << 16) | ((unsigned long long)sc << 8) | a, cbase + p);
        }
    });
}

__global__ void k_fill(unsigned long long *p, size_t n) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = ~0ull;
}

__global__ void k_lookup(const Params P, const unsigned long long *trunc, int kind, const unsigned long long *keys, size_t n, long long *out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long key = keys[i], tr = *trunc;
    unsigned long long line = KX_NO_OFF;
    if (kind == 0) {
        if (key < 65536ull) line = P.tab.vendor_first[key];
    } else if (kind == 2 && (key >> 24) == 1ull && (key & 0xffffull) == 0ull) {
        line = P.class_first[(key >> 16) & 0xffull];
    } else if (kind == 2 && (key >> 24) == 2ull && (key & 0xffull) == 0ull) {
        line = P.sub_line[(key >> 8) & 0xffffull];
    } else if (kind == 1) {
        line = hash_get(P.hs, P.hcap, P.hshift, key);
    } else if (kind == 2 && (key >> 24) == 3ull) {
        line = hash_get(P.hp, P.pcap, P.pshift, key);
    }
    out[i] = (line != KX_NO_OFF && line < tr) ? (long long)line : -1ll;
}

}  // namespace kxfull

using namespace kxfull;

struct kxpu_full {
    uint8_t *arena = nullptr;
    Params P{};
    const unsigned long long *trunc = nullptr;  // the (vendor,device) table's cut-off
    kxpu_table *table = nullptr;                // borrowed: must outlive this object
};

extern "C" int32_t kxpu_full_free(kxpu_ctx *ctx, kxpu_full *f) {
    KX_ENTER(ctx);
    if (!f) return KXPU_OK;
    cudaStreamSynchronize(ctx->stream);
    if (f->arena) cudaFree(f->arena);
    delete f;
    return KXPU_OK;
}

extern "C" int32_t kxpu_pciids_full_load_device(kxpu_ctx *ctx, const void *d_text, size_t n, kxpu_table *t, kxpu_full **out) {
    KX_ENTER(ctx);
    if (!out || !t || (!d_text && n)) return KXPU_E_INVALID;
    if (n >= (1ull << 44)) return KXPU_E_UNSUPPORTED;
    *out = nullptr;
    const uint32_t num_chunks = (uint32_t)((n + CW - 1) / CW);
    uint32_t hcap = 1u << 17, pcap = 1u << 12;
    for (int attempt = 0; attempt < 12; attempt++) {
        kxpu_full *f = new (std::nothrow) kxpu_full();
        if (!f) return KXPU_E_NOMEM;
        uint32_t lg = 0, plg = 0;
        while ((1u << lg) < hcap) lg++;
        while ((1u << plg) < pcap) plg++;
        size_t off = 0;
        auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
        const size_t o_cf = take(256 * 8), o_sl = take(65536 * 8), o_hs = take((size_t)(hcap + 1) * sizeof(HSlot)), o_hp = take((size_t)(pcap + 1) * sizeof(HSlot));
        const size_t ff_words = off / 8;
        const size_t o_fl = take(64), o_ts = take((size_t)(num_chunks + 1) * 8), o_ds = take((size_t)(num_chunks + 1) * 8);
        if (cudaMalloc((void **)&f->arena, off) != cudaSuccess) {
            cudaGetLastError();
            delete f;
            return KXPU_E_NOMEM;
        }
        Params &P = f->P;
        P.text = (const uint8_t *)d_text; P.n = n; P.num_chunks = num_chunks;
        P.class_first = (unsigned long long *)(f->arena + o_cf); P.sub_line = (unsigned long long *)(f->arena + o_sl);
        P.hs = (HSlot *)(f->arena + o_hs); P.hcap = hcap; P.hshift = 64 - lg;
        P.hp = (HSlot *)(f->arena + o_hp); P.pcap = pcap; P.pshift = 64 - plg;
        P.flags = (uint32_t *)(f->arena + o_fl);
        P.top_state = (unsigned long long *)(f->arena + o_ts); P.tab_state = (unsigned long long *)(f->arena + o_ds);
        P.tab = t->dev;
        f->trunc = t->dev.trunc;
        f->table = t;
        k_fill<<<4 * ctx->sm_count, 256, 0, ctx->stream>>>((unsigned long long *)f->arena, ff_words);
        cudaMemsetAsync(P.flags, 0, 64, ctx->stream);
        ctx->launches++;
        if (num_chunks) {
            const unsigned grid = (num_chunks + WARPS - 1) / WARPS;
            k_summary<<<grid, WARPS * 32, 0, ctx->stream>>>(P);
            k_rows<1><<<grid, WARPS * 32, 0, ctx->stream>>>(P);
            k_rows<2><<<grid, WARPS * 32, 0, ctx->stream>>>(P);
            ctx->launches += 3;
        }
        uint32_t h_flag[2] = {0, 0};
        cudaMemcpyAsync(h_flag, P.flags, 8, cudaMemcpyDeviceToHost, ctx->stream);
        const cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) {
            KX_SET_ERR(ctx, "full model build failed: %s", cudaGetErrorString(e));
            cudaFree(f->arena);
            delete f;
            return KXPU_E_CUDA;
        }
        if (h_flag[0] || h_flag[1]) {  // more double-tab rows than a hash table holds: four times the slots, again
            cudaFree(f->arena);
            delete f;
            if (hcap >= (1u << 28)) return KXPU_E_CAPACITY;
            if (h_flag[0]) hcap <<= 2;
            if (h_flag[1]) pcap <<= 2;
            continue;
        }
        *out = f;
        return KXPU_OK;
    }
    return KXPU_E_CAPACITY;
}

extern "C" int32_t kxpu_full_export(kxpu_ctx *ctx, kxpu_full *f, int32_t kind, uint64_t *keys, uint64_t *line_off, size_t cap,
                                    uint32_t *n_rows) {
    KX_ENTER(ctx);
    if (!f || !n_rows || kind < 0 || kind > 2) return KXPU_E_INVALID;
    unsigned long long tr = KX_NO_OFF;
    KX_CUDA(ctx, cudaMemcpyAsync(&tr, f->trunc, 8, cudaMemcpyDeviceToHost, ctx->stream));
    std::vector<std::pair<uint64_t, uint64_t>> rows;  // (line, key)
    auto take_array = [&](const unsigned long long *d, size_t cnt, auto keyfn) -> int32_t {
        std::vector<unsigned long long> h(cnt);
        KX_CUDA(ctx, cudaMemcpyAsync(h.data(), d, cnt * 8, cudaMemcpyDeviceToHost, ctx->stream));
        KX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (size_t i = 0; i < cnt; i++)
            if (h[i] != KX_NO_OFF && h[i] < tr) rows.emplace_back(h[i], keyfn(i));
        return KXPU_OK;
    };
    int32_t rc = KXPU_OK;
    if (kind == 0) rc = take_array(f->P.tab.vendor_first, 65536, [](size_t i) { return (uint64_t)i; });
    if (kind == 2) {
        rc = take_array(f->P.class_first, 256, [](size_t i) { return (1ull << 24) | ((uint64_t)i << 16); });
        if (rc == KXPU_OK) rc = take_array(f->P.sub_line, 65536, [](size_t i) { return (2ull << 24) | ((uint64_t)i << 8); });
    }
    if (rc != KXPU_OK) return rc;
    if (kind == 1 || kind == 2) {
        const HSlot *d = kind == 1 ? f->P.hs : f->P.hp;
        const uint32_t cnt = kind == 1 ? f->P.hcap : f->P.pcap;
        std::vector<HSlot> h((size_t)cnt + 1);  // + the dedicated slot [cnt], whose key reads KEY_EMPTY
        KX_CUDA(ctx, cudaMemcpyAsync(h.data(), d, ((size_t)cnt + 1) * sizeof(HSlot), cudaMemcpyDeviceToHost, ctx->stream));
        KX_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (size_t i = 0; i <= cnt; i++)
            if ((h[i].key != KEY_EMPTY || i == cnt) && h[i].line != KX_NO_OFF && h[i].line < tr) rows.emplace_back(h[i].line, h[i].key);
    }
    std::sort(rows.begin(), rows.end());  // file order
    *n_rows = (uint32_t)rows.size();
    if (cap < rows.size()) return KXPU_E_NOSPACE;
    if (rows.size() && (!keys || !line_off)) return KXPU_E_INVALID;
    for (size_t i = 0; i < rows.size(); i++) { keys[i] = rows[i].second; line_off[i] = rows[i].first; }
    return KXPU_OK;
}

extern "C" int32_t kxpu_full_lookup(kxpu_ctx *ctx, kxpu_full *f, int32_t kind, const uint64_t *keys, size_t n, int64_t *line_off_out) {
    KX_ENTER(ctx);
    if (!f || kind < 0 || kind > 2 || (n && (!keys || !line_off_out))) return KXPU_E_INVALID;
    if (n == 0) return KXPU_OK;
    KxScratch sc(ctx);
    unsigned long long *d_keys = nullptr;
    long long *d_out = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&d_keys, n * 8));
    KX_CUDA(ctx, sc.alloc((void **)&d_out, n * 8));
    cudaMemcpyAsync(d_keys, keys, n * 8, cudaMemcpyHostToDevice, ctx->stream);
    k_lookup<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(f->P, f->trunc, kind, d_keys, n, d_out);
    KX_LAUNCHED(ctx);
    cudaMemcpyAsync(line_off_out, d_out, n * 8, cudaMemcpyDeviceToHost, ctx->stream);
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "full lookup failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}
