// read_ceiling.cu -- how fast the H100 reads the pci.ids text with the parse kernel's copy pattern, and with others.
//
// stage_probe reproduces the former staging engine of kxparse5::parse_kernel_v5 (before the 6 KiB copies of DESIGN
// K1) without the parse: ranges of 8 chunks of
// 2 KiB handed out to warps by ticket (drawn one range early), a private ring of 1-D TMA bulk copies per warp
// (cp.async.bulk + mbarrier), a copy of the next range's first chunks issued while the current one drains.  Per
// chunk every lane XORs one word of the staged bytes, so the copies cannot be optimised away.  The template
// arguments change one thing at a time: chunks per copy, ring depth, warps per CTA, the L2 evict-first hint, the
// 16 trailing bytes per copy, and CTA-contiguous tickets (one ticket per CTA and round, warp w takes range
// 8 * T + w).  ldg_probe is the plain grid-stride 16-byte read the others are measured against.
// Built by scripts/read_ceiling.py (nvcc -shared for sm_90a); C entry points at the end.
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

constexpr uint32_t CW = 2048, TRAIL = 16, RCH = 8, RANGE_BYTES = CW * RCH;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned long long evict_first() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_copy(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar, bool hint,
                                          unsigned long long pol) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    if (hint)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
                     "l"(src), "r"(bytes), "r"(bar), "l"(pol)
                     : "memory");
    else
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                     "r"(bytes), "r"(bar)
                     : "memory");
}
__device__ __forceinline__ bool bar_try(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok)
                 : "r"(bar), "r"(parity)
                 : "memory");
    return ok != 0u;
}

template <int CPC, int S, int WARPS, bool TRAILB>
struct Geo {
    static constexpr uint32_t COPY = CPC * CW + (TRAILB ? TRAIL : 0);  // bytes per bulk copy
    static constexpr uint32_t CPR = RCH / CPC;                         // copies per range
    static constexpr uint32_t WARP_SMEM = (S * COPY + 8 * S + 15) / 16 * 16;  // ring + its mbarriers; bulk copies land 16-B aligned
    static constexpr uint32_t SMEM = WARPS * WARP_SMEM + 16;           // + the CTA's ticket slots
};

template <int CPC, int S, int WARPS, bool HINT, bool TRAILB, bool CTA_T>
__global__ void __launch_bounds__(WARPS * 32) stage_probe(const uint8_t *text, uint32_t num_ranges, uint32_t *ticket, uint32_t *sink) {
    using G = Geo<CPC, S, WARPS, TRAILB>;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
    const uint32_t ring = smem_u32(smem) + w * G::WARP_SMEM, bars = ring + S * G::COPY;
    volatile uint32_t *slots = reinterpret_cast<volatile uint32_t *>(smem + WARPS * G::WARP_SMEM);  // CTA tickets, rounds k % 3
    const unsigned long long pol = evict_first();
    if (lane == 0) {
        for (int s = 0; s < S; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bars + 8u * s));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // range of a round (CTA tickets) or of a drawn ticket (warp tickets)
    uint32_t round = 0;    // CTA tickets: round of the range the issue cursor is in
    uint32_t pending = 0;  // CTA tickets, thread 0: the ticket of the round after the next
    if (CTA_T) {
        if (threadIdx.x == 0) {
            slots[0] = atomicAdd(ticket, 1u);
            slots[1] = atomicAdd(ticket, 1u);
            pending = atomicAdd(ticket, 1u);
        }
        __syncthreads();
    }
    auto range_of = [&](uint32_t k) -> uint32_t {  // CTA tickets: warp w's range in round k
        const uint32_t T = slots[k % 3u];
        return T * (uint32_t)WARPS + w < num_ranges && T < num_ranges / WARPS ? T * (uint32_t)WARPS + w : 0xffffffffu;
    };
    // issue cursor (lane 0's registers): range ir, copy ik of it; ir_pre is the ticket drawn one range early
    uint32_t ir = 0, ir_pre = 0, ik = 0;
    if (CTA_T) {
        ir = range_of(0);
    } else if (lane == 0) {
        ir = atomicAdd(ticket, 1u);
        ir_pre = atomicAdd(ticket, 1u);
    }
    ir = __shfl_sync(0xffffffffu, ir, 0);
    uint32_t s_issue = 0, s_cons = 0, phase = 0, inflight = 0, acc = 0;
    // CTA tickets: every warp of the CTA ends its ranges together (a barrier per round); a warp without a range in
    // a round still takes part
    const bool cta_done0 = CTA_T && slots[0] >= num_ranges / WARPS;
    if (cta_done0) return;
    auto issue_next = [&]() {
        bool ok = ir < num_ranges;
        if (ok && lane == 0)
            bulk_copy(ring + s_issue * G::COPY, text + (unsigned long long)ir * RANGE_BYTES + (unsigned long long)ik * CPC * CW, G::COPY,
                      bars + 8u * s_issue, HINT, pol);
        if (ok) {
            s_issue = s_issue + 1u == (uint32_t)S ? 0u : s_issue + 1u;
            inflight++;
            if (++ik == G::CPR) {
                ik = 0;
                if (CTA_T) {
                    ir = range_of(++round);
                } else {
                    if (lane == 0) {
                        ir = ir_pre;
                        ir_pre = atomicAdd(ticket, 1u);
                    }
                    ir = __shfl_sync(0xffffffffu, ir, 0);
                }
            }
        }
        return ok;
    };
    for (int j = 0; j < S; j++) issue_next();
    uint32_t cons_k = 0, cons_round = 0;
    while (inflight) {
        const uint32_t bar = bars + 8u * s_cons;
        while (!bar_try(bar, (phase >> s_cons) & 1u)) {
        }
        phase ^= 1u << s_cons;
#pragma unroll
        for (int c = 0; c < CPC; c++) {
            uint32_t v;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(ring + s_cons * G::COPY + c * CW + lane * 4u));
            acc ^= v;
        }
        __syncwarp();
        inflight--;
        s_cons = s_cons + 1u == (uint32_t)S ? 0u : s_cons + 1u;
        if (CTA_T && ++cons_k == G::CPR) {
            // round cons_round is through: the ticket of round cons_round + 2 (drawn a round ago) goes into the slot
            // of round cons_round - 1, which nobody reads any more; the barrier publishes it
            cons_k = 0;
            if (threadIdx.x == 0) {
                slots[(cons_round + 2u) % 3u] = pending;
                pending = atomicAdd(ticket, 1u);
            }
            __syncthreads();
            ++cons_round;
            if (slots[cons_round % 3u] >= num_ranges / WARPS) break;  // the whole CTA is through
        }
        issue_next();
    }
    if (acc == 0x9e3779b9u) atomicXor(sink, acc);
}

__global__ void __launch_bounds__(256) ldg_probe(const uint4 *p, unsigned long long n16, uint32_t *sink) {
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t acc = 0;
    for (; i + 3 * stride < n16; i += 4 * stride) {
        const uint4 a = __ldg(p + i), b = __ldg(p + i + stride), c = __ldg(p + i + 2 * stride), d = __ldg(p + i + 3 * stride);
        acc ^= a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w ^ c.x ^ c.y ^ c.z ^ c.w ^ d.x ^ d.y ^ d.z ^ d.w;
    }
    for (; i < n16; i += stride) {
        const uint4 a = __ldg(p + i);
        acc ^= a.x ^ a.y ^ a.z ^ a.w;
    }
    if (acc == 0x9e3779b9u) atomicXor(sink, acc);
}

struct Variant {
    const char *name;
    const void *fn;
    uint32_t smem, threads;
    bool cta_tickets;
};

#define V(name, CPC, S, W, HINT, TR, CT)                                                                              \
    { name, (const void *)stage_probe<CPC, S, W, HINT, TR, CT>, Geo<CPC, S, W, TR>::SMEM, W * 32, CT }
const Variant VARIANTS[] = {
    V("a_parse_staging", 1, 3, 8, true, true, false),  // the parse kernel's geometry
    V("copy_4k", 2, 3, 8, true, true, false),
    V("copy_4k_ring2", 2, 2, 8, true, true, false),  // the ring bytes of ring_4
    V("copy_8k", 4, 3, 8, true, true, false),
    V("copy_16k_ring2_6w", 8, 2, 6, true, true, false),  // 3 x 16 KiB per warp does not fit; two stages, six warps
    V("ring_2", 1, 2, 8, true, true, false),
    V("ring_4", 1, 4, 8, true, true, false),
    V("no_evict_first", 1, 3, 8, false, true, false),
    V("exact_cw", 1, 3, 8, true, false, false),
    V("cta_tickets", 1, 3, 8, true, true, true),
};
constexpr int NV = sizeof(VARIANTS) / sizeof(VARIANTS[0]);

struct State {
    uint8_t *text = nullptr;
    unsigned long long n = 0;
    uint32_t *ticket = nullptr, *sink = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    int sms = 0;
} g;

}  // namespace

extern "C" {

int rc_num_variants() { return NV + 1; }
const char *rc_variant_name(int v) { return v < NV ? VARIANTS[v].name : "c_ldg128_grid_stride"; }

// CTAs per SM the variant runs at (occupancy of its registers and shared memory)
int rc_ctas_per_sm(int v) {
    int per_sm = 0;
    if (v < NV) {
        cudaFuncSetAttribute(VARIANTS[v].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)VARIANTS[v].smem);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, VARIANTS[v].fn, (int)VARIANTS[v].threads, VARIANTS[v].smem);
    } else {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ldg_probe, 256, 0);
    }
    return per_sm;
}

// uploads the text (n bytes) into a fresh HBM buffer
int rc_setup(const uint8_t *host, unsigned long long n) {
    if (cudaDeviceGetAttribute(&g.sms, cudaDevAttrMultiProcessorCount, 0) != cudaSuccess) return -1;
    if (cudaMalloc(&g.text, n + 65536) != cudaSuccess) return -2;
    if (cudaMemcpy(g.text, host, n, cudaMemcpyHostToDevice) != cudaSuccess) return -3;
    if (cudaMalloc(&g.ticket, 64) != cudaSuccess || cudaMalloc(&g.sink, 64) != cudaSuccess) return -4;
    cudaEventCreate(&g.e0);
    cudaEventCreate(&g.e1);
    g.n = n;
    return 0;
}

// ranges of 16 KiB the variant reads: whole ranges only; CTA tickets read whole rounds of one range per warp
static uint32_t ranges_of(int v) {
    const uint32_t nr = (uint32_t)((g.n - TRAIL) / RANGE_BYTES), warps = VARIANTS[v].threads / 32;
    return VARIANTS[v].cta_tickets ? nr / warps * warps : nr;
}

// bytes one launch of the variant reads
unsigned long long rc_bytes(int v) { return v < NV ? (unsigned long long)ranges_of(v) * RANGE_BYTES : g.n / 16 * 16; }

// one launch, timed with CUDA events; returns ms (negative: CUDA error)
float rc_time(int v) {
    const int per_sm = rc_ctas_per_sm(v);
    cudaMemset(g.ticket, 0, 4);
    cudaEventRecord(g.e0);
    if (v < NV) {
        const uint32_t nr = ranges_of(v);
        void *args[] = {(void *)&g.text, (void *)&nr, (void *)&g.ticket, (void *)&g.sink};
        cudaLaunchKernel(VARIANTS[v].fn, dim3(per_sm * g.sms), dim3(VARIANTS[v].threads), args, VARIANTS[v].smem, 0);
    } else {
        ldg_probe<<<per_sm * g.sms, 256>>>(reinterpret_cast<const uint4 *>(g.text), g.n / 16, g.sink);
    }
    cudaEventRecord(g.e1);
    if (cudaEventSynchronize(g.e1) != cudaSuccess || cudaPeekAtLastError() != cudaSuccess) return -1.0f;
    float ms = 0;
    cudaEventElapsedTime(&ms, g.e0, g.e1);
    return ms;
}

const char *rc_last_error() { return cudaGetErrorString(cudaGetLastError()); }

void rc_teardown() {
    cudaFree(g.text);
    cudaFree(g.ticket);
    cudaFree(g.sink);
    cudaEventDestroy(g.e0);
    cudaEventDestroy(g.e1);
}
}
