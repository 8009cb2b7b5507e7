// emit.cu -- K6 CDI spec emit (YAML / JSON), K7 Allocate names, ListAndWatch wire bytes.
//
// Reference: generateCDISpec (pkg/device_plugin/device_plugin.go:55-80), CdiSpec.Save
// (cdi/spec.go:85-127), updateResponseForCDI / QualifiedName
// (pkg/device_plugin/generic_device_plugin.go:274-299, cdi/cdi-utils.go:9) and the
// ListAndWatchResponse send (generic_device_plugin.go:224).
//
// Every output is a concatenation of per-device fragments whose length depends on the data
// (decimal widths, the YAML quoting predicate).  The CDI emitter is ONE kernel: a CTA takes a tile
// of 128 devices, computes the fragment lengths, scans them, gets the tile's output offset by a
// decoupled look-back over the tile aggregates (scan.cuh), builds the tile's bytes in shared memory
// (one warp per device, literal segments copied from a shared-memory pool) at the same 16-byte
// phase as their destination, and writes the tile with ONE TMA bulk store (cp.async.bulk
// shared -> global) plus at most 15 head / tail bytes.  Document header and tail belong to the first
// and the last tile.  Allocate names and ListAndWatch bytes (<= 24 B per item) are length -> single-
// pass scan -> thread-per-item write.
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "cdi.cuh"
#include "common.cuh"
#include "mdev.cuh"
#include "scan.cuh"

namespace kxemit {

constexpr int TILE = 128;      // devices per CTA
constexpr int EMIT_THREADS = 256;
constexpr int MAX_FRAG = 368;  // upper bound of one fragment: literals (<= 267 + kind) + 2 x 20 + 2 x 10 + 15 + 2 + slack; with the
                               // rest of TileSmem this keeps a CTA under 56.7 KB: four CTAs per SM, the 512 tiles of cfg5 are ONE
                               // wave.  Holds every kind up to 22 bytes.
constexpr int MAX_FRAG_LONG = 416;  // kinds of 23..63 bytes: 62.7 KB per CTA, three CTAs per SM
constexpr int MAX_FRAG_MDEV = 480;  // kxpu_cdi_emit_mdev, every kind: the PCI bound + the mdev annotation (<= 20 + 36 bytes);
                                    // 69.8 KB per CTA, three CTAs per SM
// kxpu_cdi_emit_cdev: the node literal is "devices/vfio" longer, and N takes the place of the group's second copy (both
// at most 10 digits), so every fragment bound grows by exactly that literal and the kind split stays at 22 bytes
#define KX_CDEV_NODE "devices/vfio"
constexpr int CDEV_EXTRA = sizeof(KX_CDEV_NODE) - 1;
constexpr int MAX_FRAG_CDEV = MAX_FRAG + CDEV_EXTRA;
constexpr int MAX_FRAG_CDEV_LONG = MAX_FRAG_LONG + CDEV_EXTRA;
// kxpu_cdi_emit_mdev_cdev: the same for the mdev bound; 71.3 KB per CTA, still three CTAs per SM
constexpr int MAX_FRAG_MDEV_CDEV = MAX_FRAG_MDEV + CDEV_EXTRA;
constexpr int LAYOUT_PCI = KX_CDI_PCI, LAYOUT_MDEV = KX_CDI_MDEV, LAYOUT_CDEV = KX_CDI_CDEV,
              LAYOUT_MDEV_CDEV = KX_CDI_MDEV_CDEV, LAYOUT_TYPED = KX_CDI_TYPED, LAYOUT_TYPED_CDEV = KX_CDI_TYPED_CDEV;
// kxpu_cdi_emit_vf_vgpu[_cdev]: two more annotations, vgpu-type: "<id>" and vgpu-type-key: "<key>".  The fragment grows
// by the JSON literals (the YAML ones are shorter), a 10-digit ID and a 40-byte key, for every kind, so the kind split
// stays at 22 bytes
#define KX_YV4 "\n      vgpu-type: \""
#define KX_YV9 "\"\n      vgpu-type-key: \""
#define KX_JV4 "\",\n        \"vgpu-type\": \""
#define KX_JV9 "\",\n        \"vgpu-type-key\": \""
constexpr int TYPED_EXTRA = (int)sizeof(KX_JV4 KX_JV9) - 1 + 10 + 40;  // 104
static_assert(sizeof(KX_YV4 KX_YV9 "\"") <= sizeof(KX_JV4 KX_JV9), "the YAML annotations must not outgrow the JSON ones");
constexpr int MAX_FRAG_TYPED = MAX_FRAG + TYPED_EXTRA, MAX_FRAG_TYPED_LONG = MAX_FRAG_LONG + TYPED_EXTRA;
constexpr int MAX_FRAG_TYPED_CDEV = MAX_FRAG_CDEV + TYPED_EXTRA, MAX_FRAG_TYPED_CDEV_LONG = MAX_FRAG_CDEV_LONG + TYPED_EXTRA;
static_assert(MAX_FRAG_MDEV <= KX_CDI_FRAG_MAX && MAX_FRAG_CDEV_LONG <= KX_CDI_FRAG_MAX, "the parse halo must follow");
static_assert(MAX_FRAG_MDEV_CDEV <= KX_CDI_FRAG_MAX_MDEV_CDEV, "the mdev cdev parse halo must follow");
static_assert(MAX_FRAG_TYPED_LONG <= KX_CDI_FRAG_MAX_TYPED && MAX_FRAG_TYPED_CDEV_LONG <= KX_CDI_FRAG_MAX_TYPED,
              "the typed parse halo must follow");
// the records of the two mdev layouts: kxpu_mdevcdev starts with the kxpu_mdevcdi the group layout reads
template <int LAYOUT> constexpr bool is_mdev_layout = LAYOUT == LAYOUT_MDEV || LAYOUT == LAYOUT_MDEV_CDEV;
template <int LAYOUT> constexpr bool is_typed_layout = LAYOUT == LAYOUT_TYPED || LAYOUT == LAYOUT_TYPED_CDEV;
template <int LAYOUT>
constexpr bool is_cdev_layout = LAYOUT == LAYOUT_CDEV || LAYOUT == LAYOUT_MDEV_CDEV || LAYOUT == LAYOUT_TYPED_CDEV;
template <int LAYOUT> using MdevRec = std::conditional_t<LAYOUT == LAYOUT_MDEV_CDEV, kxpu_mdevcdev, kxpu_mdevcdi>;
// the records of the PCI layouts: kxpu_vfvgpucdi starts with the kxpu_cdidev the untyped layouts read
template <int LAYOUT> using PciRec = std::conditional_t<is_typed_layout<LAYOUT>, kxpu_vfvgpucdi, kxpu_cdidev>;
constexpr int POOL_MAX = 640;
constexpr int KIND_MAX = 63;

// ------------------------------------------------------------------ templates
// YAML (yaml.v3, indent 2) and JSON (MarshalIndent "  ") literals between the variable
// fields: see SURVEY.md 8a-fmt for the derivation.  The CDI kind (CdiVendorClass, "nvidia.com/gpu" in the
// reference, generic_device_plugin.go:31) is a runtime argument: literal 3 and the document head are
// <before> kind <after>, assembled on the host into the pool the kernel receives as a parameter.
// KX_*A / KX_*B: the text before / after the kind
#define KX_Y0 "  - name: \""
#define KX_Y1 "\"\n    annotations:\n      attach-pci: \"true\"\n      bdf: "
#define KX_Y2 "\n      cdi.k8s.io/vfio"
#define KX_Y3A ": "
#define KX_Y3B "="
#define KX_Y4 "\n    containerEdits:\n      deviceNodes:\n        - path: /dev/vfio/"
#define KX_Y5 "\n"
#define KX_YHA "cdiVersion: 0.6.0\nkind: "
#define KX_YHB "\ndevices:\n"
#define KX_YT ""
#define KX_YEB "\ndevices: []\n"
#define KX_J0 "    {\n      \"name\": \""
#define KX_J1 "\",\n      \"annotations\": {\n        \"attach-pci\": \"true\",\n        \"bdf\": \""
#define KX_J2 "\",\n        \"cdi.k8s.io/vfio"
#define KX_J3A "\": \""
#define KX_J3B "="
#define KX_J4 "\"\n      },\n      \"containerEdits\": {\n        \"deviceNodes\": [\n          {\n            \"path\": \"/dev/vfio/"
#define KX_J5 "\"\n          }\n        ]\n      }\n    }"
#define KX_JHA "{\n  \"cdiVersion\": \"0.6.0\",\n  \"kind\": \""
#define KX_JHB "\",\n  \"devices\": [\n"
#define KX_JT "  ],\n  \"containerEdits\": {}\n}"
#define KX_JEB "\",\n  \"devices\": null,\n  \"containerEdits\": {}\n}"
// kxpu_cdi_emit_mdev: after "kind=<index>" comes the mdev annotation (literal 4 below, then the uuid) and literal 9,
// which is the PCI literal 4
#define KX_YM "\n      mdev: "
#define KX_JM "\",\n        \"mdev\": \""
// part k = before[k] (+ kind + after[k] when after[k] != NULL); parts 0-5 are the literals, 6 the document head,
// 7 the tail, 8 the whole document for zero devices (Devices stays nil, cdi/spec.go:42-49), 9 the literal after the
// mdev uuid or the type ID, 10 the literal after the type key (NULL: none)
struct Parts { const char *before[11], *after[11]; };
static const Parts h_yaml_parts = {{KX_Y0, KX_Y1, KX_Y2, KX_Y3A, KX_Y4, KX_Y5, KX_YHA, KX_YT, KX_YHA, nullptr},
                                   {nullptr, nullptr, nullptr, KX_Y3B, nullptr, nullptr, KX_YHB, nullptr, KX_YEB, nullptr}};
static const Parts h_json_parts = {{KX_J0, KX_J1, KX_J2, KX_J3A, KX_J4, KX_J5, KX_JHA, KX_JT, KX_JHA, nullptr},
                                   {nullptr, nullptr, nullptr, KX_J3B, nullptr, nullptr, KX_JHB, nullptr, KX_JEB, nullptr}};
static const Parts h_yaml_mdev_parts = {{KX_Y0, KX_Y1, KX_Y2, KX_Y3A, KX_YM, KX_Y5, KX_YHA, KX_YT, KX_YHA, KX_Y4},
                                        {nullptr, nullptr, nullptr, KX_Y3B, nullptr, nullptr, KX_YHB, nullptr, KX_YEB, nullptr}};
static const Parts h_json_mdev_parts = {{KX_J0, KX_J1, KX_J2, KX_J3A, KX_JM, KX_J5, KX_JHA, KX_JT, KX_JHA, KX_J4},
                                        {nullptr, nullptr, nullptr, KX_J3B, nullptr, nullptr, KX_JHB, nullptr, KX_JEB, nullptr}};
static const Parts h_yaml_cdev_parts = {{KX_Y0, KX_Y1, KX_Y2, KX_Y3A, KX_Y4 KX_CDEV_NODE, KX_Y5, KX_YHA, KX_YT, KX_YHA, nullptr},
                                        {nullptr, nullptr, nullptr, KX_Y3B, nullptr, nullptr, KX_YHB, nullptr, KX_YEB, nullptr}};
static const Parts h_json_cdev_parts = {{KX_J0, KX_J1, KX_J2, KX_J3A, KX_J4 KX_CDEV_NODE, KX_J5, KX_JHA, KX_JT, KX_JHA, nullptr},
                                        {nullptr, nullptr, nullptr, KX_J3B, nullptr, nullptr, KX_JHB, nullptr, KX_JEB, nullptr}};
static const Parts h_yaml_mdev_cdev_parts = {{KX_Y0, KX_Y1, KX_Y2, KX_Y3A, KX_YM, KX_Y5, KX_YHA, KX_YT, KX_YHA, KX_Y4 KX_CDEV_NODE},
                                             {nullptr, nullptr, nullptr, KX_Y3B, nullptr, nullptr, KX_YHB, nullptr, KX_YEB, nullptr}};
static const Parts h_json_mdev_cdev_parts = {{KX_J0, KX_J1, KX_J2, KX_J3A, KX_JM, KX_J5, KX_JHA, KX_JT, KX_JHA, KX_J4 KX_CDEV_NODE},
                                             {nullptr, nullptr, nullptr, KX_J3B, nullptr, nullptr, KX_JHB, nullptr, KX_JEB, nullptr}};
// the typed layouts: literal 4 opens vgpu-type, 9 sits between the ID and the key, 10 closes the key and is the PCI
// literal 4 (typed cdev: with the node literal)
static const Parts h_yaml_typed_parts = {{KX_Y0, KX_Y1, KX_Y2, KX_Y3A, KX_YV4, KX_Y5, KX_YHA, KX_YT, KX_YHA, KX_YV9, "\"" KX_Y4},
                                         {nullptr, nullptr, nullptr, KX_Y3B, nullptr, nullptr, KX_YHB, nullptr, KX_YEB, nullptr, nullptr}};
static const Parts h_json_typed_parts = {{KX_J0, KX_J1, KX_J2, KX_J3A, KX_JV4, KX_J5, KX_JHA, KX_JT, KX_JHA, KX_JV9, KX_J4},
                                         {nullptr, nullptr, nullptr, KX_J3B, nullptr, nullptr, KX_JHB, nullptr, KX_JEB, nullptr, nullptr}};
static const Parts h_yaml_typed_cdev_parts = {{KX_Y0, KX_Y1, KX_Y2, KX_Y3A, KX_YV4, KX_Y5, KX_YHA, KX_YT, KX_YHA, KX_YV9,
                                               "\"" KX_Y4 KX_CDEV_NODE},
                                              {nullptr, nullptr, nullptr, KX_Y3B, nullptr, nullptr, KX_YHB, nullptr, KX_YEB, nullptr, nullptr}};
static const Parts h_json_typed_cdev_parts = {{KX_J0, KX_J1, KX_J2, KX_J3A, KX_JV4, KX_J5, KX_JHA, KX_JT, KX_JHA, KX_JV9,
                                               KX_J4 KX_CDEV_NODE},
                                              {nullptr, nullptr, nullptr, KX_J3B, nullptr, nullptr, KX_JHB, nullptr, KX_JEB, nullptr, nullptr}};
static const char *kDefaultKind = "nvidia.com/gpu";  // CdiVendorClass, generic_device_plugin.go:31

// The supported kind domain (include/kxpu.h): "vendor/class", <= 63 bytes; vendor = letter [A-Za-z0-9_.-]*
// alnum, class = letter [A-Za-z0-9_-]* alnum (a subset of CDI v0.8.0 pkg/parser's vendor / class rules).
static bool kind_ok(const char *kind) {
    if (!kind) return false;
    const size_t len = strnlen(kind, KIND_MAX + 1);
    if (len > (size_t)KIND_MAX) return false;
    const char *slash = (const char *)memchr(kind, '/', len);
    if (!slash) return false;
    auto alpha = [](char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); };
    auto alnum = [&](char c) { return alpha(c) || (c >= '0' && c <= '9'); };
    auto part = [&](const char *s, size_t l, bool dots) {
        if (l == 0 || !alpha(s[0]) || !alnum(s[l - 1])) return false;
        for (size_t k = 0; k < l; k++)
            if (!(alnum(s[k]) || s[k] == '_' || s[k] == '-' || (dots && s[k] == '.'))) return false;
        return true;
    };
    const size_t vl = (size_t)(slash - kind);
    return part(kind, vl, true) && part(slash + 1, len - vl - 1, false);
}

static std::string part_text(const Parts &P, int k, const char *kind) {
    std::string s = P.before[k] ? P.before[k] : "";
    if (P.after[k]) { s += kind; s += P.after[k]; }
    return s;
}

__device__ __forceinline__ uint32_t dec_len(unsigned long long v) {
    uint32_t l = 1;
    while (v >= 10ull) { v /= 10ull; l++; }
    return l;
}
__device__ __forceinline__ void dec_write(unsigned long long v, uint32_t len, uint8_t *dst) {
    for (uint32_t k = len; k > 0; k--) { dst[k - 1] = (uint8_t)('0' + (uint32_t)(v % 10ull)); v /= 10ull; }
}
__device__ __forceinline__ uint32_t bdf_len16(const uint8_t *b) {
    uint32_t l = 0;
    while (l < 16u && b[l]) l++;
    return l;
}
// yaml.v3 isBase60Float: ^[-+]?[0-9][0-9_]*(?::[0-5]?[0-9])+(?:\.[0-9_]*)?$  (resolve.go);
// such a string would be read back as a sexagesimal number, so encode.go quotes it.
__device__ __forceinline__ bool is_base60(const uint8_t *s, uint32_t len) {
    uint32_t i = 0;
    auto dig = [](uint8_t c) { return c >= '0' && c <= '9'; };
    if (i < len && (s[i] == '-' || s[i] == '+')) i++;
    if (!(i < len && dig(s[i]))) return false;
    i++;
    while (i < len && (dig(s[i]) || s[i] == '_')) i++;
    uint32_t groups = 0;
    while (i < len && s[i] == ':') {
        uint32_t j = i + 1;
        if (!(j < len && dig(s[j]))) break;
        if (j + 1 < len && dig(s[j + 1])) j += s[j] <= '5' ? 2u : 1u;
        else j += 1;
        i = j; groups++;
    }
    if (!groups) return false;
    if (i < len && s[i] == '.') { i++; while (i < len && (dig(s[i]) || s[i] == '_')) i++; }
    return i == len;
}
// bytes Go's encoders would escape or that change YAML plain-scalar rules are outside the
// supported domain; PCI addresses only use [0-9a-f:.]
__device__ __forceinline__ bool bdf_charset_ok(const uint8_t *s, uint32_t len) {
    if (len == 0) return false;
    for (uint32_t i = 0; i < len; i++) {
        uint8_t c = s[i];
        if (!((c >= '0' && c <= '9') || (c >= 'a' && c <= 'f') || c == ':' || c == '.')) return false;
    }
    return true;
}
// a bdf over [0-9a-f:.] that yaml.v3 writes as a plain string, or as the double-quoted base-60 form above (include/kxpu.h
// states the classes and why): not all digits, not 0b + binary digits, not a float of resolve.go's yamlStyleFloat
// ([0-9]+(\.[0-9]*)?(e[0-9]+)? or \.[0-9]+(e[0-9]+)?), no trailing ':' and no leading "..."
__device__ __forceinline__ bool bdf_yaml_plain(const uint8_t *s, uint32_t len) {
    auto dig = [](uint8_t c) { return c >= '0' && c <= '9'; };
    if (len == 0 || s[len - 1] == ':') return false;
    if (len >= 3 && s[0] == '.' && s[1] == '.' && s[2] == '.') return false;
    if (len >= 3 && s[0] == '0' && s[1] == 'b') {
        uint32_t i = 2;
        while (i < len && (s[i] == '0' || s[i] == '1')) i++;
        if (i == len) return false;
    }
    uint32_t i = 0, m = 0;  // m: mantissa digits
    while (i < len && dig(s[i])) { i++; m++; }
    if (i < len && s[i] == '.') {
        const bool lead = m == 0;
        i++;
        while (i < len && dig(s[i])) { i++; m++; }
        if (lead && m == 0) return true;  // "." alone or "." followed by no digit
    }
    if (m == 0) return true;
    if (i < len && s[i] == 'e') {
        const uint32_t e0 = ++i;
        while (i < len && dig(s[i])) i++;
        if (i == e0) return true;
    }
    return i != len;
}

// The store epilogue of a staged tile: stg[0, total) sits in shared memory at g's 16-byte phase and goes to g with one
// bulk store for the 16-byte aligned body and byte stores for the ragged ends.  Called by every thread of a CTA of at
// least 80 threads, after the staging writes.
__device__ __forceinline__ void tile_store(uint8_t *g, const uint8_t *stg, uint32_t total) {
    const uint32_t tid = threadIdx.x;
    // generic-proxy writes to shared memory must be visible to the async proxy (TMA) that reads them
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(g) & 15u);
    const uint32_t lead = total < 16u ? total : ((16u - mis) & 15u);
    const uint32_t body = (total - lead) & ~15u;
    if (tid == 0 && body) {
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g + lead),
                     "r"((uint32_t)__cvta_generic_to_shared(stg + lead)), "r"(body)
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    if (tid >= 32 && tid < 32 + lead) g[tid - 32] = stg[tid - 32];
    const uint32_t rest = total - lead - body;
    if (tid >= 64 && tid < 64 + rest) g[lead + body + tid - 64] = stg[lead + body + tid - 64];
    if (tid == 0 && body) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // smem must outlive the read
}

struct EmitParams {
    const void *devs;         // kxpu_cdidev[n] or kxpu_mdevcdi[n]
    uint32_t n;
    uint16_t off[9], len[9];  // literal k / head (6) / tail (7) / the literal after the mdev uuid (8) inside the pool
    uint32_t pool_len, lit_total;
    uint8_t *out;
    unsigned long long *state;  // tile status words (scan.cuh look-back)
    uint32_t epoch;
    unsigned long long *total_out;
    uint32_t *flags;          // [0]: a bdf outside [0-9a-f:.], [1]: a uuid outside the canonical form
    uint8_t pool[POOL_MAX];   // literals | head | tail, built on the host for the call's kind
    uint16_t off10, len10;    // the typed layouts: the literal after the type key inside the pool
};

template <int MAXF>
struct TileSmem {
    alignas(16) uint8_t stage[TILE * MAXF + 512];
    uint8_t pool[POOL_MAX];
    uint8_t idx[TILE][20], grp[TILE][12], bdf[TILE][16];
    uint32_t meta[TILE];    // il | gl << 8 | bl << 16 | quoted << 24
    uint32_t start[TILE];   // fragment offset inside the tile
    unsigned long long base;
    uint32_t wsum[EMIT_THREADS / 32];
    uint32_t tile_total;
};
// the typed layouts: the type ID's digits and the key's length, appended so that the untyped tiles keep their layout
template <int MAXF>
struct TileSmemTyped : TileSmem<MAXF> {
    uint8_t tdec[TILE][12];  // type ID digits at 0, their count at 10, the key length at 11
};
template <int MAXF, int LAYOUT> using EmitSmem = std::conditional_t<is_typed_layout<LAYOUT>, TileSmemTyped<MAXF>, TileSmem<MAXF>>;
// four CTAs per SM (228 KB of shared memory, 1 KB of it reserved per CTA) for the short-kind tiles of both node layouts
static_assert(4 * (sizeof(TileSmem<MAX_FRAG_CDEV>) + 1024) <= 228 * 1024, "the cdev short-kind tile lost an SM slot");
// three CTAs per SM for the tiles of both mdev layouts
static_assert(3 * (sizeof(TileSmem<MAX_FRAG_MDEV_CDEV>) + 1024) <= 228 * 1024, "the mdev cdev tile lost an SM slot");
// the typed layouts: three CTAs per SM for kinds up to 22 bytes, two for longer ones
static_assert(3 * (sizeof(TileSmemTyped<MAX_FRAG_TYPED_CDEV>) + 1024) <= 228 * 1024, "the typed short-kind tile lost an SM slot");
static_assert(2 * (sizeof(TileSmemTyped<MAX_FRAG_TYPED_CDEV_LONG>) + 1024) <= 228 * 1024, "the typed long-kind tile lost an SM slot");

// a type key byte: [A-Za-z0-9_.-]; the first kl of the 40 key bytes in k must all be one
__device__ __forceinline__ bool type_key_ok(const uint32_t (&k)[10], uint32_t kl) {
    bool good = true;
#pragma unroll
    for (int b = 0; b < 40; b++) {
        const uint32_t c = (k[b >> 2] >> (8 * (b & 3))) & 0xffu;
        const bool ok = (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '_' || c == '.' ||
                        c == '-';
        if ((uint32_t)b < kl && !ok) good = false;
    }
    return good;
}

template <int FMT, int MAXF, int LAYOUT>
__global__ void __launch_bounds__(EMIT_THREADS) k_cdi_fused(const __grid_constant__ EmitParams E) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    EmitSmem<MAXF, LAYOUT> &S = *reinterpret_cast<EmitSmem<MAXF, LAYOUT> *>(smem_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    const uint32_t tile = blockIdx.x, i0 = tile * TILE;
    const bool first_tile = tile == 0, last_tile = tile == gridDim.x - 1;
    for (uint32_t k = tid; k < E.pool_len; k += EMIT_THREADS) S.pool[k] = E.pool[k];

    // ---- fragment lengths and variable fields: one thread per device
    uint32_t flen = 0;
    if (tid < TILE && i0 + tid < E.n) {
        uint4 bq;  // the bdf / parent address
        uint32_t group, node = 0;
        unsigned long long index;
        uint32_t typed_len = 0;  // the typed layouts: the type ID's digits and the key
        if (!is_mdev_layout<LAYOUT>) {  // bdf[16] | iommu_group | vfio_cdev | index
            const uint4 *p = reinterpret_cast<const uint4 *>(static_cast<const PciRec<LAYOUT> *>(E.devs) + i0 + tid);
            const uint4 q0 = p[0], q1 = p[1];
            bq = q0;
            group = q1.x;
            if constexpr (LAYOUT == LAYOUT_CDEV || LAYOUT == LAYOUT_TYPED_CDEV) node = q1.y;
            index = ((unsigned long long)q1.w << 32) | q1.z;
            if constexpr (is_typed_layout<LAYOUT>) {  // then type_id | key_len | reserved[3] | key[40]
                const uint4 q2 = p[2], q3 = p[3], q4 = p[4];
                const uint32_t key[10] = {q2.z, q2.w, q3.x, q3.y, q3.z, q3.w, q4.x, q4.y, q4.z, q4.w};
                const uint32_t type_id = q2.x, kl_raw = q2.y & 0xffu;
                const uint32_t kl = kl_raw <= 40u ? kl_raw : 40u;  // out of the domain: reported, and bounded here
                if (type_id == 0u || kl_raw == 0u || kl_raw > 40u || !type_key_ok(key, kl)) E.flags[1] = 1u;
                const uint32_t tl = dec_len(type_id);
                dec_write(type_id, tl, S.tdec[tid]);
                S.tdec[tid][10] = (uint8_t)tl;
                S.tdec[tid][11] = (uint8_t)kl;
                typed_len = tl + kl;
            }
        } else {  // uuid[36] | iommu_group | parent[16] | index (mdev cdev: the first 64 of 80 bytes; N is read below)
            const uint4 *p = reinterpret_cast<const uint4 *>(static_cast<const MdevRec<LAYOUT> *>(E.devs) + i0 + tid);
            const uint4 q0 = p[0], q1 = p[1], q2 = p[2], q3 = p[3];
            const uint32_t uw[9] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x};
            if (!kxmdev::uuid_ok(uw)) E.flags[1] = 1u;
            bq = make_uint4(q2.z, q2.w, q3.x, q3.y);
            group = q2.y;
            index = ((unsigned long long)q3.w << 32) | q3.z;
        }
        const uint8_t *bdf = reinterpret_cast<const uint8_t *>(&bq);
        const uint32_t bl = bdf_len16(bdf), il = dec_len(index), gl = dec_len(group);
        if (!bdf_charset_ok(bdf, bl) || !bdf_yaml_plain(bdf, bl)) E.flags[0] = 1u;
        const bool quoted = FMT == KXPU_FMT_YAML && is_base60(bdf, bl);
        dec_write(index, il, S.idx[tid]);
        dec_write(group, gl, S.grp[tid]);
        *reinterpret_cast<uint4 *>(S.bdf[tid]) = bq;
        S.meta[tid] = il | (gl << 8) | (bl << 16) | ((quoted ? 1u : 0u) << 24);
        flen = E.lit_total + 2u * il + 2u * gl + bl + (quoted ? 2u : 0u) + (is_mdev_layout<LAYOUT> ? 36u : 0u);
        if constexpr (LAYOUT == LAYOUT_MDEV_CDEV) node = static_cast<const kxpu_mdevcdev *>(E.devs)[i0 + tid].vfio_cdev;
        if constexpr (is_cdev_layout<LAYOUT>) {  // N in place of the group's second copy; its length in grp's spare byte 11
            uint32_t nl = 1;
            for (uint32_t p = 10u; nl < 10u && node >= p; p *= 10u) nl++;
            S.grp[tid][11] = (uint8_t)nl;
            flen = flen - gl + nl;
        }
        if constexpr (is_typed_layout<LAYOUT>) flen += typed_len;
        if (FMT == KXPU_FMT_JSON) flen += (i0 + tid + 1u < E.n) ? 2u : 1u;  // ",\n" between devices, "\n" after the last
    }
    // ---- scan of the 128 lengths (threads >= TILE contribute 0)
    uint32_t incl = kxscan::warp_incl(flen);
    if (lane == 31) S.wsum[w] = incl;
    __syncthreads();
    if (w == 0) {
        const uint32_t x = lane < EMIT_THREADS / 32 ? S.wsum[lane] : 0u;
        const uint32_t xi = kxscan::warp_incl(x);
        if (lane < EMIT_THREADS / 32) S.wsum[lane] = xi - x;
        if (lane == EMIT_THREADS / 32 - 1) S.tile_total = xi;
    }
    __syncthreads();
    const uint32_t head_len = first_tile ? E.len[6] : 0u, tail_len = last_tile ? E.len[7] : 0u;
    const uint32_t tile_total = S.tile_total;
    if (tid < TILE) S.start[tid] = head_len + S.wsum[w] + incl - flen;
    // ---- the tile's offset in the document: decoupled look-back over the tile aggregates
    if (w == 0) {
        const unsigned long long agg = (unsigned long long)head_len + tile_total + tail_len;
        const unsigned long long excl = kxscan::lookback(E.state, tile, agg, E.epoch);
        if (lane == 0) {
            S.base = excl;
            if (last_tile) *E.total_out = excl + agg;
        }
    }
    __syncthreads();
    const unsigned long long base = S.base;
    const uint32_t mis = (uint32_t)((reinterpret_cast<uintptr_t>(E.out) + base) & 15u);  // same 16-byte phase in smem and global
    uint8_t *stg = S.stage + mis;
    if (first_tile) for (uint32_t k = tid; k < head_len; k += EMIT_THREADS) stg[k] = S.pool[E.off[6] + k];
    if (last_tile) for (uint32_t k = tid; k < tail_len; k += EMIT_THREADS) stg[head_len + tile_total + k] = S.pool[E.off[7] + k];
    // ---- fragments: one warp per device, segment by segment
    uint32_t cdev_n = 0;  // cdev: lane j holds N of the warp's j-th device, read from the device array (L2) ahead of the loop
    if constexpr (is_cdev_layout<LAYOUT>) {
        const uint32_t dj = w + lane * (EMIT_THREADS / 32);
        if (dj < (uint32_t)TILE && i0 + dj < E.n) {
            if constexpr (LAYOUT == LAYOUT_CDEV) cdev_n = static_cast<const kxpu_cdidev *>(E.devs)[i0 + dj].vfio_cdev;
            else if constexpr (LAYOUT == LAYOUT_TYPED_CDEV) cdev_n = static_cast<const kxpu_vfvgpucdi *>(E.devs)[i0 + dj].dev.vfio_cdev;
            else cdev_n = static_cast<const kxpu_mdevcdev *>(E.devs)[i0 + dj].vfio_cdev;
        }
    }
    for (uint32_t d = w; d < (uint32_t)TILE && i0 + d < E.n; d += EMIT_THREADS / 32) {
        const uint32_t m = S.meta[d];
        const uint32_t il = m & 0xffu, gl = (m >> 8) & 0xffu, bl = (m >> 16) & 0xffu;
        const bool quoted = (m >> 24) != 0u;
        uint8_t *dst = stg + S.start[d];
        uint32_t o = 0;
        auto lit = [&](int k) {
            const uint32_t L = E.len[k];
            const uint8_t *src = S.pool + E.off[k];
            for (uint32_t l = lane; l < L; l += 32u) dst[o + l] = src[l];
            o += L;
        };
        auto var = [&](const uint8_t *src, uint32_t L) {  // L <= 20
            if (lane < L) dst[o + lane] = src[lane];
            o += L;
        };
        auto quote = [&]() {
            if (FMT == KXPU_FMT_YAML && quoted) { if (lane == 0) dst[o] = (uint8_t)'"'; o += 1u; }
        };
        lit(0); var(S.idx[d], il); lit(1); quote(); var(S.bdf[d], bl); quote(); lit(2); var(S.grp[d], gl);
        lit(3); var(S.idx[d], il); lit(4);
        if constexpr (is_typed_layout<LAYOUT>) {  // the type ID, literal 9, the key straight from the device array (L2),
                                                  // literal 10 (the node literal)
            var(S.tdec[d], S.tdec[d][10]);
            lit(8);
            const uint32_t kl = S.tdec[d][11];
            const uint8_t *k = reinterpret_cast<const uint8_t *>(static_cast<const kxpu_vfvgpucdi *>(E.devs)[i0 + d].key);
            for (uint32_t l = lane; l < kl; l += 32u) dst[o + l] = k[l];
            o += kl;
            for (uint32_t l = lane; l < E.len10; l += 32u) dst[o + l] = S.pool[E.off10 + l];
            o += E.len10;
        }
        if (is_mdev_layout<LAYOUT>) {  // the uuid straight from the device array (L2), then the PCI literal 4 (mdev cdev:
                                       // with the node literal)
            const uint8_t *u = static_cast<const uint8_t *>(E.devs) + (size_t)(i0 + d) * sizeof(MdevRec<LAYOUT>);
            for (uint32_t l = lane; l < 36u; l += 32u) dst[o + l] = u[l];
            o += 36u;
            lit(8);
        }
        if constexpr (is_cdev_layout<LAYOUT>) {  // lane k writes digit k of N
            const uint32_t N = __shfl_sync(0xffffffffu, cdev_n, d / (EMIT_THREADS / 32));
            const uint32_t nl = S.grp[d][11];
            if (lane < nl) {
                uint32_t v = N;
                for (uint32_t k = lane + 1u; k < nl; k++) v /= 10u;
                dst[o + lane] = (uint8_t)('0' + v % 10u);
            }
            o += nl;
        } else {
            var(S.grp[d], gl);
        }
        lit(5);
        if (FMT == KXPU_FMT_JSON) {
            const bool more = i0 + d + 1u < E.n;
            if (lane == 0) { if (more) { dst[o] = (uint8_t)','; dst[o + 1] = (uint8_t)'\n'; } else dst[o] = (uint8_t)'\n'; }
        }
    }
    tile_store(E.out + base, stg, head_len + tile_total + tail_len);
}

// ------------------------------------------------------------------ K11: DRA ResourceSlices (kxpu_dra_slices[_mdev])
// One CTA per slice of TILE devices; k_dra_slices<LAYOUT> reads kxpu_dradev (LAYOUT_PCI) or kxpu_dramdev (LAYOUT_MDEV)
// records.  A PCI device fragment is literal D0, the variable fields and literals D1..D8 (D3 / D5 / D6 with their field
// only when present), then ',' unless it is the slice's last device.  Every literal but D0 opens with the closing bytes
// of the value before it, so an absent optional attribute simply drops its literal and field.
#define KX_D0 "{\"name\":\"vfio"
#define KX_D1 "\",\"attributes\":{\"deviceID\":{\"string\":\""
#define KX_D2 "\"},\"iommuGroup\":{\"int\":"
#define KX_D3 "},\"numaNode\":{\"int\":"
#define KX_D4 "},\"pciAddress\":{\"string\":\""
#define KX_D5 "\"},\"productName\":{\"string\":\""
#define KX_D6 "\"},\"resource.kubernetes.io/pcieRoot\":{\"string\":\""
#define KX_D7 "\"},\"vendorID\":{\"string\":\""
#define KX_D8 "\"}}}"
#define KX_DRA_TAIL "]}}\n"
static const char *const h_dra_lits[9] = {KX_D0, KX_D1, KX_D2, KX_D3, KX_D4, KX_D5, KX_D6, KX_D7, KX_D8};
constexpr uint32_t DRA_LIT_TOTAL = sizeof(KX_D0 KX_D1 KX_D2 KX_D3 KX_D4 KX_D5 KX_D6 KX_D7 KX_D8) - 1;
// the longest fragment: every literal, a 10-digit group twice, node 63, a 16-byte bdf and root, 64 product bytes, two
// 6-byte ids, the separator
constexpr int MAX_FRAG_DRA = (int)DRA_LIT_TOTAL + 2 * 10 + 2 + 16 + 16 + 64 + 6 + 6 + 1;
// literals | slice head | slice tail: the head holds the node name twice, the driver twice and the pool once
// (2 * 253 + 2 * 63 + 253 bytes of names, about 1.1 KB in all)
constexpr int DRA_POOL_MAX = 1536;
constexpr int DRA_PARTS = 11;  // nine literals, the slice head, the slice tail

// An mdev device fragment: literal M0, the group, M1, the group and its closer; then for each attribute in key order its
// opening literal (M2..M9), its value and the value's own closer (MS after a string, MI after an int); then ME and the
// separator.  A value is never closed by the next attribute's literal: numaNode is an int between two strings, so an
// absent attribute drops its opening literal, value and closer, and nothing else changes.
#define KX_M0 "{\"name\":\"vfio"
#define KX_M1 "\",\"attributes\":{\"iommuGroup\":{\"int\":"
#define KX_M2 ",\"mdevType\":{\"string\":\""
#define KX_M3 ",\"numaNode\":{\"int\":"
#define KX_M4 ",\"parentAddress\":{\"string\":\""
#define KX_M5 ",\"parentDeviceID\":{\"string\":\""
#define KX_M6 ",\"parentVendorID\":{\"string\":\""
#define KX_M7 ",\"productName\":{\"string\":\""
#define KX_M8 ",\"resource.kubernetes.io/pcieRoot\":{\"string\":\""
#define KX_M9 ",\"uuid\":{\"string\":\""
#define KX_MS "\"}"
#define KX_MI "}"
#define KX_ME "}}"
constexpr int DRAM_S = 10, DRAM_I = 11, DRAM_E = 12, DRAM_LITS = 13;
static const char *const h_dram_lits[DRAM_LITS] = {KX_M0, KX_M1, KX_M2, KX_M3, KX_M4, KX_M5, KX_M6,
                                                   KX_M7, KX_M8, KX_M9, KX_MS, KX_MI, KX_ME};
// the longest fragment: every literal, seven string closers, two int closers, a 10-digit group twice, a 40-byte type,
// node 63, a 16-byte parent and root, two 6-byte ids, 64 product bytes, the uuid, the separator
constexpr int MAX_FRAG_DRA_MDEV = (int)sizeof(KX_M0 KX_M1 KX_M2 KX_M3 KX_M4 KX_M5 KX_M6 KX_M7 KX_M8 KX_M9 KX_ME) - 1 +
                                  7 * ((int)sizeof(KX_MS) - 1) + 2 * ((int)sizeof(KX_MI) - 1) + 2 * 10 + 40 + 2 + 16 +
                                  16 + 6 + 6 + 64 + 36 + 1;
constexpr int DRAM_PARTS = DRAM_LITS + 2;

// Taints (kxpu_dra_slices[_mdev]_taint[s]).  A device that carries some taint ends with its last literal less that
// literal's final '}' (the one that closes the device), then KX_TAINTS_OPEN, for each carried taint in table order its
// entry head (the table's key, value and effect, assembled on the host like the slice head), the 20-byte timeAdded and
// KX_TAINT_ECLOSE, with ',' between entries, then KX_TAINTS_CLOSE.  Slices hold TAINT_TILE devices whether or not one
// is tainted.
#define KX_TAINTS_OPEN ",\"taints\":["
#define KX_TAINT_ECLOSE "\"}"
#define KX_TAINTS_CLOSE "]}"
constexpr int TAINT_TILE = 64;
constexpr long long TAINT_SINCE_MAX = 253402300799ll;  // 9999-12-31T23:59:59Z
constexpr int TAINT_ENTRY_MAX =  // {"key":"<key>","value":"<value>","effect":"<effect>","timeAdded":"  at the longest
    (int)sizeof("{\"key\":\"\",\"value\":\"\",\"effect\":\"\",\"timeAdded\":\"") - 1 + 127 + 63 + 10;
// what nt carried taints add to a fragment at most
constexpr int taints_part_max(int nt) {
    return (int)sizeof(KX_TAINTS_OPEN) - 1 + nt * (TAINT_ENTRY_MAX + 20 + (int)sizeof(KX_TAINT_ECLOSE) - 1 + 1) - 1 +
           (int)sizeof(KX_TAINTS_CLOSE) - 1 - 1;  // less one ',' and the '}' it replaces
}
// the pool of a table of up to nt entries: the untainted bound (its longest content is about 1.4 KB: the 1.1 KB head
// and the vGPU literals) plus room for KX_TAINTS_OPEN, nt entry heads, KX_TAINT_ECLOSE and KX_TAINTS_CLOSE: 272 bytes
// for the 261 of one entry, 1 KB for the 999 of four
constexpr int dra_pool_max(int nt) { return DRA_POOL_MAX + (nt == 0 ? 0 : nt == 1 ? 272 : 1024); }
constexpr int taints_pool_need(int nt) {
    return (int)sizeof(KX_TAINTS_OPEN KX_TAINT_ECLOSE KX_TAINTS_CLOSE) - 1 + nt * TAINT_ENTRY_MAX;
}

// PARTS = literals + head + tail; the head is part PARTS - 2, the tail PARTS - 1
template <int PARTS, int POOL>
struct DraParams {
    const void *devs;               // kxpu_dradev[n] or kxpu_dramdev[n]
    uint32_t n;
    uint16_t off[PARTS], len[PARTS];  // literal k / head / tail inside the pool
    uint32_t pool_len;
    uint8_t *out;
    unsigned long long *slice_off;  // [gridDim.x + 1]
    unsigned long long *state;      // slice status words (scan.cuh look-back)
    uint32_t epoch;
    uint32_t *flags;                // one word per KXPU_E_UNSUPPORTED reason, DRA_F_* / DRAM_F_*
    uint8_t pool[POOL];
};
// the tainted instantiations, for tables of up to NT entries: the literals, KX_TAINTS_OPEN (part PARTS - NT - 5), the
// entry heads (PARTS - NT - 4 .. PARTS - 5), KX_TAINT_ECLOSE, KX_TAINTS_CLOSE, the slice head and tail
template <int PARTS, int NT>
struct DraTaintsParams : DraParams<PARTS, dra_pool_max(NT)> {
    const long long *since;  // [n * nt], device-major: taint t of device i, < 0 = not carried
    uint32_t nt;             // table entries, 1..NT
    uint8_t dup[NT];         // dup[t]: the earlier entries with taint t's key and effect
};
constexpr int DRA_F_PRODUCT = 0, DRA_F_BDF = 1, DRA_F_ROOT = 2, DRA_F_VENDOR = 3, DRA_F_DEVICE = 4, DRA_F_GROUP = 5,
              DRA_F_PLEN = 6, DRA_F_COUNT = 7;
// the order of the header's domain list, which the oracle's `why` follows
constexpr int DRAM_F_PRODUCT = 0, DRAM_F_TYPE = 1, DRAM_F_UUID = 2, DRAM_F_PARENT = 3, DRAM_F_ROOT = 4, DRAM_F_VENDOR = 5,
              DRAM_F_DEVICE = 6, DRAM_F_GROUP = 7, DRAM_F_PLEN = 8, DRAM_F_COUNT = 9;

// T devices per slice, FRAG bytes per fragment, a POOL-byte pool
template <int T, int FRAG, int POOL>
struct DraSmem {
    alignas(16) uint8_t stage[T * FRAG + POOL + 16];
    uint8_t pool[POOL];
    uint8_t dec[T][12];  // group digits at 0, NUMA node digits at 10
    uint32_t meta[T];    // gl | nl << 4 | bl << 8 | rl << 13 | vl << 18 | dl << 21 | pl << 24
    uint32_t start[T];   // fragment offset inside the slice
    unsigned long long base;
    uint32_t wsum[EMIT_THREADS / 32];
    uint32_t tile_total;
};
template <int T, int FRAG, int POOL>
struct DraMdevSmem {
    alignas(16) uint8_t stage[T * FRAG + POOL + 16];
    uint8_t pool[POOL];
    uint8_t dec[T][12];  // group digits at 0, NUMA node digits at 10
    uint32_t meta[T];    // as DraSmem's, bl being the parent's length
    uint8_t tlen[T];     // mdev_type length
    uint32_t start[T];   // fragment offset inside the slice
    unsigned long long base;
    uint32_t wsum[EMIT_THREADS / 32];
    uint32_t tile_total;
};
template <typename Base, int NT>
struct DraTaintsSmem : Base {
    uint8_t ts[TAINT_TILE][NT][20];  // timeAdded of taint t of device d
    uint8_t carried[TAINT_TILE];     // bit t: device d carries taint t
};
template <int LAYOUT> struct DraLayout {  // LAYOUT_PCI
    using Rec = kxpu_dradev;
    template <int T, int FRAG, int POOL> using Smem = DraSmem<T, FRAG, POOL>;
    static constexpr int PARTS = DRA_PARTS, LAST = 8, F_COUNT = DRA_F_COUNT, MAX_FRAG = MAX_FRAG_DRA;
};
template <> struct DraLayout<LAYOUT_MDEV> {
    using Rec = kxpu_dramdev;
    template <int T, int FRAG, int POOL> using Smem = DraMdevSmem<T, FRAG, POOL>;
    static constexpr int PARTS = DRAM_PARTS, LAST = DRAM_E, F_COUNT = DRAM_F_COUNT, MAX_FRAG = MAX_FRAG_DRA_MDEV;
};
// one k_dra_slices instantiation for tables of up to NT taints (NT = 0: untainted): LAST is the literal that closes a
// device; a taint time above the maximum reports F_SINCE, a device with two taints of one key and effect F_DUP
template <int LAYOUT, int NT> struct DraKernel {
    using L = DraLayout<LAYOUT>;
    static constexpr bool TAINT = NT > 0;
    static constexpr int T = TAINT ? TAINT_TILE : TILE;
    static constexpr int PARTS = L::PARTS + (TAINT ? NT + 3 : 0);
    static constexpr int T_OPEN = L::PARTS - 2, T_ENTRY = T_OPEN + 1, T_ECLOSE = T_ENTRY + NT, T_CLOSE = T_ECLOSE + 1;
    static constexpr int F_SINCE = L::F_COUNT, F_DUP = F_SINCE + 1, F_COUNT = L::F_COUNT + (TAINT ? 2 : 0);
    static constexpr int POOL = dra_pool_max(NT);
    static_assert(!TAINT || taints_pool_need(NT) <= POOL - DRA_POOL_MAX, "taint pool bound");
    static constexpr int MAXF = L::MAX_FRAG + (TAINT ? taints_part_max(NT) : 0);
    // CTAs per SM asked of ptxas, 0 for none.  Left to itself ptxas gives NT = 1 96 registers (PCI) or 101 (vGPU), so
    // two CTAs per SM, where its 47 / 56 KB of shared memory allow four; asked for three it takes 48, without spills
    static constexpr int MIN_CTAS = NT == 1 ? 3 : 0;
    using Base = typename L::template Smem<T, MAXF, POOL>;
    using Params = std::conditional_t<TAINT, DraTaintsParams<PARTS, NT>, DraParams<PARTS, POOL>>;
    using Smem = std::conditional_t<TAINT, DraTaintsSmem<Base, NT>, Base>;
};

template <int W>
__device__ __forceinline__ uint32_t byte_at(const uint32_t (&w)[W], int k) { return (w[k >> 2] >> (8 * (k & 3))) & 0xffu; }
// bytes before the first NUL (all 4 W when there is none)
template <int W>
__device__ __forceinline__ uint32_t nul_len(const uint32_t (&w)[W]) {
    uint32_t l = 4u * W;
#pragma unroll
    for (int k = 4 * W - 1; k >= 0; k--) if (byte_at(w, k) == 0u) l = (uint32_t)k;
    return l;
}
__device__ __forceinline__ bool is_lhex(uint32_t c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f'); }
// every byte k in [from, len) satisfies ok(c)
template <int W, typename F>
__device__ __forceinline__ bool bytes_ok(const uint32_t (&w)[W], uint32_t from, uint32_t len, F ok) {
    bool good = true;
#pragma unroll
    for (int k = 0; k < 4 * W; k++) if ((uint32_t)k >= from && (uint32_t)k < len && !ok(byte_at(w, k))) good = false;
    return good;
}

// t in [0, TAINT_SINCE_MAX] as RFC 3339 in UTC, "YYYY-MM-DDTHH:MM:SSZ": the days since 1970-01-01 become a proleptic
// Gregorian date by the 400-year-era arithmetic of civil_from_days (H. Hinnant, "chrono-Compatible Low-Level Date
// Algorithms"), all in 32 bits
__device__ __forceinline__ void rfc3339(unsigned long long t, uint8_t *o) {
    const uint32_t days = (uint32_t)(t >> 7) / 675u;  // t / 86400, 86400 = 2^7 * 675, t >> 7 < 2^31
    const uint32_t sod = (uint32_t)(t - (unsigned long long)days * 86400ull);
    const uint32_t z = days + 719468u, era = z / 146097u, doe = z - era * 146097u;  // days since 0000-03-01
    const uint32_t yoe = (doe - doe / 1460u + doe / 36524u - doe / 146096u) / 365u;
    const uint32_t doy = doe - (365u * yoe + yoe / 4u - yoe / 100u), mp = (5u * doy + 2u) / 153u;  // March = 0
    const uint32_t day = doy - (153u * mp + 2u) / 5u + 1u, month = mp < 10u ? mp + 3u : mp - 9u;
    const uint32_t year = era * 400u + yoe + (month <= 2u ? 1u : 0u);
    dec_write(year, 4u, o);
    const uint32_t two[5] = {month, day, sod / 3600u, sod / 60u % 60u, sod % 60u};
    const char sep[6] = "--T::";
#pragma unroll
    for (int k = 0; k < 5; k++) {
        o[4 + 3 * k] = (uint8_t)sep[k];
        o[5 + 3 * k] = (uint8_t)('0' + two[k] / 10u);
        o[6 + 3 * k] = (uint8_t)('0' + two[k] % 10u);
    }
    o[19] = (uint8_t)'Z';
}

// NT = 0: kxpu_dra_slices[_mdev], TILE devices per slice.  NT > 0: the taint calls with a table of up to NT entries,
// TAINT_TILE devices per slice and a list of taints after a tainted device's attributes.  Everything the taints add sits
// behind `if constexpr`.
template <int LAYOUT, int NT = 0>
__global__ void __launch_bounds__(EMIT_THREADS, DraKernel<LAYOUT, NT>::MIN_CTAS)
    k_dra_slices(const __grid_constant__ typename DraKernel<LAYOUT, NT>::Params E) {
    using K = DraKernel<LAYOUT, NT>;
    using Rec = typename DraLayout<LAYOUT>::Rec;
    constexpr int HEAD = K::PARTS - 2, TAIL = K::PARTS - 1, T = K::T;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    typename K::Smem &S = *reinterpret_cast<typename K::Smem *>(smem_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    const uint32_t slice = blockIdx.x, i0 = slice * T;
    const uint32_t in_slice = E.n > i0 ? min(E.n - i0, (uint32_t)T) : 0u;
    for (uint32_t k = tid; k < E.pool_len; k += EMIT_THREADS) S.pool[k] = E.pool[k];
    const auto name_ok = [](uint32_t c) {
        return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '_' || c == '.' || c == '-';
    };

    // ---- fragment lengths, digits and the domain checks: one thread per device
    uint32_t flen = 0;
    if (LAYOUT == LAYOUT_PCI && tid < in_slice) {
        const uint4 *p = reinterpret_cast<const uint4 *>(static_cast<const Rec *>(E.devs) + i0 + tid);
        const uint4 q0 = p[0], q1 = p[1], q2 = p[2], q3 = p[3], q4 = p[4], q5 = p[5], q6 = p[6], q7 = p[7];
        const uint32_t prod[16] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
        const uint32_t bdf[4] = {q4.x, q4.y, q4.z, q4.w}, root[4] = {q5.x, q5.y, q5.z, q5.w};
        const uint32_t ven[2] = {q6.x, q6.y}, dev[2] = {q6.z, q6.w};
        const unsigned long long mask = ((unsigned long long)q7.y << 32) | q7.x;
        const uint32_t group = q7.z, plen_raw = q7.w & 0xffu;
        const uint32_t pl = plen_raw <= 64u ? plen_raw : 64u;  // out of the domain: reported below, bounded here
        const uint32_t bl = nul_len(bdf), rl = nul_len(root), vl_raw = nul_len(ven), dl_raw = nul_len(dev);
        const uint32_t vl = min(vl_raw, 6u), dl = min(dl_raw, 6u);  // bounded like pl
        const auto hex = [](uint32_t c) { return is_lhex(c); };
        if (plen_raw > 64u) E.flags[DRA_F_PLEN] = 1u;
        if (!bytes_ok(prod, 0u, pl, name_ok)) E.flags[DRA_F_PRODUCT] = 1u;
        if (bl == 0u || !bytes_ok(bdf, 0u, bl, [](uint32_t c) { return is_lhex(c) || c == ':' || c == '.'; })) E.flags[DRA_F_BDF] = 1u;
        if (rl != 0u && (rl < 4u || byte_at(root, 0) != 'p' || byte_at(root, 1) != 'c' || byte_at(root, 2) != 'i' ||
                         !bytes_ok(root, 3u, rl, [](uint32_t c) { return is_lhex(c) || c == ':'; })))
            E.flags[DRA_F_ROOT] = 1u;
        if (vl_raw == 0u || vl_raw > 6u || !bytes_ok(ven, 0u, vl, hex)) E.flags[DRA_F_VENDOR] = 1u;
        if (dl_raw == 0u || dl_raw > 6u || !bytes_ok(dev, 0u, dl, hex)) E.flags[DRA_F_DEVICE] = 1u;
        if (group == 0xFFFFFFFFu) E.flags[DRA_F_GROUP] = 1u;
        const bool one_node = mask != 0ull && (mask & (mask - 1ull)) == 0ull;
        const uint32_t node = one_node ? (uint32_t)__ffsll((long long)mask) - 1u : 0u;
        const uint32_t gl = dec_len(group), nl = one_node ? dec_len(node) : 0u;
        dec_write(group, gl, S.dec[tid]);
        if (one_node) dec_write(node, nl, S.dec[tid] + 10);
        S.meta[tid] = gl | (nl << 4) | (bl << 8) | (rl << 13) | (vl << 18) | (dl << 21) | (pl << 24);
        flen = DRA_LIT_TOTAL - E.len[3] - E.len[5] - E.len[6] + 2u * gl + bl + vl + dl + (nl ? E.len[3] + nl : 0u) +
               (pl ? E.len[5] + pl : 0u) + (rl ? E.len[6] + rl : 0u) + (tid + 1u < in_slice ? 1u : 0u);
    }
    if constexpr (LAYOUT == LAYOUT_MDEV) {
        if (tid < in_slice) {
            // 208 bytes = 13 uint4; read field by field so that no more than a few of them are live at once
            const uint4 *p = reinterpret_cast<const uint4 *>(static_cast<const Rec *>(E.devs) + i0 + tid);
            uint32_t pl, tl, bl, rl, vl, dl;
            {  // product_len and product (q12, q0..q3)
                const uint32_t plen_raw = p[12].z & 0xffu;
                pl = plen_raw <= 64u ? plen_raw : 64u;  // out of the domain: reported, and bounded here
                if (plen_raw > 64u) E.flags[DRAM_F_PLEN] = 1u;
                const uint4 q0 = p[0], q1 = p[1], q2 = p[2], q3 = p[3];
                const uint32_t prod[16] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w,
                                           q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
                if (plen_raw <= 64u && !bytes_ok(prod, 0u, pl, name_ok)) E.flags[DRAM_F_PRODUCT] = 1u;
            }
            {  // mdev_type: bytes 64..104 (q4, q5, q6.xy)
                const uint4 q4 = p[4], q5 = p[5];
                const uint2 q6 = reinterpret_cast<const uint2 *>(p + 6)[0];
                const uint32_t ty[10] = {q4.x, q4.y, q4.z, q4.w, q5.x, q5.y, q5.z, q5.w, q6.x, q6.y};
                tl = nul_len(ty);
                if (tl == 0u || !bytes_ok(ty, 0u, tl, name_ok)) E.flags[DRAM_F_TYPE] = 1u;
            }
            {  // uuid: bytes 104..140 (q6.zw, q7, q8.xyz)
                const uint2 q6 = reinterpret_cast<const uint2 *>(p + 6)[1];
                const uint4 q7 = p[7], q8 = p[8];
                const uint32_t uw[9] = {q6.x, q6.y, q7.x, q7.y, q7.z, q7.w, q8.x, q8.y, q8.z};
                if (!kxmdev::uuid_ok(uw)) E.flags[DRAM_F_UUID] = 1u;
            }
            {  // parent and pcie_root (q9, q10)
                const uint4 q9 = p[9], q10 = p[10];
                const uint32_t par[4] = {q9.x, q9.y, q9.z, q9.w}, root[4] = {q10.x, q10.y, q10.z, q10.w};
                bl = nul_len(par);
                rl = nul_len(root);
                if (bl == 0u || !bytes_ok(par, 0u, bl, [](uint32_t c) { return is_lhex(c) || c == ':' || c == '.'; }))
                    E.flags[DRAM_F_PARENT] = 1u;
                if (rl != 0u && (rl < 4u || byte_at(root, 0) != 'p' || byte_at(root, 1) != 'c' || byte_at(root, 2) != 'i' ||
                                 !bytes_ok(root, 3u, rl, [](uint32_t c) { return is_lhex(c) || c == ':'; })))
                    E.flags[DRAM_F_ROOT] = 1u;
            }
            {  // vendor and device (q11)
                const uint4 q11 = p[11];
                const uint32_t ven[2] = {q11.x, q11.y}, dev[2] = {q11.z, q11.w};
                const uint32_t vl_raw = nul_len(ven), dl_raw = nul_len(dev);
                vl = min(vl_raw, 6u);
                dl = min(dl_raw, 6u);
                const auto hex = [](uint32_t c) { return is_lhex(c); };
                if (vl_raw == 0u || vl_raw > 6u || !bytes_ok(ven, 0u, vl, hex)) E.flags[DRAM_F_VENDOR] = 1u;
                if (dl_raw > 6u || !bytes_ok(dev, 0u, dl, hex)) E.flags[DRAM_F_DEVICE] = 1u;
            }
            const uint32_t group = p[8].w;
            const uint2 qm = reinterpret_cast<const uint2 *>(p + 12)[0];
            const unsigned long long mask = ((unsigned long long)qm.y << 32) | qm.x;
            if (group == 0xFFFFFFFFu) E.flags[DRAM_F_GROUP] = 1u;
            const bool one_node = mask != 0ull && (mask & (mask - 1ull)) == 0ull;
            const uint32_t node = one_node ? (uint32_t)__ffsll((long long)mask) - 1u : 0u;
            const uint32_t gl = dec_len(group), nl = one_node ? dec_len(node) : 0u;
            dec_write(group, gl, S.dec[tid]);
            if (one_node) dec_write(node, nl, S.dec[tid] + 10);
            S.meta[tid] = gl | (nl << 4) | (bl << 8) | (rl << 13) | (vl << 18) | (dl << 21) | (pl << 24);
            S.tlen[tid] = (uint8_t)tl;
            const uint32_t ls = E.len[DRAM_S], li = E.len[DRAM_I];
            flen = E.len[0] + E.len[1] + 2u * gl + li + E.len[2] + tl + ls + E.len[4] + bl + ls + E.len[6] + vl + ls +
                   E.len[9] + 36u + ls + E.len[DRAM_E] + (nl ? E.len[3] + nl + li : 0u) + (dl ? E.len[5] + dl + ls : 0u) +
                   (pl ? E.len[7] + pl + ls : 0u) + (rl ? E.len[8] + rl + ls : 0u) + (tid + 1u < in_slice ? 1u : 0u);
        }
    }
    if constexpr (K::TAINT) {  // the device's row of the table: which taints it carries, and their times
        if (tid < in_slice) {
            const long long *row = E.since + (size_t)(i0 + tid) * E.nt;
            uint32_t carried = 0, part = 0;
            for (uint32_t t = 0; t < E.nt; t++) {
                const long long since = row[t];
                if (since > TAINT_SINCE_MAX) E.flags[K::F_SINCE] = 1u;
                if (since < 0 || since > TAINT_SINCE_MAX) continue;
                if (carried & E.dup[t]) E.flags[K::F_DUP] = 1u;
                rfc3339((unsigned long long)since, S.ts[tid][t]);
                part += (carried ? 1u : 0u) + E.len[K::T_ENTRY + t] + 20u + E.len[K::T_ECLOSE];
                carried |= 1u << t;
            }
            S.carried[tid] = (uint8_t)carried;
            if (carried) flen += E.len[K::T_OPEN] + part + E.len[K::T_CLOSE] - 1u;
        }
    }
    // ---- scan of the 128 lengths (threads >= TILE contribute 0)
    const uint32_t incl = kxscan::warp_incl(flen);
    if (lane == 31) S.wsum[w] = incl;
    __syncthreads();
    if (w == 0) {
        const uint32_t x = lane < EMIT_THREADS / 32 ? S.wsum[lane] : 0u;
        const uint32_t xi = kxscan::warp_incl(x);
        if (lane < EMIT_THREADS / 32) S.wsum[lane] = xi - x;
        if (lane == EMIT_THREADS / 32 - 1) S.tile_total = xi;
    }
    __syncthreads();
    const uint32_t head_len = E.len[HEAD], tail_len = E.len[TAIL], tile_total = S.tile_total;
    if (tid < T) S.start[tid] = head_len + S.wsum[w] + incl - flen;
    // ---- the slice's offset in the output: decoupled look-back over the slice totals; its exclusive prefix is slice_off[s]
    if (w == 0) {
        const unsigned long long agg = (unsigned long long)head_len + tile_total + tail_len;
        const unsigned long long excl = kxscan::lookback(E.state, slice, agg, E.epoch);
        if (lane == 0) {
            S.base = excl;
            E.slice_off[slice] = excl;
            if (slice == gridDim.x - 1) E.slice_off[slice + 1] = excl + agg;
        }
    }
    __syncthreads();
    const unsigned long long base = S.base;
    uint8_t *stg = S.stage + ((reinterpret_cast<uintptr_t>(E.out) + base) & 15u);  // same 16-byte phase in smem and global
    for (uint32_t k = tid; k < head_len; k += EMIT_THREADS) stg[k] = S.pool[E.off[HEAD] + k];
    for (uint32_t k = tid; k < tail_len; k += EMIT_THREADS) stg[head_len + tile_total + k] = S.pool[E.off[TAIL] + k];
    // ---- fragments: one warp per device; the string fields straight from the record (L1 / L2)
    for (uint32_t d = w; d < in_slice; d += EMIT_THREADS / 32) {
        const uint32_t m = S.meta[d];
        const uint32_t gl = m & 15u, nl = (m >> 4) & 3u, bl = (m >> 8) & 31u, rl = (m >> 13) & 31u, vl = (m >> 18) & 7u,
                       dl = (m >> 21) & 7u, pl = m >> 24;
        const Rec *r = static_cast<const Rec *>(E.devs) + i0 + d;
        uint8_t *dst = stg + S.start[d];
        uint32_t o = 0;
        auto put = [&](const uint8_t *src, uint32_t L) {
            for (uint32_t l = lane; l < L; l += 32u) dst[o + l] = src[l];
            o += L;
        };
        auto lit = [&](int k) { put(S.pool + E.off[k], E.len[k]); };
        // the literal that closes the device (K's LAST); a tainted device's taint part goes before its final '}'
        auto close = [&](int k) {
            if constexpr (K::TAINT) {
                const uint32_t carried = S.carried[d];
                if (carried) {
                    put(S.pool + E.off[k], E.len[k] - 1u);
                    lit(K::T_OPEN);
                    for (uint32_t t = 0; t < (uint32_t)NT; t++) {
                        if (!((carried >> t) & 1u)) continue;
                        if (carried & ((1u << t) - 1u)) {
                            if (lane == 0) dst[o] = (uint8_t)',';
                            o += 1u;
                        }
                        lit(K::T_ENTRY + t); put(S.ts[d][t], 20u); lit(K::T_ECLOSE);
                    }
                    lit(K::T_CLOSE);
                    return;
                }
            }
            lit(k);
        };
        const auto bytes = [](const char *s) { return reinterpret_cast<const uint8_t *>(s); };
        if constexpr (LAYOUT == LAYOUT_PCI) {
            lit(0); put(S.dec[d], gl); lit(1); put(bytes(r->device), dl);
            lit(2); put(S.dec[d], gl);
            if (nl) { lit(3); put(S.dec[d] + 10, nl); }
            lit(4); put(bytes(r->bdf), bl);
            if (pl) { lit(5); put(r->product, pl); }
            if (rl) { lit(6); put(bytes(r->pcie_root), rl); }
            lit(7); put(bytes(r->vendor), vl); close(DraLayout<LAYOUT>::LAST);
        } else {
            const uint32_t tl = S.tlen[d];
            lit(0); put(S.dec[d], gl); lit(1); put(S.dec[d], gl); lit(DRAM_I);
            lit(2); put(bytes(r->mdev_type), tl); lit(DRAM_S);
            if (nl) { lit(3); put(S.dec[d] + 10, nl); lit(DRAM_I); }
            lit(4); put(bytes(r->parent), bl); lit(DRAM_S);
            if (dl) { lit(5); put(bytes(r->device), dl); lit(DRAM_S); }
            lit(6); put(bytes(r->vendor), vl); lit(DRAM_S);
            if (pl) { lit(7); put(r->product, pl); lit(DRAM_S); }
            if (rl) { lit(8); put(bytes(r->pcie_root), rl); lit(DRAM_S); }
            lit(9); put(bytes(r->uuid), 36u); lit(DRAM_S); close(DraLayout<LAYOUT>::LAST);
        }
        if (d + 1u < in_slice && lane == 0) dst[o] = (uint8_t)',';
    }
    tile_store(E.out + base, stg, head_len + tile_total + tail_len);
}

// ------------------------------------------------------------------ Allocate names
// name i = prefix + decimal(idx[i]), prefix = kind + "=" (<= 64 bytes)
struct NamePrefix {
    uint8_t b[KIND_MAX + 1];
    uint32_t len;
};
__global__ void __launch_bounds__(256) k_alloc_len(const unsigned long long *__restrict__ idx, uint32_t n,
                                                   uint32_t *__restrict__ lens, uint32_t prefix_len) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    lens[i] = i < n ? prefix_len + dec_len(idx[i]) : 0u;
}
__global__ void __launch_bounds__(256) k_alloc_write(const unsigned long long *__restrict__ idx, uint32_t n,
                                                     const uint32_t *__restrict__ offs, uint8_t *__restrict__ out,
                                                     const __grid_constant__ NamePrefix P) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t *dst = out + offs[i];
    for (uint32_t k = 0; k < P.len; k++) dst[k] = P.b[k];
    unsigned long long v = idx[i];
    dec_write(v, dec_len(v), dst + P.len);
}

// ------------------------------------------------------------------ vGPU type keys (kxpu_mdev_names)
// one gathered 128-byte record per thread: the key length, then the key bytes at their offset
__device__ __forceinline__ uint32_t mdev_key(const kxpu_mdevrec *rec, uint8_t *dst) {
    const uint4 *rp = reinterpret_cast<const uint4 *>(rec);
    const uint4 q4 = rp[4], q5 = rp[5], q6 = rp[6], q7 = rp[7];
    const uint32_t nw[10] = {q4.w, q5.x, q5.y, q5.z, q5.w, q6.x, q6.y, q6.z, q6.w, q7.x};  // type_name @76
    const uint32_t nlen = (q7.z >> 8) & 0xffu, fl = (q7.z >> 16) & 0xffu;
    if ((fl & KXPU_REC_NAME_ERR) || nlen > kxmdev::NAME_MAX_BYTES) return 0u;
    return kxmdev::type_key(nw, nlen, [&](uint32_t p, uint8_t c) { if (dst) dst[p] = c; });
}
__global__ void __launch_bounds__(256) k_mdev_name_len(const kxpu_mdevrec *__restrict__ recs, uint32_t n, uint32_t *__restrict__ lens) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    lens[i] = i < n ? mdev_key(recs + i, nullptr) : 0u;
}
__global__ void __launch_bounds__(256) k_mdev_name_write(const kxpu_mdevrec *__restrict__ recs, uint32_t n,
                                                         const uint32_t *__restrict__ offs, uint8_t *__restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    mdev_key(recs + i, out + offs[i]);
}

// ------------------------------------------------------------------ ListAndWatchResponse
// repeated Device devices = 1; Device { string ID = 1; string health = 2; TopologyInfo topology = 3; }
// TOPO = false: kxpu_lw_encode (no topology, every length fits one byte).  TOPO = true: kxpu_lw_encode_topo, field 3
// when the device's mask is non-zero: TopologyInfo { repeated NUMANode nodes = 1 { int64 ID = 1 } }, nodes ascending.
// A NUMANode of node k > 0 is 0a 02 08 k (4 bytes, k < 128 is one varint byte); node 0 is 0a 00 (proto3 drops the zero
// ID).  Up to 64 nodes make the topology 254 bytes and the Device 280: both lengths become two-byte varints.
__device__ __forceinline__ uint32_t topo_len(unsigned long long mask) {  // TopologyInfo body
    return 4u * (uint32_t)__popcll(mask) - 2u * (uint32_t)(mask & 1ull);
}
__device__ __forceinline__ uint32_t varint_len(uint32_t v) { return v < 128u ? 1u : 2u; }  // v < 2^14 here
__device__ __forceinline__ uint8_t *varint_write(uint32_t v, uint8_t *d) {
    if (v < 128u) { d[0] = (uint8_t)v; return d + 1; }
    d[0] = (uint8_t)(0x80u | (v & 0x7fu)); d[1] = (uint8_t)(v >> 7); return d + 2;
}
// the Device body length of device i
template <bool TOPO>
__device__ __forceinline__ uint32_t lw_body(uint32_t group, bool ok, unsigned long long mask) {
    uint32_t l = 2u + dec_len(group) + 2u + (ok ? 7u : 9u);
    if (TOPO && mask) { const uint32_t t = topo_len(mask); l += 1u + varint_len(t) + t; }
    return l;
}
template <bool TOPO>
__global__ void __launch_bounds__(256) k_lw_len(const uint32_t *__restrict__ groups, const uint8_t *__restrict__ healthy,
                                                const unsigned long long *__restrict__ masks, uint32_t n, uint32_t *__restrict__ lens) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n) return;
    if (i == n) { lens[i] = 0; return; }
    const uint32_t body = lw_body<TOPO>(groups[i], !healthy || healthy[i], TOPO && masks ? masks[i] : 0ull);
    lens[i] = 1u + (TOPO ? varint_len(body) : 1u) + body;
}
template <bool TOPO>
__global__ void __launch_bounds__(256) k_lw_write(const uint32_t *__restrict__ groups, const uint8_t *__restrict__ healthy,
                                                  const unsigned long long *__restrict__ masks, uint32_t n,
                                                  const uint32_t *__restrict__ offs, uint8_t *__restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool ok = !healthy || healthy[i];
    const char hs[10] = "Unhealthy";
    const unsigned long long mask = TOPO && masks ? masks[i] : 0ull;
    const uint32_t hl = ok ? 7u : 9u, gl = dec_len(groups[i]);
    uint8_t *d = out + offs[i];
    d[0] = 0x0a;
    if (TOPO) d = varint_write(lw_body<TOPO>(groups[i], ok, mask), d + 1) - 2;  // d + 2 = start of the body
    else d[1] = (uint8_t)(2u + gl + 2u + hl);
    d[2] = 0x0a; d[3] = (uint8_t)gl;
    dec_write(groups[i], gl, d + 4);
    d[4 + gl] = 0x12; d[5 + gl] = (uint8_t)hl;
    for (uint32_t k = 0; k < hl; k++) d[6 + gl + k] = (uint8_t)hs[ok ? k + 2 : k];  // "Healthy" = "Unhealthy"+2 with 'h'->'H'
    if (ok) d[6 + gl] = (uint8_t)'H';
    if (TOPO && mask) {
        uint8_t *t = d + 6 + gl + hl;
        *t++ = 0x1a;
        t = varint_write(topo_len(mask), t);
        for (unsigned long long m = mask; m; m &= m - 1ull) {
            const uint32_t k = (uint32_t)__ffsll((long long)m) - 1u;
            t[0] = 0x0a;
            if (k == 0u) { t[1] = 0x00; t += 2; }
            else { t[1] = 0x02; t[2] = 0x08; t[3] = (uint8_t)k; t += 4; }
        }
    }
}

}  // namespace kxemit

using namespace kxemit;

template <int FMT, int MAXF, int LAYOUT>
static void emit_launch(kxpu_ctx *ctx, uint32_t tiles, const EmitParams &E) {
    k_cdi_fused<FMT, MAXF, LAYOUT><<<tiles, EMIT_THREADS, sizeof(EmitSmem<MAXF, LAYOUT>), ctx->stream>>>(E);
}

static const Parts &parts_of(int32_t format, int layout) {
    const bool yaml = format == KXPU_FMT_YAML;
    if (layout == LAYOUT_MDEV) return yaml ? h_yaml_mdev_parts : h_json_mdev_parts;
    if (layout == LAYOUT_CDEV) return yaml ? h_yaml_cdev_parts : h_json_cdev_parts;
    if (layout == LAYOUT_MDEV_CDEV) return yaml ? h_yaml_mdev_cdev_parts : h_json_mdev_cdev_parts;
    if (layout == LAYOUT_TYPED) return yaml ? h_yaml_typed_parts : h_json_typed_parts;
    if (layout == LAYOUT_TYPED_CDEV) return yaml ? h_yaml_typed_cdev_parts : h_json_typed_cdev_parts;
    return yaml ? h_yaml_parts : h_json_parts;
}

bool kx_cdi_kind_ok(const char *kind) { return kind_ok(kind); }

std::string kx_cdi_part(int32_t format, int layout, int k, const char *kind) { return part_text(parts_of(format, layout), k, kind); }

template <int MAXF, int LAYOUT>
static void emit_smem_attr() {
    cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_YAML, MAXF, LAYOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)sizeof(EmitSmem<MAXF, LAYOUT>));
    cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_JSON, MAXF, LAYOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)sizeof(EmitSmem<MAXF, LAYOUT>));
}

int32_t kx_cdi_emit_enqueue(kxpu_ctx *ctx, int32_t format, const char *kind, const void *d_devs, size_t n, int layout,
                            KxScratch &sc, uint8_t **d_out_p, unsigned long long **d_total_p, bool timed) {
    const bool mdev = layout == LAYOUT_MDEV || layout == LAYOUT_MDEV_CDEV;
    const Parts &parts = parts_of(format, layout);
    static bool cdev_attr_done = false;
    if (layout == LAYOUT_CDEV && !cdev_attr_done) {
        emit_smem_attr<MAX_FRAG_CDEV, LAYOUT_CDEV>();
        emit_smem_attr<MAX_FRAG_CDEV_LONG, LAYOUT_CDEV>();
        cdev_attr_done = true;
    }
    static bool mdev_cdev_attr_done = false;
    if (layout == LAYOUT_MDEV_CDEV && !mdev_cdev_attr_done) {
        emit_smem_attr<MAX_FRAG_MDEV_CDEV, LAYOUT_MDEV_CDEV>();
        mdev_cdev_attr_done = true;
    }
    const bool typed = layout == LAYOUT_TYPED || layout == LAYOUT_TYPED_CDEV;
    static bool typed_attr_done = false;
    if (typed && !typed_attr_done) {
        emit_smem_attr<MAX_FRAG_TYPED, LAYOUT_TYPED>();
        emit_smem_attr<MAX_FRAG_TYPED_LONG, LAYOUT_TYPED>();
        emit_smem_attr<MAX_FRAG_TYPED_CDEV, LAYOUT_TYPED_CDEV>();
        emit_smem_attr<MAX_FRAG_TYPED_CDEV_LONG, LAYOUT_TYPED_CDEV>();
        typed_attr_done = true;
    }
    static bool attr_done = false;
    if (!attr_done) {
        cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_YAML, MAX_FRAG, LAYOUT_PCI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)sizeof(TileSmem<MAX_FRAG>));
        cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_JSON, MAX_FRAG, LAYOUT_PCI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)sizeof(TileSmem<MAX_FRAG>));
        cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_YAML, MAX_FRAG_LONG, LAYOUT_PCI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)sizeof(TileSmem<MAX_FRAG_LONG>));
        cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_JSON, MAX_FRAG_LONG, LAYOUT_PCI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)sizeof(TileSmem<MAX_FRAG_LONG>));
        cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_YAML, MAX_FRAG_MDEV, LAYOUT_MDEV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)sizeof(TileSmem<MAX_FRAG_MDEV>));
        cudaFuncSetAttribute(k_cdi_fused<KXPU_FMT_JSON, MAX_FRAG_MDEV, LAYOUT_MDEV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)sizeof(TileSmem<MAX_FRAG_MDEV>));
        attr_done = true;
    }
    EmitParams E;
    memset(&E, 0, sizeof E);
    uint32_t acc = 0;
    for (int k = 0; k < 9; k++) {
        const std::string s = part_text(parts, k < 8 ? k : 9, kind);  // slot 8 <- part 9 (part 8 is the zero-device document)
        if (acc + s.size() > (size_t)POOL_MAX) return KXPU_E_INVALID;  // the literals grew: POOL_MAX must follow
        memcpy(E.pool + acc, s.data(), s.size());
        E.off[k] = (uint16_t)acc;
        E.len[k] = (uint16_t)s.size();
        acc += E.len[k];
        if (k < 6 || k == 8) E.lit_total += E.len[k];
    }
    if (typed) {  // part 10, the literal after the type key
        const std::string s = part_text(parts, 10, kind);
        if (acc + s.size() > (size_t)POOL_MAX) return KXPU_E_INVALID;
        memcpy(E.pool + acc, s.data(), s.size());
        E.off10 = (uint16_t)acc;
        E.len10 = (uint16_t)s.size();
        acc += E.len10;
        E.lit_total += E.len10;
    }
    E.pool_len = acc;
    const uint32_t N = (uint32_t)n;
    const uint32_t tiles = (N + TILE - 1) / TILE;
    const uint32_t frag = E.lit_total + 2 * 20 + 2 * 10 + 15 + 2 + 2 + (mdev ? 36 : 0) + (typed ? 10 + 40 : 0);  // no fragment is longer
    const size_t bound = (size_t)n * frag + E.len[6] + E.len[7] + 64;
    // kinds up to 22 bytes fit the four-CTAs-per-SM tile, longer ones take the MAX_FRAG_LONG instantiation (cdev: both
    // bounds CDEV_EXTRA larger, so the same kinds); every mdev kind the MAX_FRAG_MDEV one (mdev cdev: MAX_FRAG_MDEV_CDEV).
    // The typed layouts split the kinds the same way, with bounds TYPED_EXTRA larger.
    const bool cdev = layout == LAYOUT_CDEV;
    const bool long_frag = layout == LAYOUT_TYPED        ? frag > (uint32_t)MAX_FRAG_TYPED
                           : layout == LAYOUT_TYPED_CDEV ? frag > (uint32_t)MAX_FRAG_TYPED_CDEV
                                                         : frag > (uint32_t)(cdev ? MAX_FRAG_CDEV : MAX_FRAG);
    const int max_frag = layout == LAYOUT_TYPED        ? MAX_FRAG_TYPED_LONG
                         : layout == LAYOUT_TYPED_CDEV ? MAX_FRAG_TYPED_CDEV_LONG
                         : layout == LAYOUT_MDEV_CDEV  ? MAX_FRAG_MDEV_CDEV
                         : mdev                        ? MAX_FRAG_MDEV
                         : cdev                        ? MAX_FRAG_CDEV_LONG : MAX_FRAG_LONG;
    if (frag > (uint32_t)max_frag) return KXPU_E_INVALID;  // the literals grew: the bound must follow
    uint8_t *d_out = nullptr;
    unsigned long long *d_total = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&d_out, bound));
    KX_CUDA(ctx, sc.alloc((void **)&d_total, 16));
    cudaMemsetAsync(d_total, 0, 16, ctx->stream);
    E.devs = d_devs; E.n = N; E.out = d_out; E.total_out = d_total; E.flags = (uint32_t *)(d_total + 1);
    E.state = kx_scan_state(ctx, tiles);
    if (!E.state) return KXPU_E_NOMEM;
    E.epoch = kx_next_epoch(ctx);
    auto launch = [&]() {
        if (layout == LAYOUT_TYPED) {
            if (format == KXPU_FMT_YAML) {
                if (long_frag) emit_launch<KXPU_FMT_YAML, MAX_FRAG_TYPED_LONG, LAYOUT_TYPED>(ctx, tiles, E);
                else emit_launch<KXPU_FMT_YAML, MAX_FRAG_TYPED, LAYOUT_TYPED>(ctx, tiles, E);
            } else {
                if (long_frag) emit_launch<KXPU_FMT_JSON, MAX_FRAG_TYPED_LONG, LAYOUT_TYPED>(ctx, tiles, E);
                else emit_launch<KXPU_FMT_JSON, MAX_FRAG_TYPED, LAYOUT_TYPED>(ctx, tiles, E);
            }
        } else if (layout == LAYOUT_TYPED_CDEV) {
            if (format == KXPU_FMT_YAML) {
                if (long_frag) emit_launch<KXPU_FMT_YAML, MAX_FRAG_TYPED_CDEV_LONG, LAYOUT_TYPED_CDEV>(ctx, tiles, E);
                else emit_launch<KXPU_FMT_YAML, MAX_FRAG_TYPED_CDEV, LAYOUT_TYPED_CDEV>(ctx, tiles, E);
            } else {
                if (long_frag) emit_launch<KXPU_FMT_JSON, MAX_FRAG_TYPED_CDEV_LONG, LAYOUT_TYPED_CDEV>(ctx, tiles, E);
                else emit_launch<KXPU_FMT_JSON, MAX_FRAG_TYPED_CDEV, LAYOUT_TYPED_CDEV>(ctx, tiles, E);
            }
        } else if (layout == LAYOUT_MDEV_CDEV) {
            if (format == KXPU_FMT_YAML) emit_launch<KXPU_FMT_YAML, MAX_FRAG_MDEV_CDEV, LAYOUT_MDEV_CDEV>(ctx, tiles, E);
            else emit_launch<KXPU_FMT_JSON, MAX_FRAG_MDEV_CDEV, LAYOUT_MDEV_CDEV>(ctx, tiles, E);
        } else if (mdev) {
            if (format == KXPU_FMT_YAML) emit_launch<KXPU_FMT_YAML, MAX_FRAG_MDEV, LAYOUT_MDEV>(ctx, tiles, E);
            else emit_launch<KXPU_FMT_JSON, MAX_FRAG_MDEV, LAYOUT_MDEV>(ctx, tiles, E);
        } else if (cdev) {
            if (format == KXPU_FMT_YAML) {
                if (long_frag) emit_launch<KXPU_FMT_YAML, MAX_FRAG_CDEV_LONG, LAYOUT_CDEV>(ctx, tiles, E);
                else emit_launch<KXPU_FMT_YAML, MAX_FRAG_CDEV, LAYOUT_CDEV>(ctx, tiles, E);
            } else {
                if (long_frag) emit_launch<KXPU_FMT_JSON, MAX_FRAG_CDEV_LONG, LAYOUT_CDEV>(ctx, tiles, E);
                else emit_launch<KXPU_FMT_JSON, MAX_FRAG_CDEV, LAYOUT_CDEV>(ctx, tiles, E);
            }
        } else if (format == KXPU_FMT_YAML) {
            if (long_frag) emit_launch<KXPU_FMT_YAML, MAX_FRAG_LONG, LAYOUT_PCI>(ctx, tiles, E);
            else emit_launch<KXPU_FMT_YAML, MAX_FRAG, LAYOUT_PCI>(ctx, tiles, E);
        } else {
            if (long_frag) emit_launch<KXPU_FMT_JSON, MAX_FRAG_LONG, LAYOUT_PCI>(ctx, tiles, E);
            else emit_launch<KXPU_FMT_JSON, MAX_FRAG, LAYOUT_PCI>(ctx, tiles, E);
        }
        KX_LAUNCHED(ctx);
    };
    if (timed) {
        KxTimer tm(ctx, KXPU_T_EMIT);
        launch();
    } else {
        launch();
    }
    *d_out_p = d_out;
    *d_total_p = d_total;
    return KXPU_OK;
}

// LAYOUT_MDEV: devs is kxpu_mdevcdi[n], LAYOUT_MDEV_CDEV: kxpu_mdevcdev[n], the typed layouts kxpu_vfvgpucdi[n], else
// kxpu_cdidev[n]
static int32_t cdi_emit(kxpu_ctx *ctx, int32_t format, const char *kind, const void *devs, size_t n, uint8_t *out,
                        size_t cap, size_t *len, int layout = LAYOUT_PCI) {
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    if (n == 0) {  // Devices stays nil: yaml "devices: []", json "devices": null (cdi/spec.go:42-49)
        const std::string doc = kx_cdi_part(format, layout, 8, kind);
        *len = doc.size();
        if (cap < *len || !out) return KXPU_E_NOSPACE;
        memcpy(out, doc.data(), *len);
        return KXPU_OK;
    }
    const bool typed = layout == LAYOUT_TYPED || layout == LAYOUT_TYPED_CDEV;
    const size_t dev_bytes = layout == LAYOUT_MDEV ? sizeof(kxpu_mdevcdi)
                             : layout == LAYOUT_MDEV_CDEV ? sizeof(kxpu_mdevcdev)
                             : typed ? sizeof(kxpu_vfvgpucdi) : sizeof(kxpu_cdidev);
    KxScratch sc(ctx);
    void *d_devs = nullptr;
    uint8_t *d_out = nullptr;
    unsigned long long *d_total = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&d_devs, n * dev_bytes));
    cudaMemcpyAsync(d_devs, devs, n * dev_bytes, cudaMemcpyHostToDevice, ctx->stream);
    const int32_t rc = kx_cdi_emit_enqueue(ctx, format, kind, d_devs, n, layout, sc, &d_out, &d_total, true);
    if (rc != KXPU_OK) return rc;
    unsigned long long h[2] = {0, 0};
    cudaMemcpyAsync(h, d_total, 16, cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "cdi_emit failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if ((uint32_t)h[1]) {
        KX_SET_ERR(ctx, "cdi_emit: bdf outside [0-9a-f:.]{1,16}, or one YAML would read as a number or not as a plain string");
        return KXPU_E_UNSUPPORTED;
    }
    if ((uint32_t)(h[1] >> 32) && typed) {
        KX_SET_ERR(ctx, "cdi_emit_vf_vgpu: a type ID of 0, or a type key that is empty, longer than 40 bytes or outside [A-Za-z0-9_.-]");
        return KXPU_E_UNSUPPORTED;
    }
    if ((uint32_t)(h[1] >> 32)) { KX_SET_ERR(ctx, "cdi_emit_mdev: uuid outside the canonical lowercase form"); return KXPU_E_UNSUPPORTED; }
    const size_t total = (size_t)h[0];
    *len = total;
    if (cap < total || !out) return KXPU_E_NOSPACE;
    cudaMemcpyAsync(out, d_out, total, cudaMemcpyDeviceToHost, ctx->stream);
    e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "cdi_emit D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}

extern "C" int32_t kxpu_cdi_emit(kxpu_ctx *ctx, int32_t format, const kxpu_cdidev *devs, size_t n, uint8_t *out,
                                 size_t cap, size_t *len) {
    if (!ctx || !len || (n && !devs) || (format != KXPU_FMT_YAML && format != KXPU_FMT_JSON)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    return cdi_emit(ctx, format, kDefaultKind, devs, n, out, cap, len);
}

extern "C" int32_t kxpu_cdi_emit_kind(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_cdidev *devs, size_t n,
                                      uint8_t *out, size_t cap, size_t *len) {
    if (!ctx || !len || !kind || (n && !devs) || (format != KXPU_FMT_YAML && format != KXPU_FMT_JSON)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (!kind_ok(kind)) { KX_SET_ERR(ctx, "cdi_emit_kind: kind is not a CDI vendor/class of at most 63 bytes"); return KXPU_E_UNSUPPORTED; }
    return cdi_emit(ctx, format, kind, devs, n, out, cap, len);
}

extern "C" int32_t kxpu_cdi_emit_mdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_mdevcdi *devs, size_t n,
                                      uint8_t *out, size_t cap, size_t *len) {
    static_assert(sizeof(kxpu_mdevcdi) == 64 && offsetof(kxpu_mdevcdi, parent) == 40, "kxpu_mdevcdi layout");
    if (!ctx || !len || !kind || (n && !devs) || (format != KXPU_FMT_YAML && format != KXPU_FMT_JSON)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (!kind_ok(kind)) { KX_SET_ERR(ctx, "cdi_emit_mdev: kind is not a CDI vendor/class of at most 63 bytes"); return KXPU_E_UNSUPPORTED; }
    return cdi_emit(ctx, format, kind, devs, n, out, cap, len, LAYOUT_MDEV);
}

extern "C" int32_t kxpu_cdi_emit_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_cdidev *devs, size_t n,
                                      uint8_t *out, size_t cap, size_t *len) {
    static_assert(offsetof(kxpu_cdidev, vfio_cdev) == 20, "kxpu_cdidev layout");
    if (!ctx || !len || !kind || (n && !devs) || (format != KXPU_FMT_YAML && format != KXPU_FMT_JSON)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (!kind_ok(kind)) { KX_SET_ERR(ctx, "cdi_emit_cdev: kind is not a CDI vendor/class of at most 63 bytes"); return KXPU_E_UNSUPPORTED; }
    return cdi_emit(ctx, format, kind, devs, n, out, cap, len, LAYOUT_CDEV);
}

extern "C" int32_t kxpu_cdi_emit_mdev_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_mdevcdev *devs,
                                           size_t n, uint8_t *out, size_t cap, size_t *len) {
    static_assert(sizeof(kxpu_mdevcdev) == 80 && offsetof(kxpu_mdevcdev, vfio_cdev) == 64, "kxpu_mdevcdev layout");
    if (!ctx || !len || !kind || (n && !devs) || (format != KXPU_FMT_YAML && format != KXPU_FMT_JSON)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (!kind_ok(kind)) { KX_SET_ERR(ctx, "cdi_emit_mdev_cdev: kind is not a CDI vendor/class of at most 63 bytes"); return KXPU_E_UNSUPPORTED; }
    return cdi_emit(ctx, format, kind, devs, n, out, cap, len, LAYOUT_MDEV_CDEV);
}

static int32_t cdi_emit_typed(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_vfvgpucdi *devs, size_t n,
                              uint8_t *out, size_t cap, size_t *len, int layout, const char *what) {
    static_assert(sizeof(kxpu_vfvgpucdi) == 80 && offsetof(kxpu_vfvgpucdi, type_id) == 32 && offsetof(kxpu_vfvgpucdi, key) == 40,
                  "kxpu_vfvgpucdi layout");
    if (!ctx || !len || !kind || (n && !devs) || (format != KXPU_FMT_YAML && format != KXPU_FMT_JSON)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (!kind_ok(kind)) { KX_SET_ERR(ctx, "%s: kind is not a CDI vendor/class of at most 63 bytes", what); return KXPU_E_UNSUPPORTED; }
    return cdi_emit(ctx, format, kind, devs, n, out, cap, len, layout);
}

extern "C" int32_t kxpu_cdi_emit_vf_vgpu(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_vfvgpucdi *devs,
                                         size_t n, uint8_t *out, size_t cap, size_t *len) {
    return cdi_emit_typed(ctx, format, kind, devs, n, out, cap, len, LAYOUT_TYPED, "cdi_emit_vf_vgpu");
}

extern "C" int32_t kxpu_cdi_emit_vf_vgpu_cdev(kxpu_ctx *ctx, int32_t format, const char *kind, const kxpu_vfvgpucdi *devs,
                                              size_t n, uint8_t *out, size_t cap, size_t *len) {
    return cdi_emit_typed(ctx, format, kind, devs, n, out, cap, len, LAYOUT_TYPED_CDEV, "cdi_emit_vf_vgpu_cdev");
}

// shared driver of the "thread per item" emitters.  h_in3 (optional, in3_bytes): one more input, uploaded like the
// others; its device address is stored to *d_in3 before the kernels are enqueued (the lambdas read it from there).
template <typename LenK, typename WriteK>
static int32_t emit_items(kxpu_ctx *ctx, size_t n, size_t in_bytes, const void *h_in, const uint8_t *h_in2, uint8_t *out,
                          size_t cap, uint32_t *offsets, size_t *need, LenK lenk, WriteK writek, const void *h_in3 = nullptr,
                          size_t in3_bytes = 0, const uint8_t **d_in3 = nullptr) {
    const uint32_t N = (uint32_t)n;
    uint8_t *b = nullptr;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    size_t o_in = take(in_bytes), o_in2 = take(h_in2 ? n : 16), o_lens = take((n + 1) * 4), o_offs = take((n + 1) * 4);
    const size_t o_in3 = h_in3 ? take(in3_bytes) : 0;
    KxScratch sc(ctx);
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaMemcpyAsync(b + o_in, h_in, in_bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (h_in2) cudaMemcpyAsync(b + o_in2, h_in2, n, cudaMemcpyHostToDevice, ctx->stream);
    if (h_in3) {
        cudaMemcpyAsync(b + o_in3, h_in3, in3_bytes, cudaMemcpyHostToDevice, ctx->stream);
        *d_in3 = b + o_in3;
    }
    uint32_t *d_lens = (uint32_t *)(b + o_lens), *d_offs = (uint32_t *)(b + o_offs);
    lenk(b + o_in, h_in2 ? b + o_in2 : nullptr, N, d_lens);
    ctx->launches++;
    int32_t rc = kxscan::exclusive_scan<uint32_t>(ctx, d_lens, n + 1, d_offs, nullptr);
    if (rc != KXPU_OK) return rc;  // no offsets were computed: nothing to copy or size
    std::vector<uint32_t> tmp;
    uint32_t *h_offs = offsets;
    if (!h_offs) { tmp.resize(n + 1); h_offs = tmp.data(); }
    cudaMemcpyAsync(h_offs, d_offs, (n + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "emit sizing failed: %s", cudaGetErrorString(e)); rc = KXPU_E_CUDA; }
    const size_t total = rc == KXPU_OK ? h_offs[n] : 0;
    if (need) *need = total;
    if (rc == KXPU_OK && (cap < total || (!out && total))) rc = KXPU_E_NOSPACE;
    if (rc == KXPU_OK && total) {
        uint8_t *d_out = nullptr;
        e = sc.alloc((void **)&d_out, total);
        if (e == cudaSuccess) {
            writek(b + o_in, h_in2 ? b + o_in2 : nullptr, N, d_offs, d_out);
            ctx->launches++;
            cudaMemcpyAsync(out, d_out, total, cudaMemcpyDeviceToHost, ctx->stream);
            e = cudaStreamSynchronize(ctx->stream);
        }
        if (e != cudaSuccess) { KX_SET_ERR(ctx, "emit write failed: %s", cudaGetErrorString(e)); rc = KXPU_E_CUDA; }
    }
    return rc;
}

static int32_t alloc_names(kxpu_ctx *ctx, const char *kind, const uint64_t *idx, size_t n, uint8_t *out, size_t cap,
                           uint32_t *offsets, size_t *need) {
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    if (n == 0) { offsets[0] = 0; if (need) *need = 0; return KXPU_OK; }
    NamePrefix P;
    memset(&P, 0, sizeof P);
    P.len = (uint32_t)strlen(kind) + 1u;  // kind_ok: <= 63 bytes
    memcpy(P.b, kind, P.len - 1u);
    P.b[P.len - 1u] = (uint8_t)'=';
    cudaStream_t st = ctx->stream;
    return emit_items(
        ctx, n, n * 8, idx, nullptr, out, cap, offsets, need,
        [st, &P](const uint8_t *in, const uint8_t *, uint32_t N, uint32_t *lens) {
            k_alloc_len<<<(N + 1 + 255) / 256, 256, 0, st>>>((const unsigned long long *)in, N, lens, P.len);
        },
        [st, &P](const uint8_t *in, const uint8_t *, uint32_t N, const uint32_t *offs, uint8_t *o) {
            k_alloc_write<<<(N + 255) / 256, 256, 0, st>>>((const unsigned long long *)in, N, offs, o, P);
        });
}

extern "C" int32_t kxpu_alloc_names(kxpu_ctx *ctx, const uint64_t *idx, size_t n, uint8_t *out, size_t cap,
                                    uint32_t *offsets, size_t *need) {
    if (!ctx || !offsets || (n && !idx)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    return alloc_names(ctx, kDefaultKind, idx, n, out, cap, offsets, need);
}

extern "C" int32_t kxpu_alloc_names_kind(kxpu_ctx *ctx, const char *kind, const uint64_t *idx, size_t n, uint8_t *out,
                                         size_t cap, uint32_t *offsets, size_t *need) {
    if (!ctx || !offsets || !kind || (n && !idx)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    if (!kind_ok(kind)) { KX_SET_ERR(ctx, "alloc_names_kind: kind is not a CDI vendor/class of at most 63 bytes"); return KXPU_E_UNSUPPORTED; }
    return alloc_names(ctx, kind, idx, n, out, cap, offsets, need);
}

extern "C" int32_t kxpu_mdev_names(kxpu_ctx *ctx, const kxpu_mdevrec *recs, size_t n, const uint32_t *rec_idx, size_t k,
                                   uint8_t *out, size_t cap, uint32_t *offsets, size_t *need) {
    if (!ctx || !offsets || (k && (!recs || !rec_idx))) return KXPU_E_INVALID;
    if (k >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    std::vector<kxpu_mdevrec> pick(k);  // only the k records travel to the device
    for (size_t j = 0; j < k; j++) {
        if (rec_idx[j] >= n) { KX_SET_ERR(ctx, "mdev_names: rec_idx[%zu] = %u is not below n = %zu", j, rec_idx[j], n); return KXPU_E_INVALID; }
        pick[j] = recs[rec_idx[j]];
    }
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    if (k == 0) { offsets[0] = 0; if (need) *need = 0; return KXPU_OK; }
    cudaStream_t st = ctx->stream;
    return emit_items(
        ctx, k, k * sizeof(kxpu_mdevrec), pick.data(), nullptr, out, cap, offsets, need,
        [st](const uint8_t *in, const uint8_t *, uint32_t N, uint32_t *lens) {
            k_mdev_name_len<<<(N + 1 + 255) / 256, 256, 0, st>>>((const kxpu_mdevrec *)in, N, lens);
        },
        [st](const uint8_t *in, const uint8_t *, uint32_t N, const uint32_t *offs, uint8_t *o) {
            k_mdev_name_write<<<(N + 255) / 256, 256, 0, st>>>((const kxpu_mdevrec *)in, N, offs, o);
        });
}

extern "C" int32_t kxpu_lw_encode(kxpu_ctx *ctx, const uint32_t *group_ids, const uint8_t *healthy, size_t n,
                                  uint8_t *out, size_t cap, size_t *len) {
    if (!ctx || !len || (n && !group_ids)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    if (n == 0) { *len = 0; return KXPU_OK; }
    cudaStream_t st = ctx->stream;
    return emit_items(
        ctx, n, n * 4, group_ids, healthy, out, cap, nullptr, len,
        [st](const uint8_t *in, const uint8_t *in2, uint32_t N, uint32_t *lens) {
            k_lw_len<false><<<(N + 1 + 255) / 256, 256, 0, st>>>((const uint32_t *)in, in2, nullptr, N, lens);
        },
        [st](const uint8_t *in, const uint8_t *in2, uint32_t N, const uint32_t *offs, uint8_t *o) {
            k_lw_write<false><<<(N + 255) / 256, 256, 0, st>>>((const uint32_t *)in, in2, nullptr, N, offs, o);
        });
}

extern "C" int32_t kxpu_lw_encode_topo(kxpu_ctx *ctx, const uint32_t *group_ids, const uint8_t *healthy, const uint64_t *numa_mask,
                                       size_t n, uint8_t *out, size_t cap, size_t *len) {
    if (!ctx || !len || (n && !group_ids)) return KXPU_E_INVALID;
    if (n >= 0xFFFFFFFFull / 283u) return KXPU_E_UNSUPPORTED;  // the uint32 offsets of the longest Devices
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    if (n == 0) { *len = 0; return KXPU_OK; }
    cudaStream_t st = ctx->stream;
    const uint8_t *d_masks = nullptr;  // the masks' device copy (emit_items), NULL without masks
    return emit_items(
        ctx, n, n * 4, group_ids, healthy, out, cap, nullptr, len,
        [st, &d_masks](const uint8_t *in, const uint8_t *in2, uint32_t N, uint32_t *lens) {
            k_lw_len<true><<<(N + 1 + 255) / 256, 256, 0, st>>>((const uint32_t *)in, in2, (const unsigned long long *)d_masks, N, lens);
        },
        [st, &d_masks](const uint8_t *in, const uint8_t *in2, uint32_t N, const uint32_t *offs, uint8_t *o) {
            k_lw_write<true><<<(N + 255) / 256, 256, 0, st>>>((const uint32_t *)in, in2, (const unsigned long long *)d_masks, N,
                                                             offs, o);
        },
        numa_mask, n * 8, &d_masks);
}

// ------------------------------------------------------------------ K11: DRA ResourceSlices
// a lowercase RFC 1123 DNS subdomain of at most `max` bytes: labels of [a-z0-9-], 1..63 bytes, starting and ending with
// [a-z0-9], joined by '.'
static bool dns_subdomain_ok(const char *s, size_t max) {
    if (!s) return false;
    const size_t len = strnlen(s, max + 1);
    if (len == 0 || len > max) return false;
    size_t label = 0;
    for (size_t i = 0; i <= len; i++) {
        const char c = i < len ? s[i] : '.';
        const bool alnum = (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9');
        if (c == '.') {
            if (label == 0 || label > 63 || s[i - 1] == '-') return false;
            label = 0;
        } else if (alnum || (c == '-' && label > 0)) {
            label++;
        } else {
            return false;
        }
    }
    return true;
}

// a Kubernetes name part: 1..max bytes, [A-Za-z0-9] at both ends, [-A-Za-z0-9_.] between
static bool k8s_name_ok(const char *s, size_t len, size_t max) {
    if (len == 0 || len > max) return false;
    auto alnum = [](char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9'); };
    if (!alnum(s[0]) || !alnum(s[len - 1])) return false;
    for (size_t i = 0; i < len; i++)
        if (!alnum(s[i]) && s[i] != '-' && s[i] != '_' && s[i] != '.') return false;
    return true;
}
// a taint key: a qualified name of at most 127 bytes, [<lowercase DNS subdomain>/]<name of 1..63 bytes>
static bool taint_key_ok(const char *k) {
    if (!k) return false;
    const size_t len = strnlen(k, 128);
    if (len == 0 || len > 127) return false;
    const char *slash = (const char *)memchr(k, '/', len);
    if (!slash) return k8s_name_ok(k, len, 63);
    const size_t pl = (size_t)(slash - k);
    return pl > 0 && dns_subdomain_ok(std::string(k, pl).c_str(), 253) && k8s_name_ok(slash + 1, len - pl - 1, 63);
}
// a taint value: empty or a name of at most 63 bytes
static bool taint_value_ok(const char *v) {
    if (!v) return false;
    const size_t len = strnlen(v, 64);
    return len == 0 || k8s_name_ok(v, len, 63);
}

static bool taint_ok(const kxpu_dra_taint &t) {
    return taint_key_ok(t.key) && taint_value_ok(t.value) && t.effect &&
           (strcmp(t.effect, "NoSchedule") == 0 || strcmp(t.effect, "NoExecute") == 0);
}
// {"key":"<key>"[,"value":"<value>"],"effect":"<effect>","timeAdded":"  -- one taint up to its time
static std::string taint_entry(const kxpu_dra_taint &t) {
    std::string s = std::string("{\"key\":\"") + t.key + "\"";
    if (t.value[0]) s += std::string(",\"value\":\"") + t.value + "\"";
    return s + ",\"effect\":\"" + t.effect + "\",\"timeAdded\":\"";
}

// the taint arguments of the _taint (one entry) and _taints calls; since == NULL: the untainted call
struct DraTaint {
    const kxpu_dra_taint *table;
    size_t n;
    const int64_t *since;  // [devices * n]
};

// kxpu_dra_slices[_mdev][_taint[s]]: the argument checks, the pool (literals | taint parts | head | tail), one
// k_dra_slices<LAYOUT, NT> launch, the domain flags and the copies
template <int LAYOUT, int NT = 0>
static int32_t dra_slices(kxpu_ctx *ctx, const char *what, const char *driver, const char *pool, const char *node,
                          uint64_t generation, const typename DraLayout<LAYOUT>::Rec *devs, size_t n, uint8_t *out, size_t cap,
                          size_t *len, uint64_t *slice_off, size_t *n_slices, const DraTaint taint = DraTaint{}) {
    using Rec = typename DraLayout<LAYOUT>::Rec;
    using K = DraKernel<LAYOUT, NT>;
    constexpr bool TAINT = K::TAINT;
    constexpr int PARTS = K::PARTS, HEAD = PARTS - 2, TAIL = PARTS - 1;
    constexpr int LITS = LAYOUT == LAYOUT_PCI ? 9 : DRAM_LITS;
    constexpr int MAXF = K::MAXF;
    constexpr int F_COUNT = K::F_COUNT;
    const char *const *lits = LAYOUT == LAYOUT_PCI ? h_dra_lits : h_dram_lits;
    if (!ctx || !len || !n_slices || (n && !devs)) return KXPU_E_INVALID;
    if (!dns_subdomain_ok(driver, 63) || !dns_subdomain_ok(pool, 253) || !dns_subdomain_ok(node, 253) ||
        generation >= (1ull << 63)) {
        KX_SET_ERR(ctx, "%s: driver (<= 63 bytes), pool and node (<= 253 bytes) must be lowercase DNS subdomains "
                        "and generation below 2^63", what);
        return KXPU_E_INVALID;
    }
    // callers see the bound of the NT = KXPU_DRA_MAX_TAINTS instantiation, which gets every table but the one-entry one
    if (TAINT && (!taint.table || taint.n == 0 || taint.n > (size_t)NT)) {
        KX_SET_ERR(ctx, "%s: taints must hold 1..%d entries", what, KXPU_DRA_MAX_TAINTS);
        return KXPU_E_INVALID;
    }
    for (size_t t = 0; TAINT && t < taint.n; t++)
        if (!taint_ok(taint.table[t])) {
            KX_SET_ERR(ctx, "%s: taint %zu: the key must be a qualified name of at most 127 bytes, the value empty or a "
                            "label value and the effect NoSchedule or NoExecute", what, t);
            return KXPU_E_INVALID;
        }
    if (n >= KXPU_DRA_MAX_DEVICES) {
        KX_SET_ERR(ctx, "%s: n = %zu is not below %u", what, n, KXPU_DRA_MAX_DEVICES);
        return KXPU_E_UNSUPPORTED;
    }
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    const uint32_t N = (uint32_t)n, slices = N ? (N + K::T - 1) / K::T : 1u;
    const std::string d = driver, p = pool, nd = node;
    const std::string head = "{\"kind\":\"ResourceSlice\",\"apiVersion\":\"resource.k8s.io/v1\",\"metadata\":{\"generateName\":\"" +
                             nd + "-" + d + "-\"},\"spec\":{\"driver\":\"" + d + "\",\"pool\":{\"name\":\"" + p +
                             "\",\"generation\":" + std::to_string(generation) +
                             ",\"resourceSliceCount\":" + std::to_string(slices) + "},\"nodeName\":\"" + nd +
                             "\",\"devices\":[";
    // the taint parts, from part LITS on: KX_TAINTS_OPEN, NT entry heads (empty past the table), KX_TAINT_ECLOSE and
    // KX_TAINTS_CLOSE
    std::vector<std::string> taint_parts;
    if constexpr (TAINT) {
        taint_parts.push_back(KX_TAINTS_OPEN);
        for (size_t t = 0; t < (size_t)NT; t++) taint_parts.push_back(t < taint.n ? taint_entry(taint.table[t]) : "");
        taint_parts.push_back(KX_TAINT_ECLOSE);
        taint_parts.push_back(KX_TAINTS_CLOSE);
    }
    typename K::Params E;
    memset(&E, 0, sizeof E);
    uint32_t acc = 0;
    for (int k = 0; k < PARTS; k++) {
        const std::string s = k < LITS ? std::string(lits[k]) : k == HEAD ? head : k == TAIL ? std::string(KX_DRA_TAIL)
                                                                                  : taint_parts[k - LITS];
        if (acc + s.size() > (size_t)K::POOL) return KXPU_E_INVALID;  // the literals grew: the pool bound must follow
        memcpy(E.pool + acc, s.data(), s.size());
        E.off[k] = (uint16_t)acc;
        E.len[k] = (uint16_t)s.size();
        acc += E.len[k];
    }
    E.pool_len = acc;
    const size_t bound = (size_t)slices * (E.len[HEAD] + E.len[TAIL]) + (size_t)n * MAXF + 64;
    const size_t smem = sizeof(typename K::Smem);
    static bool attr_done = false;
    if (!attr_done) {
        cudaFuncSetAttribute(k_dra_slices<LAYOUT, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        attr_done = true;
    }
    KxScratch sc(ctx);
    Rec *d_devs = nullptr;
    uint8_t *d_out = nullptr;
    unsigned long long *d_ctl = nullptr;  // slice_off [slices + 1] | F_COUNT flag words
    const size_t ctl_words = slices + 1 + (F_COUNT + 1) / 2;
    KX_CUDA(ctx, sc.alloc((void **)&d_devs, n * sizeof(Rec)));
    KX_CUDA(ctx, sc.alloc((void **)&d_out, bound));
    KX_CUDA(ctx, sc.alloc((void **)&d_ctl, ctl_words * 8));
    if (n) cudaMemcpyAsync(d_devs, devs, n * sizeof(Rec), cudaMemcpyHostToDevice, ctx->stream);
    cudaMemsetAsync(d_ctl + slices + 1, 0, (ctl_words - slices - 1) * 8, ctx->stream);
    E.devs = d_devs; E.n = N; E.out = d_out; E.slice_off = d_ctl; E.flags = (uint32_t *)(d_ctl + slices + 1);
    if constexpr (TAINT) {
        long long *d_since = nullptr;
        KX_CUDA(ctx, sc.alloc((void **)&d_since, n * taint.n * sizeof(long long)));
        if (n) cudaMemcpyAsync(d_since, taint.since, n * taint.n * sizeof(long long), cudaMemcpyHostToDevice, ctx->stream);
        E.since = d_since;
        E.nt = (uint32_t)taint.n;
        for (size_t t = 0; t < taint.n; t++)
            for (size_t j = 0; j < t; j++)
                if (strcmp(taint.table[t].key, taint.table[j].key) == 0 && strcmp(taint.table[t].effect, taint.table[j].effect) == 0)
                    E.dup[t] |= (uint8_t)(1u << j);
    }
    E.state = kx_scan_state(ctx, slices);
    if (!E.state) return KXPU_E_NOMEM;
    E.epoch = kx_next_epoch(ctx);
    {
        KxTimer tm(ctx, KXPU_T_EMIT);
        k_dra_slices<LAYOUT, NT><<<slices, EMIT_THREADS, smem, ctx->stream>>>(E);
        KX_LAUNCHED(ctx);
    }
    std::vector<unsigned long long> h(ctl_words);
    cudaMemcpyAsync(h.data(), d_ctl, ctl_words * 8, cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    static const char *const why_pci[DRA_F_COUNT] = {
        "a product byte outside [A-Za-z0-9_.-]", "a bdf that is empty or holds a byte outside [0-9a-f:.]",
        "a pcie_root that is not \"pci\" followed by [0-9a-f:]", "a vendor id that is not 1..6 bytes of [0-9a-f]",
        "a device id that is not 1..6 bytes of [0-9a-f]", "iommu_group 4294967295", "product_len above 64"};
    static const char *const why_mdev[DRAM_F_COUNT] = {
        "a product byte outside [A-Za-z0-9_.-]", "an mdev_type that is empty or holds a byte outside [A-Za-z0-9_.-]",
        "a uuid outside the canonical lowercase 8-4-4-4-12 form", "a parent that is empty or holds a byte outside [0-9a-f:.]",
        "a pcie_root that is not \"pci\" followed by [0-9a-f:]", "a vendor id that is not 1..6 bytes of [0-9a-f]",
        "a device id that is not 0..6 bytes of [0-9a-f]", "iommu_group 4294967295", "product_len above 64"};
    const char *const *why = LAYOUT == LAYOUT_PCI ? why_pci : why_mdev;
    const uint32_t *flags = reinterpret_cast<const uint32_t *>(h.data() + slices + 1);
    for (int f = 0; f < F_COUNT; f++)
        if (flags[f]) {
            KX_SET_ERR(ctx, "%s: %s", what,
                       f == K::F_SINCE ? "a taint_since above 253402300799 (9999-12-31T23:59:59Z)"
                       : f == K::F_DUP ? "a device carries two taints with the same key and effect"
                                       : why[f]);
            return KXPU_E_UNSUPPORTED;
        }
    const size_t total = (size_t)h[slices];
    *len = total;
    *n_slices = slices;
    if (cap < total || !out) return KXPU_E_NOSPACE;
    cudaMemcpyAsync(out, d_out, total, cudaMemcpyDeviceToHost, ctx->stream);
    e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s D2H failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (slice_off) memcpy(slice_off, h.data(), (slices + 1) * sizeof(uint64_t));
    return KXPU_OK;
}

extern "C" int32_t kxpu_dra_slices(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node, uint64_t generation,
                                   const kxpu_dradev *devs, size_t n, uint8_t *out, size_t cap, size_t *len,
                                   uint64_t *slice_off, size_t *n_slices) {
    static_assert(sizeof(kxpu_dradev) == 128 && offsetof(kxpu_dradev, numa_mask) == 112 &&
                      offsetof(kxpu_dradev, product_len) == 124, "kxpu_dradev layout");
    return dra_slices<LAYOUT_PCI>(ctx, "dra_slices", driver, pool, node, generation, devs, n, out, cap, len, slice_off, n_slices);
}

extern "C" int32_t kxpu_dra_slices_mdev(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node,
                                        uint64_t generation, const kxpu_dramdev *devs, size_t n, uint8_t *out, size_t cap,
                                        size_t *len, uint64_t *slice_off, size_t *n_slices) {
    static_assert(sizeof(kxpu_dramdev) == 208 && alignof(kxpu_dramdev) == 8 && offsetof(kxpu_dramdev, mdev_type) == 64 &&
                      offsetof(kxpu_dramdev, uuid) == 104 && offsetof(kxpu_dramdev, iommu_group) == 140 &&
                      offsetof(kxpu_dramdev, parent) == 144 && offsetof(kxpu_dramdev, pcie_root) == 160 &&
                      offsetof(kxpu_dramdev, vendor) == 176 && offsetof(kxpu_dramdev, numa_mask) == 192 &&
                      offsetof(kxpu_dramdev, product_len) == 200,
                  "kxpu_dramdev layout");
    return dra_slices<LAYOUT_MDEV>(ctx, "dra_slices_mdev", driver, pool, node, generation, devs, n, out, cap, len, slice_off,
                                   n_slices);
}

// kxpu_dra_slices[_mdev]_taint[s]: taint_since == NULL runs the untainted call with the taint arguments unread, one
// entry the kernel sized for one taint, any other count the one sized for KXPU_DRA_MAX_TAINTS; dra_slices checks the
// table before either instantiation reads it
template <int LAYOUT>
static int32_t dra_slices_tainted(kxpu_ctx *ctx, const char *what, const char *driver, const char *pool, const char *node,
                                  uint64_t generation, const typename DraLayout<LAYOUT>::Rec *devs, size_t n,
                                  const kxpu_dra_taint *taints, size_t n_taints, const int64_t *taint_since, uint8_t *out,
                                  size_t cap, size_t *len, uint64_t *slice_off, size_t *n_slices) {
    if (!taint_since)
        return dra_slices<LAYOUT>(ctx, LAYOUT == LAYOUT_PCI ? "dra_slices" : "dra_slices_mdev", driver, pool, node, generation,
                                  devs, n, out, cap, len, slice_off, n_slices);
    const DraTaint taint{taints, n_taints, taint_since};
    if (n_taints == 1)
        return dra_slices<LAYOUT, 1>(ctx, what, driver, pool, node, generation, devs, n, out, cap, len, slice_off, n_slices,
                                     taint);
    return dra_slices<LAYOUT, KXPU_DRA_MAX_TAINTS>(ctx, what, driver, pool, node, generation, devs, n, out, cap, len,
                                                   slice_off, n_slices, taint);
}

extern "C" int32_t kxpu_dra_slices_taint(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node,
                                         uint64_t generation, const kxpu_dradev *devs, size_t n, const char *taint_key,
                                         const char *taint_value, const char *taint_effect, const int64_t *taint_since,
                                         uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off, size_t *n_slices) {
    const kxpu_dra_taint t{taint_key, taint_value, taint_effect};
    return dra_slices_tainted<LAYOUT_PCI>(ctx, "dra_slices_taint", driver, pool, node, generation, devs, n, &t, 1, taint_since,
                                          out, cap, len, slice_off, n_slices);
}

extern "C" int32_t kxpu_dra_slices_mdev_taint(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node,
                                              uint64_t generation, const kxpu_dramdev *devs, size_t n, const char *taint_key,
                                              const char *taint_value, const char *taint_effect, const int64_t *taint_since,
                                              uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off, size_t *n_slices) {
    const kxpu_dra_taint t{taint_key, taint_value, taint_effect};
    return dra_slices_tainted<LAYOUT_MDEV>(ctx, "dra_slices_mdev_taint", driver, pool, node, generation, devs, n, &t, 1,
                                           taint_since, out, cap, len, slice_off, n_slices);
}

extern "C" int32_t kxpu_dra_slices_taints(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node,
                                          uint64_t generation, const kxpu_dradev *devs, size_t n, const kxpu_dra_taint *taints,
                                          size_t n_taints, const int64_t *taint_since, uint8_t *out, size_t cap, size_t *len,
                                          uint64_t *slice_off, size_t *n_slices) {
    return dra_slices_tainted<LAYOUT_PCI>(ctx, "dra_slices_taints", driver, pool, node, generation, devs, n, taints, n_taints,
                                          taint_since, out, cap, len, slice_off, n_slices);
}

extern "C" int32_t kxpu_dra_slices_mdev_taints(kxpu_ctx *ctx, const char *driver, const char *pool, const char *node,
                                               uint64_t generation, const kxpu_dramdev *devs, size_t n,
                                               const kxpu_dra_taint *taints, size_t n_taints, const int64_t *taint_since,
                                               uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off, size_t *n_slices) {
    return dra_slices_tainted<LAYOUT_MDEV>(ctx, "dra_slices_mdev_taints", driver, pool, node, generation, devs, n, taints,
                                           n_taints, taint_since, out, cap, len, slice_off, n_slices);
}
