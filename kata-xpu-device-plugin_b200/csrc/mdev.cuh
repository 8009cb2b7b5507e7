// mdev.cuh -- device helpers for kxpu_mdevrec / kxpu_mdevcdi shared by classify.cu (K5) and emit.cu (K6):
// the canonical-UUID test and the type key (include/kxpu.h, kxpu_classify_mdev).  Every loop is unrolled over
// constant byte positions, so the record words stay in registers.
#pragma once
#include "common.cuh"

namespace kxmdev {

constexpr uint32_t NAME_MAX_BYTES = 40;  // kxpu_mdevrec.type_name

__device__ __forceinline__ uint32_t byte_at(const uint32_t *w, uint32_t k) { return (w[k >> 2] >> (8u * (k & 3u))) & 0xffu; }

// 8-4-4-4-12 lowercase hex with '-' at 8, 13, 18, 23; w = the 36 bytes as nine little-endian words
__device__ __forceinline__ bool uuid_ok(const uint32_t w[9]) {
    bool ok = true;
#pragma unroll
    for (uint32_t k = 0; k < 36; k++) {
        const uint32_t c = byte_at(w, k);
        if (k == 8 || k == 13 || k == 18 || k == 23) ok &= c == (uint32_t)'-';
        else ok &= (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f');
    }
    return ok;
}

// The type key of name[0..len) (len <= 40; w = the 40 name bytes as ten words): trim "\t\n\v\f\r " at both ends,
// ' ' -> '_', drop bytes outside [A-Za-z0-9_.-].  put(p, c) receives key byte p; returns the key length.
template <typename Put>
__device__ __forceinline__ uint32_t type_key(const uint32_t w[10], uint32_t len, Put put) {
    uint32_t a = NAME_MAX_BYTES, b = 0;  // [a, b): the name without leading / trailing white space
#pragma unroll
    for (uint32_t k = 0; k < NAME_MAX_BYTES; k++) {
        const uint32_t c = byte_at(w, k);
        const bool ws = c == ' ' || (c >= '\t' && c <= '\r');
        if (k < len && !ws) {
            a = min(a, k);
            b = k + 1;
        }
    }
    uint32_t p = 0;
#pragma unroll
    for (uint32_t k = 0; k < NAME_MAX_BYTES; k++) {
        uint32_t c = byte_at(w, k);
        if (c == ' ') c = '_';
        const bool keep = (c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_' || c == '.' ||
                          c == '-';
        if (k >= a && k < b && keep) put(p++, (uint8_t)c);
    }
    return p;
}

}  // namespace kxmdev
