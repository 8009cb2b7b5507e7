// emit.cuh -- decimal formatting shared by the emitters (emit.cu) and the metrics writer (metrics.cu).
#pragma once
#include <stdint.h>

namespace kxemit {

__device__ __forceinline__ uint32_t dec_len(unsigned long long v) {
    uint32_t l = 1;
    while (v >= 10ull) { v /= 10ull; l++; }
    return l;
}
__device__ __forceinline__ void dec_write(unsigned long long v, uint32_t len, uint8_t *dst) {
    for (uint32_t k = len; k > 0; k--) { dst[k - 1] = (uint8_t)('0' + (uint32_t)(v % 10ull)); v /= 10ull; }
}

}  // namespace kxemit
