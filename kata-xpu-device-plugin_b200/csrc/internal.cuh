// internal.cuh -- what api.cu (table life cycle, parse / finalize / join launches) offers to
// comm.cu (sharded load).  Not part of the ABI.
#pragma once
#include "common.cuh"
#include "exchange.cuh"
#include "table.cuh"

struct kxpu_table {
    uint32_t cap = 0, shift = 0;
    KxArena arena;
    KxTableDev dev{};
    unsigned long long *range_words = nullptr;  // parse: range_state / range_carry / lead / resolve queue
    uint32_t *row_key = nullptr;
    unsigned long long *row_line = nullptr;
    unsigned long long *row_anchor = nullptr;
    uint32_t *row_name_off = nullptr;
    uint32_t *row_name_len = nullptr;
    uint8_t *blob = nullptr;
    uint32_t blob_cap = 0;
    uint32_t rows_cap = 0;  // entries of the row arrays
    uint32_t n_rows = 0;
    uint32_t blob_used = 0;
};

#define KX_ENTER(ctx)                          \
    if (!(ctx)) return KXPU_E_INVALID;         \
    std::lock_guard<std::mutex> guard__((ctx)->mu); \
    cudaSetDevice((ctx)->device)

// A clean table arena (pooled): cap slots, blob_cap name bytes, range words for num_chunks chunks.
int32_t kx_table_acquire(kxpu_ctx *ctx, uint32_t cap, uint32_t blob_cap, uint32_t num_chunks, kxpu_table **out);
// Back to the pool; the reset kernel is enqueued here so that the next load finds it clean.
void kx_table_release(kxpu_ctx *ctx, kxpu_table *t);
uint32_t kx_initial_blob_cap(kxpu_ctx *ctx, size_t n);
// parse + resolve kernels of d_text[0..n) (global offsets base + local) into t
// xa (may be null): phase-A push of the sharded load, run by the last CTA of the resolve kernel
struct KxXaHook {
    kxx::XaParams p;
    uint32_t *done;
};
int32_t kx_launch_parse(kxpu_ctx *ctx, kxpu_table *t, const uint8_t *d_text, size_t n, unsigned long long base,
                        unsigned long long carry_in, const KxXaHook *xa);
int32_t kx_launch_trunc(kxpu_ctx *ctx, kxpu_table *t, const uint8_t *d_text, size_t n, unsigned long long base);
// slab (may be null): sharded load -- rows and names go into this rank's slab instead of the table's arrays
struct KxSlabOut {
    uint8_t *rows;
    uint32_t rows_cap;
    uint8_t *blob;
    uint32_t blob_cap;
    kxx::SlabTail tail;  // header + flags by the last CTA of the finalize
};
// mv (may be null: the table's own minima): what validity is judged against
int32_t kx_launch_finalize(kxpu_ctx *ctx, kxpu_table *t, const uint8_t *d_text, size_t n, unsigned long long base,
                           const kxx::MinView *mv, const kxx::WaitSpec *wait, const KxSlabOut *slab);
int32_t kx_launch_lookup(kxpu_ctx *ctx, kxpu_table *t, const uint32_t *d_keys, size_t n, int32_t *d_rows);
// growth policy shared by the single and the sharded load; returns false when the limit is reached
bool kx_grow_cap(uint32_t *cap, bool table_full);
void kx_note_table_size(kxpu_ctx *ctx, uint32_t nkeys, uint32_t blob_used, uint32_t blob_cap);
