// cdi.cuh -- what emit.cu (the CDI spec emitter) offers to cdi_parse.cu (its inverse).  Not part of the ABI.
#pragma once
#include <string>

#include "common.cuh"

// kxpu_cdi_emit_kind's kind domain (include/kxpu.h)
bool kx_cdi_kind_ok(const char *kind);
// part k of a document's template for this format / layout and kind: 0-5 the per-device literals (4 of the mdev layout is
// the mdev annotation's opening), 6 the head, 7 the tail, 8 the whole zero-device document, 9 the literal after the mdev
// uuid (empty for the PCI layout)
std::string kx_cdi_part(int32_t format, bool mdev, int k, const char *kind);
// Enqueues the emit of n >= 1 device-resident records (kxpu_cdidev, or kxpu_mdevcdi when mdev) on the ctx stream with
// the emitter's own kernel: *d_out (scratch of sc) gets the document, (*d_total)[0] its length and (*d_total)[1] the
// flags word (low half: a bdf outside [0-9a-f:.], high half: a uuid outside the canonical form).  timed: the launch is
// recorded under KXPU_T_EMIT.
int32_t kx_cdi_emit_enqueue(kxpu_ctx *ctx, int32_t format, const char *kind, const void *d_devs, size_t n, bool mdev,
                            KxScratch &sc, uint8_t **d_out, unsigned long long **d_total, bool timed);
