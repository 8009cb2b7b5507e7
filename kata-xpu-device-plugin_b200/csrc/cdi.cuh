// cdi.cuh -- what emit.cu (the CDI spec emitter) offers to cdi_parse.cu (its inverse).  Not part of the ABI.
#pragma once
#include <string>

#include "common.cuh"

// The document layouts, and the LAYOUT template argument of both kernels: the device records and the device node
constexpr int KX_CDI_PCI = 0;        // kxpu_cdidev, /dev/vfio/<g>
constexpr int KX_CDI_MDEV = 1;       // kxpu_mdevcdi, /dev/vfio/<g>
constexpr int KX_CDI_CDEV = 2;       // kxpu_cdidev, /dev/vfio/devices/vfio<N>
constexpr int KX_CDI_MDEV_CDEV = 3;  // kxpu_mdevcdev, /dev/vfio/devices/vfio<N>
constexpr int KX_CDI_TYPED = 4;      // kxpu_vfvgpucdi, /dev/vfio/<g>, the vgpu-type / vgpu-type-key annotations
constexpr int KX_CDI_TYPED_CDEV = 5; // kxpu_vfvgpucdi, /dev/vfio/devices/vfio<N>, the same annotations
// The longest device fragment of the first three layouts and any kind (emit.cu MAX_FRAG_MDEV), and of the mdev cdev
// layout (MAX_FRAG_MDEV_CDEV), and of the two typed layouts (MAX_FRAG_TYPED_CDEV_LONG); the parse's halo of each layout
// must hold it
constexpr int KX_CDI_FRAG_MAX = 480;
constexpr int KX_CDI_FRAG_MAX_MDEV_CDEV = KX_CDI_FRAG_MAX + 12;
constexpr int KX_CDI_FRAG_MAX_TYPED = 532;

// kxpu_cdi_emit_kind's kind domain (include/kxpu.h)
bool kx_cdi_kind_ok(const char *kind);
// part k of a document's template for this format / layout and kind: 0-5 the per-device literals (4 of the mdev layouts
// is the mdev annotation's opening, 4 of the cdev layout ends in "/dev/vfio/devices/vfio"), 6 the head, 7 the tail, 8 the
// whole zero-device document, 9 the literal after the mdev uuid (empty for the PCI layouts; it ends in
// "/dev/vfio/devices/vfio" for the mdev cdev layout).  The typed layouts: 4 opens the vgpu-type annotation, 9 is the
// literal between the type ID and the key, 10 the literal after the key (the node literal, "/dev/vfio/devices/vfio" for
// the typed cdev layout); part 10 is empty for every other layout
std::string kx_cdi_part(int32_t format, int layout, int k, const char *kind);
// Enqueues the emit of n >= 1 device-resident records (kxpu_mdevcdi for KX_CDI_MDEV, kxpu_mdevcdev for
// KX_CDI_MDEV_CDEV, kxpu_vfvgpucdi for the typed layouts, else kxpu_cdidev) on the ctx stream with the emitter's own kernel: *d_out (scratch of sc) gets the
// document, (*d_total)[0] its length and (*d_total)[1] the flags word (low half: a bdf outside [0-9a-f:.], high half: a
// uuid outside the canonical form; typed layouts: a type ID or key outside the domain).  timed: the launch is recorded under KXPU_T_EMIT.
int32_t kx_cdi_emit_enqueue(kxpu_ctx *ctx, int32_t format, const char *kind, const void *d_devs, size_t n, int layout,
                            KxScratch &sc, uint8_t **d_out, unsigned long long **d_total, bool timed);
