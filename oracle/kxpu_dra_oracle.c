/*
 * kxpu_dra_oracle.c -- CPU checker of kxpu_dra_slices (include/kxpu.h, ABI v9): the ResourceSlices of one DRA pool as
 * JSON Lines, written sequentially with snprintf from the rules stated in the header.
 *
 * TEST INFRASTRUCTURE ONLY, like kxpu_oracle.c.  kxo_dra_slices takes kxpu_dra_slices' arguments without the context
 * and returns the same status codes; on KXPU_E_UNSUPPORTED *why names the first rule (the order of the header's domain
 * list) that the first record outside the domain breaks.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/kxpu.h"

static int lower_alnum(char c) { return (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9'); }

/* lowercase RFC 1123 subdomain of at most max bytes */
static int subdomain_ok(const char *s, size_t max) {
    if (!s) return 0;
    size_t len = strnlen(s, max + 1);
    if (len == 0 || len > max) return 0;
    size_t start = 0;
    while (start <= len) {
        const char *dot = memchr(s + start, '.', len - start);
        size_t end = dot ? (size_t)(dot - s) : len;
        size_t l = end - start;
        if (l == 0 || l > 63 || !lower_alnum(s[start]) || !lower_alnum(s[end - 1])) return 0;
        for (size_t i = start; i < end; i++)
            if (!lower_alnum(s[i]) && s[i] != '-') return 0;
        start = end + 1;
    }
    return 1;
}

static size_t field_len(const char *f, size_t cap) {
    size_t l = 0;
    while (l < cap && f[l]) l++;
    return l;
}

static int is_hex(char c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f'); }

/* 0 = in the domain, else 1 + the index of the first failing rule: product, bdf, pcie_root, vendor, device, group,
 * product_len */
static int record_why(const kxpu_dradev *d) {
    if (d->product_len <= 64) {
        for (size_t k = 0; k < d->product_len; k++) {
            char c = (char)d->product[k];
            if (!((c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '_' || c == '.' || c == '-'))
                return 1;
        }
    }
    size_t bl = field_len(d->bdf, 16);
    if (bl == 0) return 2;
    for (size_t k = 0; k < bl; k++)
        if (!is_hex(d->bdf[k]) && d->bdf[k] != ':' && d->bdf[k] != '.') return 2;
    size_t rl = field_len(d->pcie_root, 16);
    if (rl) {
        if (rl < 4 || memcmp(d->pcie_root, "pci", 3) != 0) return 3;
        for (size_t k = 3; k < rl; k++)
            if (!is_hex(d->pcie_root[k]) && d->pcie_root[k] != ':') return 3;
    }
    const char *ids[2] = {d->vendor, d->device};
    for (int f = 0; f < 2; f++) {
        size_t l = field_len(ids[f], 8);
        if (l == 0 || l > 6) return 4 + f;
        for (size_t k = 0; k < l; k++)
            if (!is_hex(ids[f][k])) return 4 + f;
    }
    if (d->iommu_group == 0xFFFFFFFFu) return 6;
    if (d->product_len > 64) return 7;
    return 0;
}

/* growing output buffer */
typedef struct { char *p; size_t n, cap; } Buf;
static void put(Buf *b, const char *s, size_t l) {
    if (b->n + l > b->cap) {
        b->cap = (b->n + l) * 2 + 4096;
        b->p = realloc(b->p, b->cap);
    }
    memcpy(b->p + b->n, s, l);
    b->n += l;
}
static void puts_(Buf *b, const char *s) { put(b, s, strlen(s)); }

int32_t kxo_dra_slices(const char *driver, const char *pool, const char *node, uint64_t generation, const kxpu_dradev *devs,
                       size_t n, uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off, size_t *n_slices, int32_t *why) {
    if (!len || !n_slices || (n && !devs)) return KXPU_E_INVALID;
    if (!subdomain_ok(driver, 63) || !subdomain_ok(pool, 253) || !subdomain_ok(node, 253) || generation >= (1ull << 63))
        return KXPU_E_INVALID;
    if (n >= KXPU_DRA_MAX_DEVICES) return KXPU_E_UNSUPPORTED;
    for (size_t i = 0; i < n; i++) {
        int w = record_why(&devs[i]);
        if (w) {
            if (why) *why = w - 1;
            return KXPU_E_UNSUPPORTED;
        }
    }
    size_t slices = n ? (n + KXPU_DRA_SLICE_DEVICES - 1) / KXPU_DRA_SLICE_DEVICES : 1;
    Buf b = {0, 0, 0};
    uint64_t *offs = malloc((slices + 1) * sizeof(uint64_t));
    char tmp[128];
    for (size_t s = 0; s < slices; s++) {
        offs[s] = b.n;
        puts_(&b, "{\"kind\":\"ResourceSlice\",\"apiVersion\":\"resource.k8s.io/v1\",\"metadata\":{\"generateName\":\"");
        puts_(&b, node); puts_(&b, "-"); puts_(&b, driver); puts_(&b, "-\"},\"spec\":{\"driver\":\"");
        puts_(&b, driver); puts_(&b, "\",\"pool\":{\"name\":\""); puts_(&b, pool);
        snprintf(tmp, sizeof tmp, "\",\"generation\":%llu,\"resourceSliceCount\":%zu},\"nodeName\":\"",
                 (unsigned long long)generation, slices);
        puts_(&b, tmp); puts_(&b, node); puts_(&b, "\",\"devices\":[");
        size_t end = (s + 1) * KXPU_DRA_SLICE_DEVICES < n ? (s + 1) * KXPU_DRA_SLICE_DEVICES : n;
        for (size_t i = s * KXPU_DRA_SLICE_DEVICES; i < end; i++) {
            const kxpu_dradev *d = &devs[i];
            if (i > s * KXPU_DRA_SLICE_DEVICES) puts_(&b, ",");
            snprintf(tmp, sizeof tmp, "{\"name\":\"vfio%u\",\"attributes\":{\"deviceID\":{\"string\":\"", d->iommu_group);
            puts_(&b, tmp); put(&b, d->device, field_len(d->device, 8));
            snprintf(tmp, sizeof tmp, "\"},\"iommuGroup\":{\"int\":%u}", d->iommu_group);
            puts_(&b, tmp);
            if (d->numa_mask && !(d->numa_mask & (d->numa_mask - 1))) {
                int k = 0;
                while (!((d->numa_mask >> k) & 1)) k++;
                snprintf(tmp, sizeof tmp, ",\"numaNode\":{\"int\":%d}", k);
                puts_(&b, tmp);
            }
            puts_(&b, ",\"pciAddress\":{\"string\":\""); put(&b, d->bdf, field_len(d->bdf, 16)); puts_(&b, "\"}");
            if (d->product_len) {
                puts_(&b, ",\"productName\":{\"string\":\""); put(&b, (const char *)d->product, d->product_len); puts_(&b, "\"}");
            }
            if (d->pcie_root[0]) {
                puts_(&b, ",\"resource.kubernetes.io/pcieRoot\":{\"string\":\"");
                put(&b, d->pcie_root, field_len(d->pcie_root, 16));
                puts_(&b, "\"}");
            }
            puts_(&b, ",\"vendorID\":{\"string\":\""); put(&b, d->vendor, field_len(d->vendor, 8)); puts_(&b, "\"}}}");
        }
        puts_(&b, "]}}\n");
    }
    offs[slices] = b.n;
    *len = b.n;
    *n_slices = slices;
    int32_t rc = KXPU_OK;
    if (!out || cap < b.n) rc = KXPU_E_NOSPACE;
    else {
        memcpy(out, b.p, b.n);
        if (slice_off) memcpy(slice_off, offs, (slices + 1) * sizeof(uint64_t));
    }
    free(b.p);
    free(offs);
    return rc;
}
