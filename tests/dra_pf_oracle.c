/*
 * dra_pf_oracle.c -- CPU checker of kxpu_dra_slices_pf (include/kxpu.h, addition to ABI v14), the C statement next to
 * the Python one (tests/pyref_dra_pf.py).
 * TEST INFRASTRUCTURE ONLY: tests/dra_pf_oracle.py compiles it into a temporary directory.  Restated one device at a
 * time with none of the GPU's structure: the slices are written with snprintf into a growing buffer (no literal pool,
 * no tiles, no scan), and timeAdded comes from gmtime_r.  kxd_dra_slices_pf returns the product call's status codes; on
 * KXPU_E_UNSUPPORTED *why is the index of the first rule the first record outside the domain breaks: the header's
 * record rules in order, then taint_since, then a duplicate taint.
 */
#define _POSIX_C_SOURCE 200809L
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "kxpu.h"

typedef struct { uint8_t *p; size_t len, cap; } buf_t;

static void grow(buf_t *b, size_t k) {
    if (b->len + k <= b->cap) return;
    size_t cap = b->cap ? b->cap : 4096;
    while (cap < b->len + k) cap *= 2;
    b->p = realloc(b->p, cap);
    if (!b->p) abort();
    b->cap = cap;
}
static void putn(buf_t *b, const char *s, size_t k) {
    grow(b, k);
    memcpy(b->p + b->len, s, k);
    b->len += k;
}
static void put(buf_t *b, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
static void put(buf_t *b, const char *fmt, ...) {
    char tmp[1024];
    va_list ap;
    va_start(ap, fmt);
    const int k = vsnprintf(tmp, sizeof tmp, fmt, ap);
    va_end(ap);
    if (k < 0 || (size_t)k >= sizeof tmp) abort();
    putn(b, tmp, (size_t)k);
}

static int lower_alnum(char c) { return (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9'); }
static int alnum(char c) { return lower_alnum(c) || (c >= 'A' && c <= 'Z'); }
static int name_byte(char c) { return alnum(c) || c == '_' || c == '.' || c == '-'; }
static int hex(char c) { return (c >= '0' && c <= '9') || (c >= 'a' && c <= 'f'); }
static int addr_byte(char c) { return hex(c) || c == ':' || c == '.'; }

static int subdomain_ok(const char *s, size_t max) {
    if (!s) return 0;
    const size_t len = strnlen(s, max + 1);
    if (len == 0 || len > max) return 0;
    size_t start = 0;
    while (start <= len) {
        const char *dot = memchr(s + start, '.', len - start);
        const size_t end = dot ? (size_t)(dot - s) : len, l = end - start;
        if (l == 0 || l > 63 || !lower_alnum(s[start]) || !lower_alnum(s[end - 1])) return 0;
        for (size_t i = start; i < end; i++)
            if (!lower_alnum(s[i]) && s[i] != '-') return 0;
        start = end + 1;
    }
    return 1;
}

static int k8s_name(const char *s, size_t len, size_t max) {
    if (len == 0 || len > max) return 0;
    for (size_t i = 0; i < len; i++)
        if (!alnum(s[i]) && (i == 0 || i == len - 1 || (s[i] != '-' && s[i] != '_' && s[i] != '.'))) return 0;
    return 1;
}

static int taint_ok(const kxpu_dra_taint *t) {
    if (!t->key || !t->value || !t->effect) return 0;
    const size_t kl = strnlen(t->key, 128);
    if (kl == 0 || kl > 127) return 0;
    const char *slash = memchr(t->key, '/', kl);
    if (slash) {
        char prefix[128];
        const size_t pl = (size_t)(slash - t->key);
        memcpy(prefix, t->key, pl);
        prefix[pl] = 0;
        if (!subdomain_ok(prefix, 253) || !k8s_name(slash + 1, kl - pl - 1, 63)) return 0;
    } else if (!k8s_name(t->key, kl, 63)) {
        return 0;
    }
    const size_t vl = strnlen(t->value, 64);
    if (vl && !k8s_name(t->value, vl, 63)) return 0;
    return strcmp(t->effect, "NoSchedule") == 0 || strcmp(t->effect, "NoExecute") == 0;
}

static int all_of(const char *s, size_t from, size_t len, int (*ok)(char)) {
    for (size_t k = from; k < len; k++)
        if (!ok(s[k])) return 0;
    return 1;
}

/* 0 = in the domain, else 1 + the index of the first failing rule: product, bdf, pcie_root, vendor, device,
 * iommu_group, product_len, physfn, physfn_device */
static int record_why(const kxpu_dradevpf *r) {
    const kxpu_dradev *d = &r->dev;
    if (d->product_len <= 64 && !all_of((const char *)d->product, 0, d->product_len, name_byte)) return 1;
    const size_t bl = strnlen(d->bdf, 16);
    if (bl == 0 || !all_of(d->bdf, 0, bl, addr_byte)) return 2;
    const size_t rl = strnlen(d->pcie_root, 16);
    if (rl && (rl < 4 || memcmp(d->pcie_root, "pci", 3) != 0)) return 3;
    for (size_t k = 3; rl && k < rl; k++)
        if (!hex(d->pcie_root[k]) && d->pcie_root[k] != ':') return 3;
    const size_t vl = strnlen(d->vendor, 8), dl = strnlen(d->device, 8);
    if (vl == 0 || vl > 6 || !all_of(d->vendor, 0, vl, hex)) return 4;
    if (dl == 0 || dl > 6 || !all_of(d->device, 0, dl, hex)) return 5;
    if (d->iommu_group == 0xFFFFFFFFu) return 6;
    if (d->product_len > 64) return 7;
    const size_t xl = strnlen(r->physfn, 16), yl = strnlen(r->physfn_device, 8);
    if (!all_of(r->physfn, 0, xl, addr_byte)) return 8;
    if (yl > 6 || (yl && !xl) || !all_of(r->physfn_device, 0, yl, hex)) return 9;
    return 0;
}
#define N_RULES 9

static void put_str(buf_t *b, const char *key, const char *val, size_t l) {
    put(b, ",\"%s\":{\"string\":\"", key);
    putn(b, val, l);
    putn(b, "\"}", 2);
}

/* {"name":"vfio<g>","attributes":{...}  without the device's closing '}' */
static void put_device(buf_t *b, const kxpu_dradevpf *r) {
    const kxpu_dradev *d = &r->dev;
    put(b, "{\"name\":\"vfio%u\",\"attributes\":{\"deviceID\":{\"string\":\"", d->iommu_group);
    putn(b, d->device, strnlen(d->device, 8));
    put(b, "\"},\"iommuGroup\":{\"int\":%u}", d->iommu_group);
    if (d->numa_mask && !(d->numa_mask & (d->numa_mask - 1))) put(b, ",\"numaNode\":{\"int\":%d}", __builtin_ctzll(d->numa_mask));
    put_str(b, "pciAddress", d->bdf, strnlen(d->bdf, 16));
    if (r->physfn[0]) put_str(b, "physfnAddress", r->physfn, strnlen(r->physfn, 16));
    if (r->physfn_device[0]) put_str(b, "physfnDeviceID", r->physfn_device, strnlen(r->physfn_device, 8));
    if (d->product_len) put_str(b, "productName", (const char *)d->product, d->product_len);
    if (d->pcie_root[0]) put_str(b, "resource.kubernetes.io/pcieRoot", d->pcie_root, strnlen(d->pcie_root, 16));
    put_str(b, "vendorID", d->vendor, strnlen(d->vendor, 8));
    put(b, "}");
}

/* ,"taints":[...] of one device */
static void put_taints(buf_t *b, const kxpu_dra_taint *tab, size_t nt, const int64_t *row) {
    int first = 1;
    put(b, ",\"taints\":[");
    for (size_t t = 0; t < nt; t++) {
        if (row[t] < 0) continue;
        struct tm tm;
        const time_t tt = (time_t)row[t];
        gmtime_r(&tt, &tm);
        put(b, "%s{\"key\":\"%s\"", first ? "" : ",", tab[t].key);
        if (tab[t].value[0]) put(b, ",\"value\":\"%s\"", tab[t].value);
        put(b, ",\"effect\":\"%s\",\"timeAdded\":\"%04d-%02d-%02dT%02d:%02d:%02dZ\"}", tab[t].effect, tm.tm_year + 1900,
            tm.tm_mon + 1, tm.tm_mday, tm.tm_hour, tm.tm_min, tm.tm_sec);
        first = 0;
    }
    put(b, "]");
}

int32_t kxd_dra_slices_pf(const char *driver, const char *pool, const char *node, uint64_t generation,
                          const kxpu_dradevpf *devs, size_t n, const kxpu_dra_taint *tab, size_t nt, const int64_t *since,
                          uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off, size_t *n_slices, int32_t *why) {
    if (!len || !n_slices || (n && !devs)) return KXPU_E_INVALID;
    if (!subdomain_ok(driver, 63) || !subdomain_ok(pool, 253) || !subdomain_ok(node, 253) || generation >= (1ull << 63))
        return KXPU_E_INVALID;
    if (since) {
        if (!tab || nt == 0 || nt > KXPU_DRA_MAX_TAINTS) return KXPU_E_INVALID;
        for (size_t t = 0; t < nt; t++)
            if (!taint_ok(&tab[t])) return KXPU_E_INVALID;
    }
    if (n >= KXPU_DRA_MAX_DEVICES) return KXPU_E_UNSUPPORTED;
    for (size_t i = 0; i < n; i++) {
        int w = record_why(&devs[i]);
        for (size_t t = 0; since && !w && t < nt; t++)
            if (since[i * nt + t] > KXPU_DRA_TAINT_SINCE_MAX) w = N_RULES + 1;
        for (size_t t = 0; since && !w && t < nt; t++)
            for (size_t j = 0; !w && j < t; j++)
                if (since[i * nt + t] >= 0 && since[i * nt + j] >= 0 && strcmp(tab[t].key, tab[j].key) == 0 &&
                    strcmp(tab[t].effect, tab[j].effect) == 0)
                    w = N_RULES + 2;
        if (w) {
            if (why) *why = w - 1;
            return KXPU_E_UNSUPPORTED;
        }
    }
    const size_t per = since ? KXPU_DRA_TAINT_SLICE_DEVICES : KXPU_DRA_SLICE_DEVICES;
    const size_t slices = n ? (n + per - 1) / per : 1;
    buf_t b = {0, 0, 0};
    uint64_t *offs = malloc((slices + 1) * sizeof(uint64_t));
    if (!offs) abort();
    for (size_t s = 0; s < slices; s++) {
        offs[s] = b.len;
        put(&b, "{\"kind\":\"ResourceSlice\",\"apiVersion\":\"resource.k8s.io/v1\",\"metadata\":{\"generateName\":\"%s-%s-\"},",
            node, driver);
        put(&b, "\"spec\":{\"driver\":\"%s\",\"pool\":{\"name\":\"%s\",", driver, pool);
        put(&b, "\"generation\":%llu,\"resourceSliceCount\":%zu},\"nodeName\":\"%s\",\"devices\":[",
            (unsigned long long)generation, slices, node);
        const size_t end = (s + 1) * per < n ? (s + 1) * per : n;
        for (size_t i = s * per; i < end; i++) {
            if (i > s * per) put(&b, ",");
            put_device(&b, &devs[i]);
            int any = 0;
            for (size_t t = 0; since && t < nt; t++) any |= since[i * nt + t] >= 0;
            if (any) put_taints(&b, tab, nt, since + i * nt);
            put(&b, "}");
        }
        put(&b, "]}}\n");
    }
    offs[slices] = b.len;
    *len = b.len;
    *n_slices = slices;
    int32_t rc = KXPU_OK;
    if (!out || cap < b.len) rc = KXPU_E_NOSPACE;
    else {
        memcpy(out, b.p, b.len);
        if (slice_off) memcpy(slice_off, offs, (slices + 1) * sizeof(uint64_t));
    }
    free(b.p);
    free(offs);
    return rc;
}
