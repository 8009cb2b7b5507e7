/*
 * mdev_pf_oracle.c -- CPU checker of the calls for mdev vGPUs on SR-IOV VFs (include/kxpu.h, additions to ABI v14), the
 * C statement next to the Python one (tests/pyref_mdev_pf.py):
 *   kxm_mdev_pf               kxpu_mdev_pf
 *   kxm_dra_slices_mdev_pf    kxpu_dra_slices_mdev_pf
 * TEST INFRASTRUCTURE ONLY: tests/mdev_pf_oracle.py compiles it into a temporary directory.  Restated one item at a time
 * with none of the GPU's structure: the join sorts the PCI addresses once and searches them; the slices are written one
 * device at a time with snprintf into a growing buffer (no literal pool, no tiles, no scan), and timeAdded comes from
 * gmtime_r.  kxm_dra_slices_mdev_pf returns the product call's status codes; on KXPU_E_UNSUPPORTED *why is the index of
 * the first rule the first record outside the domain breaks: the header's record rules in order, then taint_since,
 * then a duplicate taint.
 */
#define _POSIX_C_SOURCE 200809L
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "kxpu.h"

/* ---------------------------------------------------------------- kxpu_mdev_pf */

static int hexv(char c) { return (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : -1; }

/* a 16-byte field whose text before its first NUL is "dddd:bb:dd.f" in lowercase hex, device <= 1f, function 0..7 */
static int canonical(const char f[16], uint32_t *key) {
    size_t len = 0;
    while (len < 16 && f[len]) len++;
    if (len != 12 || f[4] != ':' || f[7] != ':' || f[10] != '.') return 0;
    uint32_t v[3] = {0, 0, 0};
    const int at[3] = {0, 5, 8}, w[3] = {4, 2, 2};
    for (int p = 0; p < 3; p++)
        for (int k = 0; k < w[p]; k++) {
            const int d = hexv(f[at[p] + k]);
            if (d < 0) return 0;
            v[p] = v[p] << 4 | (uint32_t)d;
        }
    if (v[2] > 0x1f || f[11] < '0' || f[11] > '7') return 0;
    *key = v[0] << 16 | v[1] << 8 | v[2] << 3 | (uint32_t)(f[11] - '0');
    return 1;
}

typedef struct { uint32_t key, idx; } addr_t;

static int addr_cmp(const void *a, const void *b) {
    const addr_t *x = a, *y = b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->idx < y->idx ? -1 : x->idx > y->idx;
}

void kxm_mdev_pf(const kxpu_devrec *recs, size_t n, const kxpu_mdevrec *mrecs, const kxpu_sriovrec *msrs, size_t m,
                 uint32_t *pf_of) {
    addr_t *addrs = malloc((n + 1) * sizeof *addrs);
    if (!addrs) abort();
    size_t na = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t k;
        if (canonical(recs[i].bdf, &k)) addrs[na++] = (addr_t){k, (uint32_t)i};
    }
    qsort(addrs, na, sizeof *addrs, addr_cmp);
    for (size_t i = 0; i < m; i++) {
        pf_of[i] = KXPU_NO_PF;
        uint32_t k;
        if ((msrs[i].flags & KXPU_SR_PHYSFN_ERR) || !canonical(msrs[i].physfn, &k)) continue;
        if (strncmp(msrs[i].physfn, mrecs[i].parent, 16) == 0) continue;  /* a parent never resolves to itself */
        size_t lo = 0, hi = na;  /* the first entry with this key: the lowest index */
        while (lo < hi) {
            const size_t mid = (lo + hi) / 2;
            if (addrs[mid].key < k) lo = mid + 1;
            else hi = mid;
        }
        if (lo < na && addrs[lo].key == k) pf_of[i] = addrs[lo].idx;
    }
    free(addrs);
}

/* ---------------------------------------------------------------- kxpu_dra_slices_mdev_pf */

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
static int hex(char c) { return hexv(c) >= 0; }
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

static int uuid_ok(const char u[36]) {
    for (int k = 0; k < 36; k++) {
        const int dash = k == 8 || k == 13 || k == 18 || k == 23;
        if (dash ? u[k] != '-' : !hex(u[k])) return 0;
    }
    return 1;
}

/* 0 = in the domain, else 1 + the index of the first failing rule: product, mdev_type, uuid, parent, pcie_root, vendor,
 * device, iommu_group, product_len, physfn, physfn_device */
static int record_why(const kxpu_dramdevpf *r) {
    const kxpu_dramdev *d = &r->dev;
    if (d->product_len <= 64 && !all_of((const char *)d->product, 0, d->product_len, name_byte)) return 1;
    const size_t tl = strnlen(d->mdev_type, 40);
    if (tl == 0 || !all_of(d->mdev_type, 0, tl, name_byte)) return 2;
    if (!uuid_ok(d->uuid)) return 3;
    const size_t bl = strnlen(d->parent, 16);
    if (bl == 0 || !all_of(d->parent, 0, bl, addr_byte)) return 4;
    const size_t rl = strnlen(d->pcie_root, 16);
    if (rl && (rl < 4 || memcmp(d->pcie_root, "pci", 3) != 0)) return 5;
    for (size_t k = 3; rl && k < rl; k++)
        if (!hex(d->pcie_root[k]) && d->pcie_root[k] != ':') return 5;
    const size_t vl = strnlen(d->vendor, 8), dl = strnlen(d->device, 8);
    if (vl == 0 || vl > 6 || !all_of(d->vendor, 0, vl, hex)) return 6;
    if (dl > 6 || !all_of(d->device, 0, dl, hex)) return 7;
    if (d->iommu_group == 0xFFFFFFFFu) return 8;
    if (d->product_len > 64) return 9;
    const size_t xl = strnlen(r->physfn, 16), yl = strnlen(r->physfn_device, 8);
    if (!all_of(r->physfn, 0, xl, addr_byte)) return 10;
    if (yl > 6 || (yl && !xl) || !all_of(r->physfn_device, 0, yl, hex)) return 11;
    return 0;
}
#define N_RULES 11

static void put_str(buf_t *b, const char *key, const char *val, size_t l) {
    put(b, ",\"%s\":{\"string\":\"", key);
    putn(b, val, l);
    putn(b, "\"}", 2);
}

/* {"name":"vfio<g>","attributes":{...}  without the device's closing '}' */
static void put_device(buf_t *b, const kxpu_dramdevpf *r) {
    const kxpu_dramdev *d = &r->dev;
    put(b, "{\"name\":\"vfio%u\",\"attributes\":{\"iommuGroup\":{\"int\":%u}", d->iommu_group, d->iommu_group);
    put_str(b, "mdevType", d->mdev_type, strnlen(d->mdev_type, 40));
    if (d->numa_mask && !(d->numa_mask & (d->numa_mask - 1))) put(b, ",\"numaNode\":{\"int\":%d}", __builtin_ctzll(d->numa_mask));
    put_str(b, "parentAddress", d->parent, strnlen(d->parent, 16));
    if (d->device[0]) put_str(b, "parentDeviceID", d->device, strnlen(d->device, 8));
    put_str(b, "parentVendorID", d->vendor, strnlen(d->vendor, 8));
    if (r->physfn[0]) put_str(b, "physfnAddress", r->physfn, strnlen(r->physfn, 16));
    if (r->physfn_device[0]) put_str(b, "physfnDeviceID", r->physfn_device, strnlen(r->physfn_device, 8));
    if (d->product_len) put_str(b, "productName", (const char *)d->product, d->product_len);
    if (d->pcie_root[0]) put_str(b, "resource.kubernetes.io/pcieRoot", d->pcie_root, strnlen(d->pcie_root, 16));
    put_str(b, "uuid", d->uuid, 36);
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

int32_t kxm_dra_slices_mdev_pf(const char *driver, const char *pool, const char *node, uint64_t generation,
                               const kxpu_dramdevpf *devs, size_t n, const kxpu_dra_taint *tab, size_t nt,
                               const int64_t *since, uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off,
                               size_t *n_slices, int32_t *why) {
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
