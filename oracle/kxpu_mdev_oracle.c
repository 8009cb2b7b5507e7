/*
 * kxpu_mdev_oracle.c -- CPU restatement of vGPU (mediated device) discovery as include/kxpu.h defines it:
 * the walk of /sys/bus/mdev/devices with a (vendor, driver) rule list (kxpu_classify_mdev), the type key
 * (kxpu_mdev_names) and the CDI spec of a vGPU class in both encoders (kxpu_cdi_emit_mdev).
 *
 * TEST INFRASTRUCTURE ONLY, like kxpu_oracle.c: loaded by tests/ through oracle/mdev_oracle.py, never by the
 * product.  A sequential walk, record by record, in the shape of createIommuDeviceMap
 * (pkg/device_plugin/device_plugin.go:126-180).  The yaml.v3 base-60 predicate comes from kxpu_oracle.c and the
 * kind domain from kxpu_xpu_oracle.c, so the three oracles agree on both.
 */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/kxpu.h"
#include "kxpu_oracle.h"

/* readIDFromFileFunc :183-191; -1 for a file under 2 or over 8 bytes */
static int read_id(const uint8_t *txt, unsigned flen, uint8_t id[8]) {
    memset(id, 0, 8);
    if (flen < 2 || flen > 8) return -1;
    const uint8_t *s = txt + 2;
    int len = (int)flen - 2;
    while (len > 0 && s[0] == '\n') { s++; len--; }
    while (len > 0 && s[len - 1] == '\n') len--;
    memcpy(id, s, (size_t)len);
    return len;
}

int kxo_uuid_ok(const char *u) {
    for (int k = 0; k < 36; k++) {
        char c = u[k];
        if (k == 8 || k == 13 || k == 18 || k == 23) { if (c != '-') return 0; }
        else if (!((c >= '0' && c <= '9') || (c >= 'a' && c <= 'f'))) return 0;
    }
    return 1;
}

/* the type key of name[0..len): trim "\t\n\v\f\r " at both ends, ' ' -> '_', keep [A-Za-z0-9_.-]; returns its length */
size_t kxo_type_key(const uint8_t *name, size_t len, uint8_t *out) {
    size_t a = 0, b = len;
    while (a < b && strchr("\t\n\v\f\r ", name[a]) && name[a]) a++;
    while (b > a && strchr("\t\n\v\f\r ", name[b - 1]) && name[b - 1]) b--;
    size_t p = 0;
    for (size_t k = a; k < b; k++) {
        uint8_t c = name[k] == ' ' ? '_' : name[k];
        if ((c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_' || c == '.' || c == '-')
            out[p++] = c;
    }
    return p;
}

/* the key of a record, or 0 when its name read failed */
static size_t rec_key(const kxpu_mdevrec *r, uint8_t key[40]) {
    if ((r->flags & KXPU_REC_NAME_ERR) || r->name_len > 40) return 0;
    return kxo_type_key(r->type_name, r->name_len, key);
}

static int field_len(const char *f, size_t cap) {
    size_t l = 0;
    while (l < cap && f[l]) l++;
    for (size_t k = l; k < cap; k++) if (f[k]) return -1;
    return (int)l;
}

/* open addressing, linear probing: h[] holds the key (or its hash), v[] the value */
typedef struct { uint64_t *h; uint32_t *v; size_t cap; } omap;
static void om_init(omap *m, size_t n) {
    size_t c = 16; while (c < 2 * n + 2) c <<= 1;
    m->cap = c; m->h = (uint64_t *)malloc(c * 8); m->v = (uint32_t *)malloc(c * 4);
    memset(m->h, 0xff, c * 8);
}
static void om_free(omap *m) { free(m->h); free(m->v); }

int32_t kxo_mdev_classify(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs, size_t n,
                          kxpu_classify_out *out, uint8_t *dev_rule) {
    if (n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    for (size_t r = 0; r < n_rules; r++) {
        int vl = field_len(rules[r].vendor, 8), dl = field_len(rules[r].driver, 16);
        if (vl < 1 || vl > 6 || memchr(rules[r].vendor, '\n', (size_t)vl)) return KXPU_E_INVALID;
        if (dl < 1 || dl > 15 || memchr(rules[r].driver, '/', (size_t)dl)) return KXPU_E_INVALID;
        for (size_t q = 0; q < r; q++)
            if (strncmp(rules[q].vendor, rules[r].vendor, 8) == 0 && strncmp(rules[q].driver, rules[r].driver, 16) == 0)
                return KXPU_E_INVALID;
    }
    omap gmap, kmap, dmap;  /* group -> ordinal | key hash -> first record | (rule, first) -> entry */
    om_init(&gmap, n); om_init(&kmap, n); om_init(&dmap, n);
    uint8_t (*keys)[40] = calloc(n + 1, 40);
    uint8_t *klen = calloc(n + 1, 1);
    uint32_t *gcount = calloc(n + 1, 4), *gord = malloc((n + 1) * 4), *dcount = calloc(n + 1, 4), *g_dev = malloc((n + 1) * 4);
    uint32_t bus_index = 0, n_groups = 0, n_devids = 0;
    for (size_t i = 0; i < n; i++) {
        const kxpu_mdevrec *r = &recs[i];
        out->accept_index[i] = KXPU_REJECTED;
        if (r->flags & (KXPU_REC_IS_DIR | KXPU_REC_VENDOR_ERR | KXPU_REC_DRIVER_ERR | KXPU_REC_IOMMU_ERR)) continue;
        if (!kxo_uuid_ok(r->uuid) || r->iommu_group == 0xFFFFFFFFu) continue;
        uint8_t id[8];
        int l = read_id(r->parent_vendor_txt, r->vendor_len, id);
        if (l < 0) continue;
        int rule = -1;
        for (size_t q = 0; q < n_rules && rule < 0; q++)
            if ((size_t)l == strnlen(rules[q].vendor, 8) && memcmp(id, rules[q].vendor, (size_t)l) == 0 &&
                strncmp(r->driver, rules[q].driver, 16) == 0)
                rule = (int)q;
        if (rule < 0) continue;
        /* a candidate: intern its type key (first record with the key) */
        klen[i] = (uint8_t)rec_key(r, keys[i]);
        uint32_t first = KXPU_REJECTED;
        if (klen[i]) {
            uint64_t h = 1469598103934665603ull;
            for (int k = 0; k < klen[i]; k++) h = (h ^ keys[i][k]) * 1099511628211ull;
            h &= 0x7FFFFFFFFFFFFFFFull;
            size_t s = (size_t)(h >> 7) & (kmap.cap - 1);
            for (;;) {
                if (kmap.h[s] == ~0ull) { kmap.h[s] = h; kmap.v[s] = (uint32_t)i; first = (uint32_t)i; break; }
                uint32_t o = kmap.v[s];
                if (kmap.h[s] == h && klen[o] == klen[i] && memcmp(keys[o], keys[i], klen[i]) == 0) { first = o; break; }
                s = (s + 1) & (kmap.cap - 1);
            }
        }
        /* its group */
        size_t s = ((uint64_t)r->iommu_group * 0x9E3779B97F4A7C15ull >> 20) & (gmap.cap - 1);
        while (gmap.h[s] != ~0ull && gmap.h[s] != r->iommu_group) s = (s + 1) & (gmap.cap - 1);
        if (gmap.h[s] == ~0ull) {
            if (!klen[i]) continue;  /* a group starts only at a record with a type key */
            gmap.h[s] = r->iommu_group; gmap.v[s] = n_groups;
            uint64_t dk = ((uint64_t)rule << 48) | first;
            size_t t = (size_t)(dk * 0x9E3779B97F4A7C15ull >> 20) & (dmap.cap - 1);
            while (dmap.h[t] != ~0ull && dmap.h[t] != dk) t = (t + 1) & (dmap.cap - 1);
            if (dmap.h[t] == ~0ull) {
                dmap.h[t] = dk; dmap.v[t] = n_devids;
                out->dev_ids[n_devids] = first;
                if (dev_rule) dev_rule[n_devids] = (uint8_t)rule;
                n_devids++;
            }
            g_dev[n_groups] = dmap.v[t];
            dcount[dmap.v[t]]++;
            out->group_ids[n_groups] = r->iommu_group;
            n_groups++;
        }
        uint32_t g = gmap.v[s];
        gord[bus_index] = g;
        gcount[g]++;
        out->accept_index[i] = bus_index++;
    }
    out->group_off[0] = 0;
    for (uint32_t g = 0; g < n_groups; g++) out->group_off[g + 1] = out->group_off[g] + gcount[g];
    out->dev_off[0] = 0;
    for (uint32_t d = 0; d < n_devids; d++) out->dev_off[d + 1] = out->dev_off[d] + dcount[d];
    uint32_t *gfill = calloc(n_groups + 1, 4), *dfill = calloc(n_devids + 1, 4);
    for (size_t i = 0; i < n; i++) {
        uint32_t b = out->accept_index[i];
        if (b == KXPU_REJECTED) continue;
        uint32_t g = gord[b];
        out->group_members[out->group_off[g] + gfill[g]++] = (uint32_t)i;
    }
    for (uint32_t g = 0; g < n_groups; g++) {
        uint32_t d = g_dev[g];
        out->dev_groups[out->dev_off[d] + dfill[d]++] = out->group_ids[g];
    }
    out->n_accepted = bus_index; out->n_groups = n_groups; out->n_devids = n_devids;
    free(gfill); free(dfill); free(gcount); free(gord); free(dcount); free(g_dev); free(keys); free(klen);
    om_free(&gmap); om_free(&kmap); om_free(&dmap);
    return 0;
}

/* the type keys of recs[idx[j]]: offsets[k+1], returns the total length */
size_t kxo_mdev_names(const kxpu_mdevrec *recs, const uint32_t *idx, size_t k, uint8_t *out, uint32_t *offsets) {
    size_t p = 0;
    for (size_t j = 0; j < k; j++) {
        offsets[j] = (uint32_t)p;
        p += rec_key(&recs[idx[j]], out + p);
    }
    offsets[k] = (uint32_t)p;
    return p;
}

typedef struct { uint8_t *p; size_t cap, len; } kxo_buf;
static void put(kxo_buf *b, const void *s, size_t n) {
    if (b->p && b->len + n <= b->cap) memcpy(b->p + b->len, s, n);
    b->len += n;
}
static void puts_(kxo_buf *b, const char *s) { put(b, s, strlen(s)); }
static void putu(kxo_buf *b, uint64_t v) { char t[24]; int k = snprintf(t, sizeof t, "%llu", (unsigned long long)v); put(b, t, (size_t)k); }

/* generateCDISpec + Save for a vGPU class; (size_t)-1 for a kind, uuid or parent outside the domain */
size_t kxo_cdi_emit_mdev(int32_t format, const char *kind, const kxpu_mdevcdi *devs, size_t n, uint8_t *out, size_t cap) {
    if (!kxo_kind_ok(kind)) return (size_t)-1;
    for (size_t i = 0; i < n; i++) {
        size_t pl = strnlen(devs[i].parent, 16);
        if (!kxo_uuid_ok(devs[i].uuid) || pl == 0) return (size_t)-1;
        for (size_t k = 0; k < pl; k++)
            if (!strchr("0123456789abcdef:.", devs[i].parent[k])) return (size_t)-1;
    }
    kxo_buf b = { out, cap, 0 };
    if (format == KXPU_FMT_YAML) {
        puts_(&b, "cdiVersion: 0.6.0\nkind: "); puts_(&b, kind); puts_(&b, "\n");
        if (n == 0) { puts_(&b, "devices: []\n"); return b.len; }
        puts_(&b, "devices:\n");
        for (size_t i = 0; i < n; i++) {
            const kxpu_mdevcdi *d = &devs[i];
            size_t pl = strnlen(d->parent, 16);
            puts_(&b, "  - name: \""); putu(&b, d->index); puts_(&b, "\"\n");
            puts_(&b, "    annotations:\n      attach-pci: \"true\"\n      bdf: ");
            if (kxo_is_base60((const uint8_t *)d->parent, pl)) { puts_(&b, "\""); put(&b, d->parent, pl); puts_(&b, "\""); }
            else put(&b, d->parent, pl);
            puts_(&b, "\n      cdi.k8s.io/vfio"); putu(&b, d->iommu_group);
            puts_(&b, ": "); puts_(&b, kind); puts_(&b, "="); putu(&b, d->index);
            puts_(&b, "\n      mdev: "); put(&b, d->uuid, 36);
            puts_(&b, "\n    containerEdits:\n      deviceNodes:\n        - path: /dev/vfio/");
            putu(&b, d->iommu_group); puts_(&b, "\n");
        }
        return b.len;
    }
    puts_(&b, "{\n  \"cdiVersion\": \"0.6.0\",\n  \"kind\": \""); puts_(&b, kind); puts_(&b, "\",\n");
    if (n == 0) { puts_(&b, "  \"devices\": null,\n  \"containerEdits\": {}\n}"); return b.len; }
    puts_(&b, "  \"devices\": [\n");
    for (size_t i = 0; i < n; i++) {
        const kxpu_mdevcdi *d = &devs[i];
        puts_(&b, "    {\n      \"name\": \""); putu(&b, d->index);
        puts_(&b, "\",\n      \"annotations\": {\n        \"attach-pci\": \"true\",\n        \"bdf\": \"");
        put(&b, d->parent, strnlen(d->parent, 16));
        puts_(&b, "\",\n        \"cdi.k8s.io/vfio"); putu(&b, d->iommu_group);
        puts_(&b, "\": \""); puts_(&b, kind); puts_(&b, "="); putu(&b, d->index);
        puts_(&b, "\",\n        \"mdev\": \""); put(&b, d->uuid, 36);
        puts_(&b, "\"\n      },\n      \"containerEdits\": {\n        \"deviceNodes\": [\n          {\n            \"path\": \"/dev/vfio/");
        putu(&b, d->iommu_group);
        puts_(&b, "\"\n          }\n        ]\n      }\n    }");
        puts_(&b, i + 1 < n ? ",\n" : "\n");
    }
    puts_(&b, "  ],\n  \"containerEdits\": {}\n}");
    return b.len;
}
