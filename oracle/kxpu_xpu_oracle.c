/*
 * kxpu_xpu_oracle.c -- CPU restatement of discovery for accelerators of any configured vendor:
 * createIommuDeviceMap (pkg/device_plugin/device_plugin.go:126-180) with a (vendor, driver) rule list in
 * place of nvidiaVendorID (:19,149) and "vfio-pci" (:156), and generateCDISpec / QualifiedName with the CDI
 * kind in place of CdiVendorClass (generic_device_plugin.go:31).  The checker of kxpu_classify_rules,
 * kxpu_cdi_emit_kind and kxpu_alloc_names_kind (include/kxpu.h).
 *
 * TEST INFRASTRUCTURE ONLY, like kxpu_oracle.c: loaded by tests/ through oracle/xpu_oracle.py, never by the
 * product.  It is a separate restatement of the walk; kxpu_oracle.c stays the pinned NVIDIA-only one, and the
 * CPU tests check that this file with the NVIDIA rule / kind gives its bytes.  The yaml.v3 base-60 predicate
 * is taken from there (kxo_is_base60, declared in kxpu_oracle.h), so both documents quote the same bdf strings.
 */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../include/kxpu.h"
#include "kxpu_oracle.h"

/* readIDFromFileFunc :183-191: data[2:] with all leading/trailing '\n' trimmed.
 * Returns length (<= 8) or -1 for "would panic" (file < 2 bytes) / unsupported. */
static int kxo_read_id(const uint8_t *txt, unsigned flen, uint8_t id[8]) {
    memset(id, 0, 8);
    if (flen < 2 || flen > 8) return -1;
    const uint8_t *s = txt + 2;
    int len = (int)flen - 2;
    while (len > 0 && s[0] == '\n') { s++; len--; }
    while (len > 0 && s[len - 1] == '\n') len--;
    memcpy(id, s, (size_t)len);
    return len;
}

typedef struct { uint64_t *keys; uint32_t *vals; size_t cap; } kxo_map;
static void map_init(kxo_map *m, size_t n) {
    size_t c = 16; while (c < 2 * n + 2) c <<= 1;
    m->cap = c; m->keys = (uint64_t *)malloc(c * 8); m->vals = (uint32_t *)malloc(c * 4);
    memset(m->keys, 0xff, c * 8);
}
static void map_free(kxo_map *m) { free(m->keys); free(m->vals); }
static uint32_t *map_get(kxo_map *m, uint64_t k, int *fresh) {
    uint64_t h = k * 0x9E3779B97F4A7C15ull;
    size_t i = (size_t)(h >> 20) & (m->cap - 1);
    for (;;) {
        if (m->keys[i] == k) { *fresh = 0; return &m->vals[i]; }
        if (m->keys[i] == ~0ull) { m->keys[i] = k; *fresh = 1; return &m->vals[i]; }
        i = (i + 1) & (m->cap - 1);
    }
}

#define KXO_UNSEEN 0xFFFFFFFEu

typedef struct { uint8_t *p; size_t cap, len; } kxo_buf;
static void put(kxo_buf *b, const void *s, size_t n) {
    if (b->p && b->len + n <= b->cap) memcpy(b->p + b->len, s, n);
    b->len += n;
}
static void puts_(kxo_buf *b, const char *s) { put(b, s, strlen(s)); }
static void putu(kxo_buf *b, uint64_t v) { char t[24]; int k = snprintf(t, sizeof t, "%llu", (unsigned long long)v); put(b, t, (size_t)k); }

static size_t bdf_len(const char *bdf) { size_t l = 0; while (l < 16 && bdf[l]) l++; return l; }

/* ------------------------------------------------------------------------- */
/* createIommuDeviceMap with a (vendor, driver) rule list.                    */
/* ------------------------------------------------------------------------- */

/* include/kxpu.h kxpu_classify_rules: the rule list is valid or the call returns -1 (KXPU_E_INVALID) */
static int kxo_rule_field(const char *f, size_t cap) {
    size_t l = 0;
    while (l < cap && f[l]) l++;
    for (size_t k = l; k < cap; k++) if (f[k]) return -1;   /* a byte after the terminating NUL */
    return (int)l;
}

int32_t kxo_classify_rules(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, size_t n,
                           kxpu_classify_out *out, uint8_t *dev_rule) {
    if (n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    for (size_t r = 0; r < n_rules; r++) {
        int vl = kxo_rule_field(rules[r].vendor, 8), dl = kxo_rule_field(rules[r].driver, 16);
        if (vl < 1 || vl > 6 || memchr(rules[r].vendor, '\n', (size_t)vl)) return KXPU_E_INVALID;
        if (dl < 1 || dl > 15 || memchr(rules[r].driver, '/', (size_t)dl)) return KXPU_E_INVALID;
        for (size_t q = 0; q < r; q++)
            if (strncmp(rules[q].vendor, rules[r].vendor, 8) == 0 && strncmp(rules[q].driver, rules[r].driver, 16) == 0)
                return KXPU_E_INVALID;
    }
    kxo_map gmap, dmap;
    map_init(&gmap, n); map_init(&dmap, n);
    uint32_t *gcount = (uint32_t *)calloc(n + 1, 4);
    uint32_t *gord = (uint32_t *)malloc((n + 1) * 4);
    uint32_t *dcount = (uint32_t *)calloc(n + 1, 4);
    uint32_t *g_dev = (uint32_t *)malloc((n + 1) * 4);
    uint32_t bus_index = 0, n_groups = 0, n_devids = 0;               /* :130, one counter for every rule */
    for (size_t i = 0; i < n; i++) {
        const kxpu_devrec *r = &recs[i];
        out->accept_index[i] = KXPU_REJECTED;
        if (r->flags & KXPU_REC_IS_DIR) continue;                    /* :137 */
        if (r->flags & KXPU_REC_VENDOR_ERR) continue;                /* :143 */
        uint8_t id[8];
        int l = kxo_read_id(r->vendor_txt, r->vendor_len, id);
        if (l < 0) continue;
        if (r->flags & KXPU_REC_DRIVER_ERR) {
            /* :152 comes after :149: whether or not the vendor matched, the record is skipped */
            continue;
        }
        int rule = -1;
        for (size_t q = 0; q < n_rules && rule < 0; q++) {
            if ((size_t)l == strnlen(rules[q].vendor, 8) && memcmp(id, rules[q].vendor, (size_t)l) == 0 &&  /* :149 */
                strncmp(r->driver, rules[q].driver, 16) == 0)                                               /* :156 */
                rule = (int)q;
        }
        if (rule < 0) continue;
        if (r->flags & KXPU_REC_IOMMU_ERR) continue;                 /* :158 */
        int fresh;
        uint32_t *g = map_get(&gmap, r->iommu_group, &fresh);        /* :162 */
        if (fresh) *g = KXO_UNSEEN;
        if (*g == KXO_UNSEEN) {
            int dl = (r->flags & KXPU_REC_DEVICE_ERR) ? -1 : kxo_read_id(r->device_txt, r->device_len, id);
            if (dl < 0) continue;                                    /* :165-168: the group stays unseen */
            *g = n_groups;
            uint64_t dk = 0; memcpy(&dk, id, 8);
            /* deviceMap key: (rule of the group's first member, device id); an id is <= 6 bytes */
            uint64_t key = dk | ((uint64_t)rule << 48);
            int dfresh;
            uint32_t *d = map_get(&dmap, key, &dfresh);
            if (dfresh) {
                *d = n_devids;
                out->dev_ids[n_devids] = dk;
                if (dev_rule) dev_rule[n_devids] = (uint8_t)rule;
                n_devids++;
            }
            g_dev[n_groups] = *d;
            dcount[*d]++;                                            /* :169 */
            out->group_ids[n_groups] = r->iommu_group;
            n_groups++;
        }
        gord[bus_index] = *g;
        gcount[*g]++;
        out->accept_index[i] = bus_index++;                          /* :171-175 */
    }
    out->group_off[0] = 0;
    for (uint32_t g = 0; g < n_groups; g++) out->group_off[g + 1] = out->group_off[g] + gcount[g];
    out->dev_off[0] = 0;
    for (uint32_t d = 0; d < n_devids; d++) out->dev_off[d + 1] = out->dev_off[d] + dcount[d];
    uint32_t *gfill = (uint32_t *)calloc(n_groups + 1, 4), *dfill = (uint32_t *)calloc(n_devids + 1, 4);
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
    free(gfill); free(dfill); free(gcount); free(gord); free(dcount); free(g_dev);
    map_free(&gmap); map_free(&dmap);
    return 0;
}

/* include/kxpu.h kxpu_cdi_emit_kind, the kind domain [mem]: CDI v0.8.0 pkg/parser IsValidVendorName /
 * IsValidClassName narrowed to "starts with a letter, ends with a letter or digit": vendor
 * [A-Za-z][A-Za-z0-9_.-]*[A-Za-z0-9] (or one letter), class [A-Za-z][A-Za-z0-9_-]*[A-Za-z0-9] (or one letter),
 * "vendor/class" at most 63 bytes.  Returns 1 when the kind is inside the domain. */
static int kxo_alpha(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
static int kxo_alnum(char c) { return kxo_alpha(c) || (c >= '0' && c <= '9'); }
int kxo_kind_ok(const char *kind) {
    size_t len = strnlen(kind, 64);
    if (len > 63) return 0;
    const char *slash = strchr(kind, '/');
    if (!slash) return 0;
    size_t vl = (size_t)(slash - kind), cl = len - vl - 1;
    if (vl == 0 || cl == 0) return 0;
    if (!kxo_alpha(kind[0]) || !kxo_alnum(kind[vl - 1])) return 0;
    for (size_t k = 0; k < vl; k++)
        if (!kxo_alnum(kind[k]) && kind[k] != '_' && kind[k] != '.' && kind[k] != '-') return 0;
    const char *c = slash + 1;
    if (!kxo_alpha(c[0]) || !kxo_alnum(c[cl - 1])) return 0;
    for (size_t k = 0; k < cl; k++)
        if (!kxo_alnum(c[k]) && c[k] != '_' && c[k] != '-') return 0;
    return 1;
}

/* generateCDISpec + Save with the kind as an argument; (size_t)-1 when the kind is outside the domain */
size_t kxo_cdi_emit_kind(int32_t format, const char *kind, const kxpu_cdidev *devs, size_t n, uint8_t *out, size_t cap) {
    if (!kxo_kind_ok(kind)) return (size_t)-1;
    kxo_buf b = { out, cap, 0 };
    if (format == KXPU_FMT_YAML) {
        puts_(&b, "cdiVersion: 0.6.0\nkind: "); puts_(&b, kind); puts_(&b, "\n");     /* spec.go:12-13,18-19 */
        if (n == 0) { puts_(&b, "devices: []\n"); return b.len; }
        puts_(&b, "devices:\n");
        for (size_t i = 0; i < n; i++) {
            const kxpu_cdidev *d = &devs[i];
            size_t bl = bdf_len(d->bdf);
            puts_(&b, "  - name: \""); putu(&b, d->index); puts_(&b, "\"\n");
            puts_(&b, "    annotations:\n      attach-pci: \"true\"\n      bdf: ");
            if (kxo_is_base60((const uint8_t *)d->bdf, bl)) { puts_(&b, "\""); put(&b, d->bdf, bl); puts_(&b, "\""); }
            else put(&b, d->bdf, bl);
            puts_(&b, "\n      cdi.k8s.io/vfio"); putu(&b, d->iommu_group);
            puts_(&b, ": "); puts_(&b, kind); puts_(&b, "="); putu(&b, d->index);  /* device_plugin.go:66 */
            puts_(&b, "\n    containerEdits:\n      deviceNodes:\n        - path: /dev/vfio/");
            putu(&b, d->iommu_group); puts_(&b, "\n");
        }
        return b.len;
    }
    puts_(&b, "{\n  \"cdiVersion\": \"0.6.0\",\n  \"kind\": \""); puts_(&b, kind); puts_(&b, "\",\n");
    if (n == 0) { puts_(&b, "  \"devices\": null,\n  \"containerEdits\": {}\n}"); return b.len; }
    puts_(&b, "  \"devices\": [\n");
    for (size_t i = 0; i < n; i++) {
        const kxpu_cdidev *d = &devs[i];
        size_t bl = bdf_len(d->bdf);
        puts_(&b, "    {\n      \"name\": \""); putu(&b, d->index);
        puts_(&b, "\",\n      \"annotations\": {\n        \"attach-pci\": \"true\",\n        \"bdf\": \"");
        put(&b, d->bdf, bl);
        puts_(&b, "\",\n        \"cdi.k8s.io/vfio"); putu(&b, d->iommu_group);
        puts_(&b, "\": \""); puts_(&b, kind); puts_(&b, "="); putu(&b, d->index);
        puts_(&b, "\"\n      },\n      \"containerEdits\": {\n        \"deviceNodes\": [\n          {\n            \"path\": \"/dev/vfio/");
        putu(&b, d->iommu_group);
        puts_(&b, "\"\n          }\n        ]\n      }\n    }");
        puts_(&b, i + 1 < n ? ",\n" : "\n");
    }
    puts_(&b, "  ],\n  \"containerEdits\": {}\n}");
    return b.len;
}

/* QualifiedName(vendor, class, idx) = kind + "=" + idx (cdi-utils.go:9); (size_t)-1 outside the domain */
size_t kxo_alloc_names_kind(const char *kind, const uint64_t *idx, size_t n, uint8_t *out, size_t cap, uint32_t *offsets) {
    if (!kxo_kind_ok(kind)) return (size_t)-1;
    kxo_buf b = { out, cap, 0 };
    for (size_t i = 0; i < n; i++) {
        offsets[i] = (uint32_t)b.len;
        puts_(&b, kind); puts_(&b, "="); putu(&b, idx[i]);
    }
    offsets[n] = (uint32_t)b.len;
    return b.len;
}
