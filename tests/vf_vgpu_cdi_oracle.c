/*
 * vf_vgpu_cdi_oracle.c -- CPU checker of kxpu_cdi_emit_vf_vgpu / kxpu_cdi_emit_vf_vgpu_cdev (include/kxpu.h, additions
 * to ABI v14), the C statement next to the Python one (tests/pyref_vf_vgpu_cdi.py).
 * TEST INFRASTRUCTURE ONLY: tests/vf_vgpu_cdi_oracle.py compiles it into a temporary directory.  Restated one device at a
 * time with snprintf into a growing buffer, with none of the GPU's structure (no literal pool, no tiles, no scan).
 */
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "kxpu.h"

typedef struct { uint8_t *p; size_t len, cap; } buf_t;

static int put(buf_t *b, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
static int put(buf_t *b, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    char tmp[1024];
    const int k = vsnprintf(tmp, sizeof tmp, fmt, ap);
    va_end(ap);
    if (k < 0 || (size_t)k >= sizeof tmp) return -1;
    if (b->len + (size_t)k > b->cap) {
        size_t cap = b->cap ? b->cap : 4096;
        while (cap < b->len + (size_t)k) cap *= 2;
        uint8_t *p = realloc(b->p, cap);
        if (!p) return -1;
        b->p = p;
        b->cap = cap;
    }
    memcpy(b->p + b->len, tmp, (size_t)k);
    b->len += (size_t)k;
    return 0;
}

static int alpha(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
static int digit(char c) { return c >= '0' && c <= '9'; }

/* kxpu_cdi_emit_kind's kind domain: vendor "/" class, <= 63 bytes */
static int kind_ok(const char *kind) {
    const size_t len = strlen(kind);
    const char *slash = strchr(kind, '/');
    if (len > 63 || !slash) return 0;
    for (int part = 0; part < 2; part++) {
        const char *s = part ? slash + 1 : kind;
        const size_t l = part ? len - (size_t)(slash - kind) - 1 : (size_t)(slash - kind);
        if (l == 0 || !alpha(s[0]) || !(alpha(s[l - 1]) || digit(s[l - 1]))) return 0;
        for (size_t k = 0; k < l; k++)
            if (!(alpha(s[k]) || digit(s[k]) || s[k] == '_' || s[k] == '-' || (!part && s[k] == '.'))) return 0;
    }
    return 1;
}

/* yaml.v3's isBase60Float: [-+]?[0-9][0-9_]*(:[0-5]?[0-9])+(\.[0-9_]*)? over the whole string */
static int base60(const char *s) {
    size_t i = 0;
    if (s[i] == '-' || s[i] == '+') i++;
    if (!digit(s[i])) return 0;
    i++;
    while (digit(s[i]) || s[i] == '_') i++;
    int groups = 0;
    while (s[i] == ':') {
        size_t j = i + 1;
        if (!digit(s[j])) break;
        if (digit(s[j + 1]) && s[j] <= '5') j += 2;
        else j += 1;
        i = j;
        groups++;
    }
    if (!groups) return 0;
    if (s[i] == '.') { i++; while (digit(s[i]) || s[i] == '_') i++; }
    return s[i] == 0;
}

/* 0: the document in *out (malloc'd, *len bytes); -7: a record or the kind outside the domain; -1: out of memory */
int kxv_cdi_vf_vgpu(int fmt, const char *kind, const kxpu_vfvgpucdi *devs, size_t n, int cdev, uint8_t **out, size_t *len) {
    if (!kind_ok(kind)) return -7;
    for (size_t i = 0; i < n; i++) {
        const kxpu_vfvgpucdi *d = &devs[i];
        const size_t bl = strnlen(d->dev.bdf, sizeof d->dev.bdf);
        if (bl == 0 || d->type_id == 0 || d->key_len == 0 || d->key_len > 40) return -7;
        for (size_t k = 0; k < bl; k++)
            if (!(digit(d->dev.bdf[k]) || (d->dev.bdf[k] >= 'a' && d->dev.bdf[k] <= 'f') || d->dev.bdf[k] == ':' ||
                  d->dev.bdf[k] == '.'))
                return -7;
        for (size_t k = 0; k < d->key_len; k++) {
            const char c = d->key[k];
            if (!(alpha(c) || digit(c) || c == '_' || c == '.' || c == '-')) return -7;
        }
    }
    buf_t b = {0, 0, 0};
    int e = 0;
    if (fmt == KXPU_FMT_YAML) {
        e |= put(&b, "cdiVersion: 0.6.0\nkind: %s\n", kind);
        e |= put(&b, n ? "devices:\n" : "devices: []\n");
    } else {
        e |= put(&b, "{\n  \"cdiVersion\": \"0.6.0\",\n  \"kind\": \"%s\",\n", kind);
        e |= put(&b, n ? "  \"devices\": [\n" : "  \"devices\": null,\n  \"containerEdits\": {}\n}");
    }
    for (size_t i = 0; i < n && !e; i++) {
        const kxpu_vfvgpucdi *d = &devs[i];
        char bdf[17], key[41], node[40];
        memcpy(bdf, d->dev.bdf, 16);
        bdf[16] = 0;
        memcpy(key, d->key, d->key_len);
        key[d->key_len] = 0;
        const unsigned long long idx = (unsigned long long)d->dev.index;
        if (cdev) snprintf(node, sizeof node, "/dev/vfio/devices/vfio%u", d->dev.vfio_cdev);
        else snprintf(node, sizeof node, "/dev/vfio/%u", d->dev.iommu_group);
        if (fmt == KXPU_FMT_YAML) {
            const char *q = base60(bdf) ? "\"" : "";
            e |= put(&b, "  - name: \"%llu\"\n    annotations:\n      attach-pci: \"true\"\n      bdf: %s%s%s\n", idx, q, bdf, q);
            e |= put(&b, "      cdi.k8s.io/vfio%u: %s=%llu\n", d->dev.iommu_group, kind, idx);
            e |= put(&b, "      vgpu-type: \"%u\"\n      vgpu-type-key: \"%s\"\n", d->type_id, key);
            e |= put(&b, "    containerEdits:\n      deviceNodes:\n        - path: %s\n", node);
        } else {
            e |= put(&b, "    {\n      \"name\": \"%llu\",\n      \"annotations\": {\n        \"attach-pci\": \"true\",\n", idx);
            e |= put(&b, "        \"bdf\": \"%s\",\n        \"cdi.k8s.io/vfio%u\": \"%s=%llu\",\n", bdf, d->dev.iommu_group, kind, idx);
            e |= put(&b, "        \"vgpu-type\": \"%u\",\n        \"vgpu-type-key\": \"%s\"\n      },\n", d->type_id, key);
            e |= put(&b, "      \"containerEdits\": {\n        \"deviceNodes\": [\n          {\n            \"path\": \"%s\"\n", node);
            e |= put(&b, "          }\n        ]\n      }\n    }%s", i + 1 < n ? ",\n" : "\n");
        }
    }
    if (n && fmt == KXPU_FMT_JSON) e |= put(&b, "  ],\n  \"containerEdits\": {}\n}");
    if (e) { free(b.p); return -1; }
    *out = b.p;
    *len = b.len;
    return 0;
}

void kxv_free(uint8_t *p) { free(p); }
