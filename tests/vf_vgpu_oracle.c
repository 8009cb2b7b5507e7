/*
 * vf_vgpu_oracle.c -- CPU checker of kxpu_vf_vgpu_types (include/kxpu.h, additions to ABI v14), the C statement next to
 * the Python one (tests/pyref_vf_vgpu.py).
 * TEST INFRASTRUCTURE ONLY: tests/vf_vgpu_oracle.py compiles it into a temporary directory.  Restated one item at a time
 * with none of the GPU's structure: every table is split line by line in priority order, each naming line is appended
 * to a list of (ID, key) unless the ID is listed already, and each record searches that list linearly.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "kxpu.h"

typedef struct { uint32_t id; uint8_t key[40]; uint8_t len; } named_t;

static int blank(uint8_t c) { return c == ' ' || c == '\t'; }

/* kxpu_classify_mdev's type key of name[0..len): trim "\t\n\v\f\r ", ' ' -> '_', keep [A-Za-z0-9_.-] */
static size_t type_key(const uint8_t *name, size_t len, uint8_t *out) {
    size_t a = 0, b = len, p = 0;
    while (a < b && (name[a] == ' ' || (name[a] >= '\t' && name[a] <= '\r'))) a++;
    while (b > a && (name[b - 1] == ' ' || (name[b - 1] >= '\t' && name[b - 1] <= '\r'))) b--;
    for (size_t k = a; k < b; k++) {
        uint8_t c = name[k] == ' ' ? '_' : name[k];
        if ((c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_' || c == '.' || c == '-')
            out[p++] = c;
    }
    return p;
}

/* one line [s, e) without its '\n': 1 and (id, key) when it names a type */
static int parse(const uint8_t *s, size_t len, uint32_t *id, uint8_t *key, uint8_t *klen) {
    if (len > 0 && s[len - 1] == '\r') len--;
    size_t p = 0;
    while (p < len && blank(s[p])) p++;
    const size_t d0 = p;
    uint64_t v = 0;
    while (p < len && s[p] >= '0' && s[p] <= '9' && p - d0 < 11) v = v * 10 + (uint64_t)(s[p++] - '0');
    if (p == d0 || s[d0] == '0' || (p < len && s[p] >= '0' && s[p] <= '9') || v > 0xFFFFFFFFull) return 0;
    while (p < len && blank(s[p])) p++;
    if (p == len || s[p] != ':') return 0;
    p++;
    while (p < len && blank(s[p])) p++;
    size_t e = len;
    while (e > p && blank(s[e - 1])) e--;
    if (e == p || e - p > 40) return 0;
    const size_t k = type_key(s + p, e - p, key);
    if (k == 0) return 0;
    *id = (uint32_t)v;
    *klen = (uint8_t)k;
    return 1;
}

int kxv_vf_vgpu_types(const kxpu_vfvgpurec *recs, size_t n, const uint8_t *blob, const uint64_t *toff, size_t n_tables,
                      kxpu_vgpukey *keys, uint32_t *type_id, uint8_t *status) {
    for (size_t t = 0; t < n_tables; t++)
        if (toff[t + 1] < toff[t]) return -1;
    named_t *list = NULL;
    size_t cnt = 0, cap = 0;
    for (size_t t = 0; t < n_tables; t++) {
        uint64_t a = toff[t];
        while (a < toff[t + 1]) {
            uint64_t e = a;
            while (e < toff[t + 1] && blob[e] != '\n') e++;
            named_t x;
            memset(&x, 0, sizeof x);
            if (parse(blob + a, (size_t)(e - a), &x.id, x.key, &x.len)) {
                size_t j = 0;
                while (j < cnt && list[j].id != x.id) j++;
                if (j == cnt) {
                    if (cnt == cap) {
                        cap = cap ? 2 * cap : 64;
                        list = realloc(list, cap * sizeof *list);
                    }
                    list[cnt++] = x;
                }
            }
            a = e + 1;  /* past the '\n'; a line that ends the table ends the loop too */
        }
    }
    for (size_t i = 0; i < n; i++) {
        const kxpu_vfvgpurec *r = &recs[i];
        memset(&keys[i], 0, sizeof keys[i]);
        type_id[i] = 0;
        status[i] = KXPU_VT_NONE;
        if (!(r->flags & KXPU_VT_READ)) continue;
        size_t len = r->cur_len;
        if ((r->flags & KXPU_VT_CUR_ERR) || len > 16) { status[i] = KXPU_VT_BAD; continue; }
        if (len > 0 && r->cur_txt[len - 1] == '\n') len--;
        int ok = len > 0 && !(len > 1 && r->cur_txt[0] == '0');
        uint64_t v = 0;
        for (size_t k = 0; ok && k < len; k++) {
            ok = r->cur_txt[k] >= '0' && r->cur_txt[k] <= '9';
            v = v * 10 + (uint64_t)(r->cur_txt[k] - '0');
            if (v > 0xFFFFFFFFull) ok = 0;
        }
        if (!ok) { status[i] = KXPU_VT_BAD; continue; }
        if (v == 0) continue;
        type_id[i] = (uint32_t)v;
        status[i] = KXPU_VT_UNNAMED;
        for (size_t j = 0; j < cnt; j++)
            if (list[j].id == v) {
                memcpy(keys[i].key, list[j].key, list[j].len);
                keys[i].len = list[j].len;
                status[i] = KXPU_VT_NAMED;
                break;
            }
    }
    free(list);
    return 0;
}
