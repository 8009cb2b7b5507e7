/*
 * pcie_mdev_oracle.c -- CPU checker of kxpu_pcie_tree_mdev (include/kxpu.h, addition to ABI v14), the C statement next
 * to the Python restatement (tests/pyref_pcie_mdev.py):
 *   kxo_pcie_parse_mdev   the mdev path grammar of one record (kxpu_mdevrec + kxpu_pcipath)
 *   kxo_pcie_tree_mdev    kxpu_pcie_tree_mdev
 * TEST INFRASTRUCTURE ONLY.  Restated one item at a time with none of the GPU's structure: a left-to-right scan of each
 * path, then a sequential walk over the groups with a (parent, key) -> child map.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "kxpu.h"

#define MAXD KXPU_PCIE_MAX_DEPTH
#define NONE KXPU_PCIE_NO_NODE

static int hexv(char c) { return (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : -1; }

/* n hex digits at s -> value, or -1 */
static int64_t hexn(const char *s, int n) {
    int64_t v = 0;
    for (int k = 0; k < n; k++) {
        const int d = hexv(s[k]);
        if (d < 0) return -1;
        v = v << 4 | d;
    }
    return v;
}

/* a domain of 4 digits, or 5..8 with a non-zero first digit, ending at the first ':' within lim bytes: its length, or 0 */
static int domain_len(const char *s, int lim) {
    int dl = 0;
    while (dl < lim && s[dl] != ':') dl++;
    if (dl == lim) return 0;
    return (dl == 4 || (dl >= 5 && dl <= 8 && s[0] != '0')) ? dl : 0;
}

/* one component: 1 = function, 2 = host bridge, 0 = neither */
static int component(const char *s, int len, uint64_t *key) {
    if (len >= 3 && !memcmp(s, "pci", 3)) {
        const int dl = domain_len(s + 3, len - 3);
        if (!dl || len != 3 + dl + 3) return 0;
        const int64_t dom = hexn(s + 3, dl), bus = hexn(s + 3 + dl + 1, 2);
        if (dom < 0 || bus < 0) return 0;
        *key = 1ull << 63 | (uint64_t)dom << 16 | (uint64_t)bus << 8;
        return 2;
    }
    const int dl = domain_len(s, len);
    if (!dl || len != dl + 8) return 0;
    const char *t = s + dl;
    if (t[0] != ':' || t[3] != ':' || t[6] != '.') return 0;
    const int64_t dom = hexn(s, dl), bus = hexn(t + 1, 2), dev = hexn(t + 4, 2);
    if (dom < 0 || bus < 0 || dev < 0 || dev > 0x1f || t[7] < '0' || t[7] > '7') return 0;
    *key = (uint64_t)dom << 16 | (uint64_t)bus << 8 | (uint64_t)dev << 3 | (uint64_t)(t[7] - '0');
    return 1;
}

/* a canonical lowercase UUID of 36 bytes at s */
static int canonical_uuid(const char *s, int len) {
    if (len != 36) return 0;
    for (int k = 0; k < 36; k++) {
        const int dash = k == 8 || k == 13 || k == 18 || k == 23;
        if (dash ? s[k] != '-' : hexv(s[k]) < 0) return 0;
    }
    return 1;
}

/* the chain of one mdev record: its length (0 = unknown), keys in chain[0 .. len) */
int32_t kxo_pcie_parse_mdev(const kxpu_mdevrec *rec, const kxpu_pcipath *p, uint64_t *chain) {
    const int len = p->len;
    if (len == 0 || len > 120) return 0;
    int comps = 1;
    for (int c = 0; c < len; c++) comps += p->path[c] == '/';
    if (comps < 2 || comps > MAXD + 1) return 0;
    size_t pl = 0;
    while (pl < sizeof rec->parent && rec->parent[pl]) pl++;
    int start = 0, k = 0;
    for (int c = 0; c <= len; c++) {
        if (c < len && p->path[c] != '/') continue;
        const char *s = p->path + start;
        const int cl = c - start;
        if (k == comps - 1) { /* the leaf: the record's own UUID */
            if (!canonical_uuid(s, cl) || memcmp(s, rec->uuid, 36)) return 0;
        } else {
            uint64_t key = 0;
            const int kind = component(s, cl, &key);
            if (kind == 0 || (k == 0 && kind != 2)) return 0;
            if (k == comps - 2 && (kind != 1 || (size_t)cl != pl || memcmp(s, rec->parent, pl))) return 0;
            chain[k] = key;
        }
        k++;
        start = c + 1;
    }
    return comps - 1;
}

typedef struct { uint32_t parent; uint64_t key; uint32_t node; int used; } child_slot;

static uint64_t mixh(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; return x ^ (x >> 33);
}

/* 0, or -1 when group_off decreases or a member is >= n (nothing written) */
int32_t kxo_pcie_tree_mdev(const kxpu_mdevrec *recs, const kxpu_pcipath *paths, size_t n, const uint32_t *group_off,
                           const uint32_t *group_members, size_t n_groups, uint32_t *group_node, uint64_t *key,
                           uint32_t *parent, uint8_t *depth, uint32_t *n_nodes) {
    for (size_t g = 0; g < n_groups; g++) {
        if (group_off[g + 1] < group_off[g]) return -1;
        for (uint32_t m = group_off[g]; m < group_off[g + 1]; m++)
            if (group_members[m] >= n) return -1;
    }
    uint64_t (*chain)[MAXD] = malloc((n ? n : 1) * sizeof *chain);
    uint8_t *clen = malloc(n ? n : 1);
    for (size_t i = 0; i < n; i++) clen[i] = (uint8_t)kxo_pcie_parse_mdev(&recs[i], &paths[i], chain[i]);
    size_t cap = 16;
    while (cap < 2 * MAXD * n_groups + 16) cap <<= 1;
    child_slot *tab = calloc(cap, sizeof *tab);
    uint32_t nn = 0;
    for (size_t g = 0; g < n_groups; g++) {
        int L = -1;
        uint64_t gc[MAXD];
        for (uint32_t m = group_off[g]; m < group_off[g + 1]; m++) {
            const uint32_t i = group_members[m];
            if (!clen[i]) continue;
            if (L < 0) { L = clen[i]; memcpy(gc, chain[i], sizeof gc); continue; }
            int k = 0;
            while (k < L && k < clen[i] && chain[i][k] == gc[k]) k++;
            L = k;
        }
        uint32_t at = NONE;
        for (int t = 0; t < L; t++) {
            size_t s = mixh(gc[t] ^ ((uint64_t)at * 0x9E3779B97F4A7C15ull)) & (cap - 1);
            while (tab[s].used && !(tab[s].parent == at && tab[s].key == gc[t])) s = (s + 1) & (cap - 1);
            if (!tab[s].used) {
                tab[s].used = 1; tab[s].parent = at; tab[s].key = gc[t]; tab[s].node = nn;
                key[nn] = gc[t]; parent[nn] = at; depth[nn] = (uint8_t)t;
                nn++;
            }
            at = tab[s].node;
        }
        group_node[g] = at;
    }
    *n_nodes = nn;
    free(tab); free(clen); free(chain);
    return 0;
}
