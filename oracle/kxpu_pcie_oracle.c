/*
 * kxpu_pcie_oracle.c -- CPU checker of the PCIe topology calls (include/kxpu.h, ABI v7):
 *   kxo_pcie_parse                    the path grammar of one record (kxpu_pcipath)
 *   kxo_pcie_tree                     kxpu_pcie_tree
 *   kxo_preferred_allocation_pcie     kxpu_preferred_allocation_pcie
 * TEST INFRASTRUCTURE ONLY.  Restated one item at a time with none of the GPU's structure: a left-to-right scan of
 * each path, a sequential walk over the groups with a (parent, key) -> child map, and per request the node counts by
 * walking every available device up to its root, X by a linear selection, and one sort of the candidates by
 * (lca level, NUMA bin rank, position).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/kxpu.h"

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

/* domain at s (length up to the next ':' within lim bytes): its digit count, or 0 when it breaks the rule */
static int domain_len(const char *s, int lim) {
    int dl = 0;
    while (dl < lim && s[dl] != ':') dl++;
    if (dl == lim) return 0;
    if (dl == 4) return 4;
    if (dl >= 5 && dl <= 8 && s[0] != '0') return dl;
    return 0;
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

/* the chain of one record: its length (0 = unknown), keys in chain[0 .. len) */
int32_t kxo_pcie_parse(const kxpu_devrec *rec, const kxpu_pcipath *p, uint64_t *chain) {
    const int len = p->len;
    if (len == 0 || len > 120) return 0;
    int start = 0, ncomp = 0;
    size_t bl = 0;
    while (bl < 16 && rec->bdf[bl]) bl++;
    for (int c = 0; c <= len; c++) {
        if (c < len && p->path[c] != '/') continue;
        const int cl = c - start;
        const int last = c == len;
        if (!last && ncomp >= MAXD) return 0; /* a ninth chain component */
        uint64_t key = 0;
        const int kind = component(p->path + start, cl, &key);
        if (kind == 0 || (ncomp == 0 && kind != 2)) return 0;
        if (last) {
            if ((size_t)cl != bl || memcmp(p->path + start, rec->bdf, bl)) return 0;
        } else {
            chain[ncomp] = key;
        }
        ncomp++;
        start = c + 1;
    }
    return ncomp >= 2 ? ncomp - 1 : 0;
}

/* ---------------------------------------------------------------- the forest */
typedef struct { uint32_t parent; uint64_t key; uint32_t node; int used; } child_slot;

static uint64_t mixh(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; return x ^ (x >> 33);
}

/* 0, or -1 when group_off decreases or a member is >= n (nothing written) */
int32_t kxo_pcie_tree(const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n, const uint32_t *group_off,
                      const uint32_t *group_members, size_t n_groups, uint32_t *group_node, uint64_t *key,
                      uint32_t *parent, uint8_t *depth, uint32_t *n_nodes) {
    for (size_t g = 0; g < n_groups; g++) {
        if (group_off[g + 1] < group_off[g]) return -1;
        for (uint32_t m = group_off[g]; m < group_off[g + 1]; m++)
            if (group_members[m] >= n) return -1;
    }
    uint64_t (*chain)[MAXD] = malloc((n ? n : 1) * sizeof *chain);
    uint8_t *clen = malloc(n ? n : 1);
    for (size_t i = 0; i < n; i++) clen[i] = (uint8_t)kxo_pcie_parse(&recs[i], &paths[i], chain[i]);
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

/* ---------------------------------------------------------------- preferred allocation */
static uint32_t home_of(uint64_t m) {
    for (uint32_t k = 0; k < 64; k++) if ((m >> k) & 1) return k;
    return 64;
}

typedef struct { uint32_t lvl, rank, pos; } cand;
static int cand_cmp(const void *a, const void *b) {
    const cand *x = a, *y = b;
    if (x->lvl != y->lvl) return x->lvl < y->lvl ? -1 : 1;
    if (x->rank != y->rank) return x->rank < y->rank ? -1 : 1;
    return x->pos < y->pos ? -1 : x->pos > y->pos;
}

/* -1 when u has the smaller key, 1 when v has (u != v) */
static int node_cmp(uint32_t u, uint32_t v, const uint32_t *av, const uint32_t *mn, const uint32_t *parent,
                    const uint8_t *depth) {
    if (av[u] != av[v]) return av[u] < av[v] ? -1 : 1;
    if (depth[u] != depth[v]) return depth[u] > depth[v] ? -1 : 1;
    for (uint32_t a = parent[u], b = parent[v]; a != NONE; a = parent[a], b = parent[b])
        if (av[a] != av[b]) return av[a] < av[b] ? -1 : 1;
    return mn[u] < mn[v] ? -1 : 1;
}

int32_t kxo_preferred_allocation_pcie(const uint64_t *dev_numa, const uint32_t *dev_node, size_t n_devs,
                                      const uint32_t *parent, const uint8_t *depth, size_t n_nodes,
                                      const uint32_t *avail_off, const uint32_t *avail, const uint32_t *must_off,
                                      const uint32_t *must, const uint32_t *size, size_t n_req, uint32_t *out,
                                      uint32_t *out_off) {
    for (size_t v = 0; v < n_nodes; v++) {
        if (depth[v] >= MAXD) return -1;
        if (parent[v] == NONE ? depth[v] != 0 : (parent[v] >= v || depth[v] != depth[parent[v]] + 1)) return -1;
    }
    for (size_t d = 0; dev_node && d < n_devs; d++)
        if (dev_node[d] != NONE && dev_node[d] >= n_nodes) return -1;
    uint8_t *mark = calloc(n_devs ? n_devs : 1, 1);
    uint32_t *av = calloc(n_nodes ? n_nodes : 1, 4), *mi = calloc(n_nodes ? n_nodes : 1, 4);
    uint32_t *mn = malloc((n_nodes ? n_nodes : 1) * 4);
    for (size_t v = 0; v < n_nodes; v++) mn[v] = 0xFFFFFFFFu;
    cand *cs = NULL;
    size_t cs_cap = 0;
    int32_t rc = 0;
    out_off[0] = 0;
#define NODE_OF(p) (dev_node ? dev_node[p] : NONE)
    for (size_t q = 0; q < n_req && rc == 0; q++) {
        const uint32_t *a = avail + avail_off[q], *mu = must + must_off[q];
        const size_t na = avail_off[q + 1] - avail_off[q], nm = must_off[q + 1] - must_off[q];
        if (size[q] < nm || size[q] > na) { rc = -1; break; }
        out_off[q + 1] = out_off[q] + size[q];
        for (size_t j = 0; j < na && rc == 0; j++) {
            if (a[j] >= n_devs || (mark[a[j]] & 1)) rc = -1;
            else mark[a[j]] |= 1;
        }
        for (size_t j = 0; j < nm && rc == 0; j++) {
            if (mu[j] >= n_devs || (mark[mu[j]] & 2) || !(mark[mu[j]] & 1)) rc = -1;
            else mark[mu[j]] |= 2;
        }
        if (rc == 0) {
            /* 1. node counts and X */
            for (size_t j = 0; j < na; j++)
                for (uint32_t v = NODE_OF(a[j]); v != NONE; v = parent[v]) {
                    av[v]++;
                    if (a[j] < mn[v]) mn[v] = a[j];
                    if (mark[a[j]] & 2) mi[v]++;
                }
            uint32_t X = NONE;
            for (size_t j = 0; j < na; j++)
                for (uint32_t v = NODE_OF(a[j]); v != NONE; v = parent[v])
                    if (mi[v] == nm && av[v] >= size[q] && (X == NONE || node_cmp(v, X, av, mn, parent, depth) < 0)) X = v;
            /* 2. candidates in X: lca level, NUMA bins over them */
            uint64_t U = 0;
            uint32_t c[65] = {0};
            for (size_t j = 0; j < nm; j++) {
                const uint32_t h = home_of(dev_numa[mu[j]]);
                if (h < 64) U |= 1ull << h;
            }
            if (na > cs_cap) { cs_cap = na; cs = realloc(cs, cs_cap * sizeof *cs); }
            size_t nc = 0;
            for (size_t j = 0; j < na; j++) {
                if (mark[a[j]] != 1) continue;
                int inX = X == NONE, lca = -1;
                for (uint32_t v = NODE_OF(a[j]); v != NONE; v = parent[v]) {
                    if (v == X) inX = 1;
                    if (lca < 0 && mi[v]) lca = depth[v];
                }
                if (!inX) continue;
                cs[nc].lvl = lca < 0 ? MAXD : (uint32_t)(MAXD - 1 - lca);
                cs[nc].rank = home_of(dev_numa[a[j]]); /* the home for now, its bin rank below */
                cs[nc].pos = a[j];
                c[cs[nc].rank]++;
                nc++;
            }
            uint32_t rank[65];
            int used[65] = {0};
            for (uint32_t r = 0; r < 65; r++) {
                int best = -1;
                for (uint32_t k = 0; k < 65; k++) {
                    if (used[k]) continue;
                    if (best < 0) { best = (int)k; continue; }
                    const int gk = k == 64 ? 2 : (((U >> k) & 1) ? 0 : 1), gb = best == 64 ? 2 : (((U >> best) & 1) ? 0 : 1);
                    if (gk < gb || (gk == gb && c[k] > c[best])) best = (int)k;
                }
                used[best] = 1;
                rank[best] = r;
            }
            for (size_t j = 0; j < nc; j++) cs[j].rank = rank[cs[j].rank];
            qsort(cs, nc, sizeof *cs, cand_cmp);
            uint32_t *o = out + out_off[q];
            for (size_t j = 0; j < nm; j++) o[j] = mu[j];
            for (size_t j = 0; j < size[q] - nm; j++) o[nm + j] = cs[j].pos;
            for (size_t j = 0; j < na; j++)
                for (uint32_t v = NODE_OF(a[j]); v != NONE; v = parent[v]) { av[v] = 0; mi[v] = 0; mn[v] = 0xFFFFFFFFu; }
        }
        for (size_t j = 0; j < na; j++) if (a[j] < n_devs) mark[a[j]] = 0;
        for (size_t j = 0; j < nm; j++) if (mu[j] < n_devs) mark[mu[j]] = 0;
    }
#undef NODE_OF
    free(cs); free(mark); free(av); free(mi); free(mn);
    return rc;
}
