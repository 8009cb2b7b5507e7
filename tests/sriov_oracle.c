/*
 * sriov_oracle.c -- CPU checker of the SR-IOV calls (include/kxpu.h, additions to ABI v14), the C statement next to the
 * Python one (tests/pyref_sriov.py):
 *   kxs_sriov             kxpu_sriov
 *   kxs_pcie_tree_sriov   kxpu_pcie_tree_sriov over chains the PCIe oracle parsed (kxo_pcie_parse)
 * TEST INFRASTRUCTURE ONLY: tests/sriov_oracle.py compiles it into a temporary directory.  Restated one item at a time
 * with none of the GPU's structure: addresses sorted once and searched, a sequential fold over the groups, and the forest
 * as a (parent, key) -> child list searched linearly.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "kxpu.h"

#define MAXD KXPU_PCIE_MAX_DEPTH

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

/* sriov_numvfs: at most one trailing '\n', then a canonical decimal 0..65535; anything else 0 */
static uint32_t numvfs_of(const kxpu_sriovrec *s) {
    if ((s->flags & KXPU_SR_NUMVFS_ERR) || s->numvfs_len > 8) return 0;
    size_t len = s->numvfs_len;
    if (len > 0 && s->numvfs_txt[len - 1] == '\n') len--;
    if (len == 0 || len > 5 || (len > 1 && s->numvfs_txt[0] == '0')) return 0;
    uint32_t v = 0;
    for (size_t k = 0; k < len; k++) {
        if (s->numvfs_txt[k] < '0' || s->numvfs_txt[k] > '9') return 0;
        v = v * 10 + (uint32_t)(s->numvfs_txt[k] - '0');
    }
    return v <= 65535 ? v : 0;
}

typedef struct { uint32_t key, idx; } addr_t;

static int addr_cmp(const void *a, const void *b) {
    const addr_t *x = a, *y = b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->idx < y->idx ? -1 : x->idx > y->idx;
}

static int csr_ok(const uint32_t *goff, const uint32_t *gmem, size_t G, size_t n) {
    for (size_t g = 0; g < G; g++) {
        if (goff[g + 1] < goff[g]) return 0;
        for (uint32_t m = goff[g]; m < goff[g + 1]; m++)
            if (gmem[m] >= n) return 0;
    }
    return 1;
}

/* 0, or -1 (nothing written) for a decreasing group_off or a member index >= n */
int kxs_sriov(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, const kxpu_sriovrec *srs, size_t n,
              const uint32_t *goff, const uint32_t *gmem, size_t G, uint32_t *pf_of, uint32_t *numvfs, uint32_t *group_sriov) {
    if (!csr_ok(goff, gmem, G, n)) return -1;
    addr_t *addrs = malloc((n + 1) * sizeof *addrs);
    size_t na = 0;
    for (size_t i = 0; i < n; i++) {
        uint32_t k;
        if (canonical(recs[i].bdf, &k)) addrs[na++] = (addr_t){k, (uint32_t)i};
    }
    qsort(addrs, na, sizeof *addrs, addr_cmp);
    for (size_t i = 0; i < n; i++) {
        numvfs[i] = numvfs_of(&srs[i]);
        pf_of[i] = KXPU_NO_PF;
        uint32_t k;
        if ((srs[i].flags & KXPU_SR_PHYSFN_ERR) || !canonical(srs[i].physfn, &k)) continue;
        size_t lo = 0, hi = na;  /* the first entry with this key: the lowest index */
        while (lo < hi) {
            const size_t mid = (lo + hi) / 2;
            if (addrs[mid].key < k) lo = mid + 1;
            else hi = mid;
        }
        if (lo < na && addrs[lo].key == k && addrs[lo].idx != i) pf_of[i] = addrs[lo].idx;
    }
    free(addrs);
    for (size_t g = 0; g < G; g++) {
        group_sriov[g] = KXPU_VIABLE;
        for (uint32_t m = goff[g]; m < goff[g + 1]; m++) {
            const uint32_t i = gmem[m], p = pf_of[i];
            int blocks = numvfs[i] > 0;
            if (p != KXPU_NO_PF && !(recs[p].flags & KXPU_REC_DRIVER_ERR))
                for (size_t r = 0; r < n_rules; r++)
                    if (strncmp(recs[p].driver, rules[r].driver, sizeof recs[p].driver) == 0) blocks = 1;
            if (blocks && i < group_sriov[g]) group_sriov[g] = i;
        }
    }
    return 0;
}

/* the node key of one path component, the grammar of kxpu_pcipath: a function or a host bridge; 0 when it is neither */
static int comp_key(const char *s, size_t len, uint64_t *key) {
    int bridge = 0;
    if (len >= 3 && memcmp(s, "pci", 3) == 0) { bridge = 1; s += 3; len -= 3; }
    size_t d = 0;
    uint64_t dom = 0;
    while (d < len && s[d] != ':') {
        if (hexv(s[d]) < 0 || d == 8) return 0;
        dom = dom << 4 | (uint64_t)hexv(s[d++]);
    }
    if (!(d == 4 || (d >= 5 && d <= 8 && s[0] != '0'))) return 0;
    if (len < d + 3 || hexv(s[d + 1]) < 0 || hexv(s[d + 2]) < 0) return 0;
    const uint64_t bus = (uint64_t)(hexv(s[d + 1]) << 4 | hexv(s[d + 2]));
    if (bridge) {
        if (len != d + 3) return 0;
        *key = 1ull << 63 | dom << 16 | bus << 8;
        return 1;
    }
    const char *t = s + d + 3;
    if (len != d + 8 || t[0] != ':' || t[3] != '.' || hexv(t[1]) < 0 || hexv(t[2]) < 0 || t[4] < '0' || t[4] > '7') return 0;
    const int dev = hexv(t[1]) << 4 | hexv(t[2]);
    if (dev > 0x1f) return 0;
    *key = dom << 16 | bus << 8 | (uint64_t)dev << 3 | (uint64_t)(t[4] - '0');
    return 1;
}

/* kxpu_pcie_tree_sriov with the chain of every record given: chain[i * MAXD ..] / clen[i] (0: unknown path).  0, or -1
 * (nothing written) for an invalid CSR or pf_of */
int kxs_pcie_tree_sriov(const kxpu_devrec *recs, const uint64_t *chain, const uint8_t *clen, size_t n, const uint32_t *goff,
                        const uint32_t *gmem, size_t G, const uint32_t *pf_of, uint32_t *group_node, uint64_t *key,
                        uint32_t *parent, uint8_t *depth, uint32_t *n_nodes) {
    if (!csr_ok(goff, gmem, G, n)) return -1;
    for (size_t i = 0; i < n; i++)
        if (pf_of[i] != KXPU_NO_PF && pf_of[i] >= n) return -1;
    uint32_t nn = 0;
    for (size_t g = 0; g < G; g++) {
        uint64_t common[MAXD + 1];
        int L = -1;
        for (uint32_t m = goff[g]; m < goff[g + 1]; m++) {
            const uint32_t i = gmem[m], p = pf_of[i];
            uint64_t c[MAXD + 1];
            int l = clen[i];
            memcpy(c, chain + (size_t)i * MAXD, sizeof(uint64_t) * MAXD);
            uint64_t own;
            if (p != KXPU_NO_PF && clen[p] > 0 && clen[p] < MAXD &&
                comp_key(recs[p].bdf, strnlen(recs[p].bdf, sizeof recs[p].bdf), &own)) {
                l = clen[p];
                memcpy(c, chain + (size_t)p * MAXD, sizeof(uint64_t) * MAXD);
                c[l++] = own;  /* the PF itself: its VFs sit below it */
            }
            if (l == 0) continue;
            if (L < 0) {
                memcpy(common, c, sizeof(uint64_t) * (size_t)l);
                L = l;
            } else {
                int k = 0;
                while (k < L && k < l && common[k] == c[k]) k++;
                L = k;
            }
        }
        uint32_t v = KXPU_PCIE_NO_NODE;
        for (int t = 0; t < L; t++) {
            uint32_t found = KXPU_PCIE_NO_NODE;
            for (uint32_t u = 0; u < nn && found == KXPU_PCIE_NO_NODE; u++)
                if (parent[u] == v && key[u] == common[t]) found = u;
            if (found == KXPU_PCIE_NO_NODE) {
                found = nn++;
                key[found] = common[t];
                parent[found] = v;
                depth[found] = (uint8_t)t;
            }
            v = found;
        }
        group_node[g] = v;
    }
    *n_nodes = nn;
    return 0;
}
