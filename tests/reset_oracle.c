/*
 * reset_oracle.c -- CPU checker of kxpu_reset_check (include/kxpu.h, an addition to ABI v14), the C statement next to the
 * Python one (tests/pyref_reset.py).  The chains come from the PCIe oracle's path parse (kxo_pcie_parse, through
 * oracle/pcie_oracle.py), so the kernel's reuse of kxpu_pcie_tree's parse is checked against an independent parse.
 * TEST INFRASTRUCTURE ONLY: tests/reset_oracle.py compiles it into a temporary directory.  Restated one item at a time
 * with none of the GPU's structure: reset_method cut into pieces with strchr and compared with strcmp, every (chain key,
 * record) pair sorted once, each bridge's run of pairs scanned in order, and each parent found by binary search.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "kxpu.h"

#define MAXD KXPU_PCIE_MAX_DEPTH
#define HOST_BRIDGE (1ull << 63)

static const char *const NAMES[7] = {"flr", "af_flr", "pm", "bus", "cxl_bus", "device_specific", "acpi"};

/* the method bits of one side record */
static uint8_t methods_of(const kxpu_resetrec *r) {
    if ((r->flags & KXPU_RS_READ_ERR) || r->len > KXPU_RESET_FILE_MAX) return 0;
    if (r->flags & KXPU_RS_ABSENT) return (r->flags & KXPU_RS_LEGACY) ? KXPU_RM_UNNAMED : 0;
    const char *t = (const char *)r->txt;
    size_t len = r->len;
    if (len > 0 && t[len - 1] == '\n') len--;
    uint8_t m = 0;
    size_t s = 0;
    for (;;) {
        size_t e = s;
        while (e < len && t[e] != ' ') e++;
        for (int k = 0; k < 7; k++)
            if (e - s == strlen(NAMES[k]) && memcmp(t + s, NAMES[k], e - s) == 0) m |= (uint8_t)(1u << k);
        if (e >= len) break;
        s = e + 1;
    }
    return m;
}

static int driver_is(const char f[16], const char *d, size_t dl) {
    size_t fl = 0;
    while (fl < 16 && f[fl]) fl++;
    return fl == dl && memcmp(f, d, dl) == 0;
}

typedef struct { uint64_t key; uint32_t j; } pair_t;

static int pair_cmp(const void *a, const void *b) {
    const pair_t *x = a, *y = b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return x->j < y->j ? -1 : x->j > y->j;
}

typedef struct { uint64_t key; uint32_t bad, lo_g, lo_j, hi_g, hi_j; } bridge_t;

static int bridge_find(const bridge_t *b, size_t nb, uint64_t key) {
    size_t lo = 0, hi = nb;
    while (lo < hi) {
        const size_t mid = (lo + hi) / 2;
        if (b[mid].key < key) lo = mid + 1;
        else hi = mid;
    }
    return lo < nb && b[lo].key == key ? (int)lo : -1;
}

/* 0; -1 (nothing written) for a decreasing group_off or a member index >= n.  chain[i * MAXD + t] / clen[i]: record i's
 * chain (clen 0: unknown path) */
int kxs_reset_check(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, const uint64_t *chain,
                    const uint8_t *clen, const kxpu_resetrec *rrs, size_t n, uint32_t allow, const uint32_t *goff,
                    const uint32_t *gmem, size_t G, uint8_t *methods, uint32_t *set_verdict, uint32_t *group_reset) {
    for (size_t g = 0; g < G; g++) {
        if (goff[g + 1] < goff[g]) return -1;
        for (uint32_t m = goff[g]; m < goff[g + 1]; m++)
            if (gmem[m] >= n) return -1;
    }
    uint8_t *bound = malloc(n + 1);
    for (size_t j = 0; j < n; j++) {
        int b = 0;
        for (size_t r = 0; r < n_rules; r++) b |= driver_is(recs[j].driver, rules[r].driver, strnlen(rules[r].driver, 16));
        bound[j] = (uint8_t)(b && !(recs[j].flags & (KXPU_REC_DRIVER_ERR | KXPU_REC_IOMMU_ERR | KXPU_REC_IS_DIR)));
        methods[j] = methods_of(&rrs[j]);
    }
    pair_t *pairs = malloc((n * MAXD + 1) * sizeof *pairs);
    size_t np = 0;
    for (size_t j = 0; j < n; j++)
        for (int t = 0; t < clen[j]; t++)
            if (!(chain[j * MAXD + t] & HOST_BRIDGE)) pairs[np++] = (pair_t){chain[j * MAXD + t], (uint32_t)j};
    qsort(pairs, np, sizeof *pairs, pair_cmp);
    bridge_t *br = malloc((np + 1) * sizeof *br);
    size_t nb = 0;
    for (size_t p = 0; p < np;) {
        bridge_t b = {pairs[p].key, KXPU_RESET_SET_OK, 0, 0, 0, 0};
        int any = 0;
        size_t q = p;
        for (; q < np && pairs[q].key == b.key; q++) {  /* ascending j: the first hit is the lowest */
            const uint32_t j = pairs[q].j, g = recs[j].iommu_group;
            if (!bound[j]) {
                if (b.bad == KXPU_RESET_SET_OK) b.bad = j;
                continue;
            }
            if (!any || g < b.lo_g) { b.lo_g = g; b.lo_j = j; }
            if (!any || g > b.hi_g) { b.hi_g = g; b.hi_j = j; }
            any = 1;
        }
        br[nb++] = b;
        p = q;
    }
    for (size_t i = 0; i < n; i++) {
        if (!clen[i]) { set_verdict[i] = KXPU_RESET_NO_PATH; continue; }
        const uint64_t parent = chain[i * MAXD + clen[i] - 1];
        if (parent & HOST_BRIDGE) { set_verdict[i] = KXPU_RESET_ROOT_BUS; continue; }
        const bridge_t *b = &br[bridge_find(br, nb, parent)];  /* i's own pair is there */
        if (b->bad != KXPU_RESET_SET_OK) set_verdict[i] = b->bad;
        else if (b->lo_g == b->hi_g) set_verdict[i] = KXPU_RESET_SET_OK;
        else set_verdict[i] = recs[i].iommu_group != b->lo_g ? b->lo_j : b->hi_j;
    }
    for (size_t g = 0; g < G; g++) {
        group_reset[g] = KXPU_VIABLE;
        for (uint32_t m = goff[g]; m < goff[g + 1]; m++) {
            const uint32_t i = gmem[m];
            const int fn = (methods[i] & allow) != 0 || ((methods[i] & KXPU_RM_UNNAMED) && allow == KXPU_RM_ALL);
            if (!fn && set_verdict[i] != KXPU_RESET_SET_OK && i < group_reset[g]) group_reset[g] = i;
        }
    }
    free(bound);
    free(pairs);
    free(br);
    return 0;
}
