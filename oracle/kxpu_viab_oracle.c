/*
 * kxpu_viab_oracle.c -- CPU checker of IOMMU group viability (include/kxpu.h, ABI v8):
 *   kxo_classify_viable   kxpu_classify_viable
 * TEST INFRASTRUCTURE ONLY.  A sequential walk: the grouping is the any-vendor oracle's (kxo_classify_rules, or
 * kxo_classify_topo with masks), then one more pass in walk order records the first blocker of every IOMMU group,
 * and every group ordinal looks its id up.  None of the GPU's structure: no shared table, no atomics.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/kxpu.h"
#include "kxpu_oracle.h"

/* readIDFromFile: data[2:] with '\n' trimmed at both ends; -1 when the file is shorter than 2 or longer than 8 bytes */
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

/* the candidate test of kxpu_classify_rules: every read worked and (vendor, driver) is one of the rules */
static int is_candidate(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *r) {
    if (r->flags & (KXPU_REC_IS_DIR | KXPU_REC_VENDOR_ERR | KXPU_REC_DRIVER_ERR | KXPU_REC_IOMMU_ERR)) return 0;
    uint8_t id[8];
    const int l = read_id(r->vendor_txt, r->vendor_len, id);
    if (l < 0) return 0;
    for (size_t q = 0; q < n_rules; q++)
        if ((size_t)l == strnlen(rules[q].vendor, 8) && memcmp(id, rules[q].vendor, (size_t)l) == 0 &&
            strncmp(r->driver, rules[q].driver, 16) == 0)
            return 1;
    return 0;
}

/* the slot holding key g, or the empty slot where it would go */
static size_t slot_of(const uint32_t *keys, size_t cap, uint32_t g) {
    size_t k = (size_t)((g * 0x9E3779B97F4A7C15ull) >> 24) & (cap - 1);
    while (keys[k] != g && keys[k] != 0xFFFFFFFFu) k = (k + 1) & (cap - 1);
    return k;
}

/* 0, KXPU_E_INVALID (rule list) or KXPU_E_UNSUPPORTED (a blocker of group 0xFFFFFFFF) */
int32_t kxo_classify_viable(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, size_t n,
                            kxpu_classify_out *out, uint8_t *dev_rule, uint64_t *group_numa, uint32_t *group_blocker) {
    const int32_t rc = group_numa ? kxo_classify_topo(rules, n_rules, recs, n, out, dev_rule, group_numa)
                                  : kxo_classify_rules(rules, n_rules, recs, n, out, dev_rule);
    if (rc != 0) return rc;
    /* group id -> first blocker: an open-addressing map, keys in slot order, 0xFFFFFFFF marks an empty slot (that id
     * is outside the domain, so it is never a key) */
    size_t cap = 16;
    while (cap < 2 * n + 2) cap <<= 1;
    uint32_t *bg = malloc(cap * 4), *bi = malloc(cap * 4);
    memset(bg, 0xff, cap * 4);
    int32_t res = 0;
    for (size_t i = 0; i < n; i++) {
        const kxpu_devrec *r = &recs[i];
        if (!(r->flags & KXPU_REC_BLOCKS) || (r->flags & KXPU_REC_IS_DIR) || is_candidate(rules, n_rules, r)) continue;
        if (r->iommu_group == 0xFFFFFFFFu) { res = KXPU_E_UNSUPPORTED; break; }
        size_t k = slot_of(bg, cap, r->iommu_group);
        if (bg[k] == 0xFFFFFFFFu) { bg[k] = r->iommu_group; bi[k] = (uint32_t)i; }  /* walk order: the first one stays */
    }
    if (res == 0) {
        for (uint32_t g = 0; g < out->n_groups; g++) {
            const size_t k = slot_of(bg, cap, out->group_ids[g]);
            group_blocker[g] = bg[k] == 0xFFFFFFFFu ? KXPU_VIABLE : bi[k];
        }
    }
    free(bg);
    free(bi);
    return res;
}
