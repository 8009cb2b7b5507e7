/*
 * kxpu_reconcile_oracle.c -- CPU checker of kxpu_reconcile (include/kxpu.h, ABI v6):
 *   kxo_reconcile                                kxpu_reconcile
 * TEST INFRASTRUCTURE ONLY.  The rule is restated with none of the GPU's structure: both lists are sorted by key
 * (qsort of positions), duplicates are adjacent equal keys, each cur entry finds its prev entry by binary search, and
 * the fresh indices are handed out by one sequential pass in walk order.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/kxpu.h"

static const kxpu_snaprec *g_sort_base;

static int cmp_pos(const void *a, const void *b) {
    const uint32_t x = *(const uint32_t *)a, y = *(const uint32_t *)b;
    return memcmp(g_sort_base[x].key, g_sort_base[y].key, sizeof g_sort_base[x].key);
}

/* positions of recs[0..n) sorted by key (not thread-safe: the checker runs single-threaded) */
static uint32_t *sorted_positions(const kxpu_snaprec *recs, size_t n) {
    uint32_t *p = (uint32_t *)malloc((n ? n : 1) * sizeof *p);
    for (size_t i = 0; i < n; i++) p[i] = (uint32_t)i;
    g_sort_base = recs;
    qsort(p, n, sizeof *p, cmp_pos);
    return p;
}

static int key_ok(const char *k) {
    if (k[0] == 0) return 0;
    int nul = 0;
    for (int b = 0; b < 40; b++) {
        if (k[b] == 0) nul = 1;
        else if (nul) return 0;
    }
    return 1;
}

static int has_dup(const kxpu_snaprec *recs, const uint32_t *pos, size_t n) {
    for (size_t i = 1; i < n; i++)
        if (memcmp(recs[pos[i - 1]].key, recs[pos[i]].key, 40) == 0) return 1;
    return 0;
}

int32_t kxo_reconcile(const kxpu_snaprec *prev, size_t n_prev, uint64_t next_index, const kxpu_snaprec *cur, size_t n_cur,
                      uint64_t *index_out, uint8_t *cur_state, uint8_t *prev_state, kxpu_reconcile_counts *counts) {
    if (next_index + (uint64_t)n_cur < next_index) return KXPU_E_INVALID;
    for (size_t j = 0; j < n_prev; j++)
        if (!key_ok(prev[j].key) || prev[j].index >= next_index) return KXPU_E_INVALID;
    for (size_t i = 0; i < n_cur; i++)
        if (!key_ok(cur[i].key)) return KXPU_E_INVALID;
    uint32_t *pp = sorted_positions(prev, n_prev), *cp = sorted_positions(cur, n_cur);
    const int dup = has_dup(prev, pp, n_prev) || has_dup(cur, cp, n_cur);
    free(cp);
    if (dup) { free(pp); return KXPU_E_INVALID; }
    uint64_t next = next_index, kept = 0, changed = 0;
    for (size_t j = 0; j < n_prev; j++) prev_state[j] = KXPU_RC_RETIRED;
    for (size_t i = 0; i < n_cur; i++) {
        size_t lo = 0, hi = n_prev;  /* first prev position (in key order) whose key >= cur[i].key */
        while (lo < hi) {
            const size_t mid = (lo + hi) / 2;
            if (memcmp(prev[pp[mid]].key, cur[i].key, 40) < 0) lo = mid + 1;
            else hi = mid;
        }
        const int found = lo < n_prev && memcmp(prev[pp[lo]].key, cur[i].key, 40) == 0;
        if (!found) {
            cur_state[i] = KXPU_RC_NEW;
            index_out[i] = next++;
            continue;
        }
        const kxpu_snaprec *p = &prev[pp[lo]];
        if (p->iommu_group == cur[i].iommu_group && p->klass == cur[i].klass && p->tag == cur[i].tag) {
            cur_state[i] = prev_state[pp[lo]] = KXPU_RC_KEPT;
            index_out[i] = p->index;
            kept++;
        } else {
            cur_state[i] = prev_state[pp[lo]] = KXPU_RC_CHANGED;
            index_out[i] = next++;
            changed++;
        }
    }
    free(pp);
    counts->n_kept = kept;
    counts->n_changed = changed;
    counts->n_new = n_cur - kept - changed;
    counts->n_retired = n_prev - kept - changed;
    counts->next_index_out = next;
    return KXPU_OK;
}
