/*
 * vf_vgpu_health_oracle.c -- CPU checker of kxpu_vf_vgpu_drift (include/kxpu.h, additions to ABI v14), the C statement
 * next to the Python one (tests/pyref_vf_vgpu_health.py).
 * TEST INFRASTRUCTURE ONLY: tests/vf_vgpu_health_oracle.py compiles it, with tests/vf_vgpu_oracle.c, into a temporary
 * directory.  The current type of a record is the one kxv_vf_vgpu_types (tests/vf_vgpu_oracle.c) gives it, so the drift
 * rule here cannot read a text differently from the type join: each record is run through that checker on its own,
 * with no name table.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "kxpu.h"

int kxv_vf_vgpu_types(const kxpu_vfvgpurec *recs, size_t n, const uint8_t *blob, const uint64_t *toff, size_t n_tables,
                      kxpu_vgpukey *keys, uint32_t *type_id, uint8_t *status);

/* 0, or -1 for a decreasing group_off or a member >= n (nothing written then) */
int kxv_vf_vgpu_drift(const kxpu_vfvgpurec *recs, const uint32_t *type_was, size_t n, const uint32_t *group_off,
                      const uint32_t *group_members, size_t n_groups, uint32_t *type_now, uint8_t *status_now,
                      uint32_t *group_first) {
    for (size_t g = 0; g < n_groups; g++) {
        if (group_off[g + 1] < group_off[g]) return -1;
        for (uint32_t m = group_off[g]; m < group_off[g + 1]; m++)
            if (group_members[m] >= n) return -1;
    }
    uint8_t *st = malloc(n ? n : 1);
    uint32_t *now = malloc((n ? n : 1) * sizeof *now);
    const uint64_t toff = 0;
    for (size_t i = 0; i < n; i++) {
        kxpu_vgpukey key;
        uint32_t id = 0;
        uint8_t vt = 0;
        kxv_vf_vgpu_types(&recs[i], 1, NULL, &toff, 0, &key, &id, &vt);
        if (!(recs[i].flags & KXPU_VT_READ)) {
            now[i] = type_was[i];
            st[i] = KXPU_VD_SAME;
        } else if (vt == KXPU_VT_BAD) {
            now[i] = 0;
            st[i] = KXPU_VD_BAD;
        } else {
            now[i] = id;  /* KXPU_VT_NONE: type 0; else the ID, named by no table here */
            st[i] = id == type_was[i] ? KXPU_VD_SAME : id == 0 ? KXPU_VD_CLEARED : KXPU_VD_CHANGED;
        }
    }
    for (size_t g = 0; g < n_groups; g++) {
        group_first[g] = KXPU_VD_STEADY;
        for (uint32_t m = group_off[g]; m < group_off[g + 1]; m++)
            if (st[group_members[m]] != KXPU_VD_SAME) { group_first[g] = m - group_off[g]; break; }
    }
    if (n) {
        memcpy(type_now, now, n * sizeof *now);
        memcpy(status_now, st, n);
    }
    free(st);
    free(now);
    return 0;
}
