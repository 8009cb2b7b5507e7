/* names_oracle.c -- the C statement of kxpu_classify_named's name table (include/kxpu.h): which tables the call
 * refuses, and the slot a candidate of a rule takes for its device id.  The walk itself is stated by the C classify
 * oracles (tests/names_oracle.py).  TEST INFRASTRUCTURE ONLY. */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "kxpu.h"

/* a NUL-padded 8-byte field is 4 lowercase hex digits, or "*" (1), or neither (0) */
static int device_kind(const char *d) {
    size_t l = 0;
    while (l < 8 && d[l]) l++;
    for (size_t k = l; k < 8; k++)
        if (d[k]) return 0;
    if (l == 1 && d[0] == '*') return 1;
    if (l != 4) return 0;
    for (size_t k = 0; k < 4; k++)
        if (!((d[k] >= '0' && d[k] <= '9') || (d[k] >= 'a' && d[k] <= 'f'))) return 0;
    return 4;
}

/* 0: the table is valid for n_rules rules with vgpu_rules; -1: KXPU_E_INVALID */
int kxn_check(const kxpu_name_entry *t, size_t n_names, size_t n_rules, uint32_t vgpu_rules) {
    if (n_names > KXPU_MAX_NAMES) return -1;
    for (size_t e = 0; e < n_names; e++) {
        if (t[e].rule >= n_rules || ((vgpu_rules >> t[e].rule) & 1u)) return -1;
        if (!device_kind(t[e].device)) return -1;
        if (t[e].slot >= n_names) return -1;
        for (size_t q = 0; q < e; q++)
            if (t[q].rule == t[e].rule && memcmp(t[q].device, t[e].device, 8) == 0) return -1;
    }
    return 0;
}

/* the slot of a candidate of `rule` whose device id (readIDFromFile's text) is id[0..len): its exact entry, else its
 * rule's "*", else KXPU_NO_SLOT */
uint32_t kxn_slot(const kxpu_name_entry *t, size_t n_names, uint32_t rule, const char *id, size_t len) {
    uint32_t star = KXPU_NO_SLOT;
    for (size_t e = 0; e < n_names; e++) {
        if (t[e].rule != rule) continue;
        if (device_kind(t[e].device) == 1) star = t[e].slot;
        else if (len == 4 && memcmp(t[e].device, id, 4) == 0) return t[e].slot;
    }
    return star;
}
