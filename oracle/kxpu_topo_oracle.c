/*
 * kxpu_topo_oracle.c -- CPU checker of the NUMA topology calls (include/kxpu.h, ABI v5):
 *   kxo_classify_topo / kxo_classify_mdev_topo   kxpu_classify_topo / kxpu_classify_mdev_topo
 *   kxo_lw_encode_topo                           kxpu_lw_encode_topo
 *   kxo_preferred_allocation                     kxpu_preferred_allocation
 * TEST INFRASTRUCTURE ONLY.  The grouping is the any-vendor and vGPU oracles' (kxo_classify_rules,
 * kxo_mdev_classify); the masks, the wire bytes and the allocation rule are restated here one item at a time, with
 * none of the GPU's structure: a sequential walk over the groups, one Device after the other, and per request a
 * sort of the candidates by (bin rank, position).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/kxpu.h"

int32_t kxo_classify_rules(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, size_t n,
                           kxpu_classify_out *out, uint8_t *dev_rule);                 /* kxpu_xpu_oracle.c  */
int32_t kxo_mdev_classify(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs, size_t n,
                          kxpu_classify_out *out, uint8_t *dev_rule);                  /* kxpu_mdev_oracle.c */

/* mask of group g = OR of 1 << numa_node over its members (the accepted records) that carry a valid node */
static void group_masks(const kxpu_classify_out *out, const uint8_t *flags, const uint8_t *node, size_t stride,
                        uint64_t *group_numa) {
    for (uint32_t g = 0; g < out->n_groups; g++) {
        uint64_t m = 0;
        for (uint32_t k = out->group_off[g]; k < out->group_off[g + 1]; k++) {
            const size_t i = out->group_members[k];
            if ((flags[i * stride] & KXPU_REC_NUMA) && node[i * stride] < KXPU_MAX_NUMA_NODES) m |= 1ull << node[i * stride];
        }
        group_numa[g] = m;
    }
}

int32_t kxo_classify_topo(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs, size_t n,
                          kxpu_classify_out *out, uint8_t *dev_rule, uint64_t *group_numa) {
    const int32_t rc = kxo_classify_rules(rules, n_rules, recs, n, out, dev_rule);
    if (rc == 0 && n) group_masks(out, &recs[0].flags, &recs[0].numa_node, sizeof *recs, group_numa);
    return rc;
}

int32_t kxo_classify_mdev_topo(const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs, size_t n,
                               kxpu_classify_out *out, uint8_t *dev_rule, uint64_t *group_numa) {
    const int32_t rc = kxo_mdev_classify(rules, n_rules, recs, n, out, dev_rule);
    if (rc == 0 && n) group_masks(out, &recs[0].flags, &recs[0].numa_node, sizeof *recs, group_numa);
    return rc;
}

/* ---------------------------------------------------------------- ListAndWatchResponse with topology */
static size_t put_varint(uint8_t *o, size_t at, size_t cap, uint64_t v) {
    do {
        uint8_t b = (uint8_t)(v & 0x7f);
        v >>= 7;
        if (v) b |= 0x80;
        if (o && at < cap) o[at] = b;
        at++;
    } while (v);
    return at;
}
static size_t varint_size(uint64_t v) { return put_varint(NULL, 0, 0, v); }
static size_t put_bytes(uint8_t *o, size_t at, size_t cap, const void *b, size_t len) {
    for (size_t k = 0; k < len; k++) if (o && at + k < cap) o[at + k] = ((const uint8_t *)b)[k];
    return at + len;
}

/* one Device: returns the bytes it takes; writes them when o != NULL */
static size_t device_bytes(uint32_t group, int healthy, uint64_t mask, uint8_t *o, size_t at, size_t cap) {
    char id[16];
    size_t il = 0;
    uint32_t v = group;
    char rev[16];
    do { rev[il++] = (char)('0' + v % 10); v /= 10; } while (v);
    for (size_t k = 0; k < il; k++) id[k] = rev[il - 1 - k];
    const char *health = healthy ? "Healthy" : "Unhealthy";
    const size_t hl = strlen(health);
    /* TopologyInfo body: one NUMANode per node */
    size_t topo = 0;
    for (int k = 0; k < 64; k++) {
        if (!((mask >> k) & 1)) continue;
        const size_t node_body = k ? 1 + varint_size((uint64_t)k) : 0;
        topo += 1 + varint_size(node_body) + node_body;
    }
    size_t body = 1 + varint_size(il) + il + 1 + varint_size(hl) + hl;
    if (mask) body += 1 + varint_size(topo) + topo;
    const size_t start = at;
    at = put_bytes(o, at, cap, "\x0a", 1);
    at = put_varint(o, at, cap, body);
    at = put_bytes(o, at, cap, "\x0a", 1);
    at = put_varint(o, at, cap, il);
    at = put_bytes(o, at, cap, id, il);
    at = put_bytes(o, at, cap, "\x12", 1);
    at = put_varint(o, at, cap, hl);
    at = put_bytes(o, at, cap, health, hl);
    if (mask) {
        at = put_bytes(o, at, cap, "\x1a", 1);
        at = put_varint(o, at, cap, topo);
        for (int k = 0; k < 64; k++) {
            if (!((mask >> k) & 1)) continue;
            const size_t node_body = k ? 1 + varint_size((uint64_t)k) : 0;
            at = put_bytes(o, at, cap, "\x0a", 1);
            at = put_varint(o, at, cap, node_body);
            if (k) { at = put_bytes(o, at, cap, "\x08", 1); at = put_varint(o, at, cap, (uint64_t)k); }
        }
    }
    return at - start;
}

/* total bytes; out (cap bytes) may be NULL */
size_t kxo_lw_encode_topo(const uint32_t *group_ids, const uint8_t *healthy, const uint64_t *masks, size_t n, uint8_t *out,
                          size_t cap) {
    size_t at = 0;
    for (size_t i = 0; i < n; i++)
        at += device_bytes(group_ids[i], !healthy || healthy[i], masks ? masks[i] : 0, out, at, cap);
    return at;
}

/* ---------------------------------------------------------------- preferred allocation */
static uint32_t home_of(uint64_t m) {
    for (uint32_t k = 0; k < 64; k++) if ((m >> k) & 1) return k;
    return 64;
}

typedef struct { uint32_t rank, pos; } cand;
static int cand_cmp(const void *a, const void *b) {
    const cand *x = a, *y = b;
    if (x->rank != y->rank) return x->rank < y->rank ? -1 : 1;
    return x->pos < y->pos ? -1 : x->pos > y->pos;
}

/* 0, or -1 when a request is invalid (then out is unspecified); out_off[n_req + 1] is always filled up to the
 * first invalid request */
int32_t kxo_preferred_allocation(const uint64_t *dev_numa, size_t n_devs, const uint32_t *avail_off, const uint32_t *avail,
                                 const uint32_t *must_off, const uint32_t *must, const uint32_t *size, size_t n_req,
                                 uint32_t *out, uint32_t *out_off) {
    uint8_t *mark = calloc(n_devs ? n_devs : 1, 1);
    cand *cs = NULL;
    size_t cs_cap = 0;
    int32_t rc = 0;
    out_off[0] = 0;
    for (size_t q = 0; q < n_req && rc == 0; q++) {
        const uint32_t *av = avail + avail_off[q], *mu = must + must_off[q];
        const size_t na = avail_off[q + 1] - avail_off[q], nm = must_off[q + 1] - must_off[q];
        if (size[q] < nm || size[q] > na) { rc = -1; break; }
        out_off[q + 1] = out_off[q] + size[q];
        /* validation: positions, duplicates, must within available */
        for (size_t j = 0; j < na && rc == 0; j++) {
            if (av[j] >= n_devs || (mark[av[j]] & 1)) rc = -1;
            else mark[av[j]] |= 1;
        }
        for (size_t j = 0; j < nm && rc == 0; j++) {
            if (mu[j] >= n_devs || (mark[mu[j]] & 2) || !(mark[mu[j]] & 1)) rc = -1;
            else mark[mu[j]] |= 2;
        }
        if (rc == 0) {
            uint64_t U = 0;
            uint32_t c[65] = {0};
            for (size_t j = 0; j < nm; j++) {
                const uint32_t h = home_of(dev_numa[mu[j]]);
                if (h < 64) U |= 1ull << h;
            }
            for (size_t j = 0; j < na; j++) if (mark[av[j]] == 1) c[home_of(dev_numa[av[j]])]++;
            /* bin ranks: a selection over the 65 bins in (group, c descending, k ascending) order */
            uint32_t rank[65];
            int used[65] = {0};
            for (uint32_t r = 0; r < 65; r++) {
                int best = -1;
                for (uint32_t k = 0; k < 65; k++) {
                    if (used[k]) continue;
                    if (best < 0) { best = (int)k; continue; }
                    const int gk = k == 64 ? 2 : (((U >> k) & 1) ? 0 : 1), gb = best == 64 ? 2 : (((U >> best) & 1) ? 0 : 1);
                    if (gk < gb || (gk == gb && c[k] > c[best])) best = (int)k;  /* ties keep the lower k */
                }
                used[best] = 1;
                rank[best] = r;
            }
            if (na > cs_cap) { cs_cap = na; cs = realloc(cs, cs_cap * sizeof *cs); }
            size_t nc = 0;
            for (size_t j = 0; j < na; j++)
                if (mark[av[j]] == 1) { cs[nc].rank = rank[home_of(dev_numa[av[j]])]; cs[nc].pos = av[j]; nc++; }
            qsort(cs, nc, sizeof *cs, cand_cmp);
            uint32_t *o = out + out_off[q];
            for (size_t j = 0; j < nm; j++) o[j] = mu[j];
            for (size_t j = 0; j < size[q] - nm; j++) o[nm + j] = cs[j].pos;
        }
        for (size_t j = 0; j < na; j++) if (av[j] < n_devs) mark[av[j]] = 0;
        for (size_t j = 0; j < nm; j++) if (mu[j] < n_devs) mark[mu[j]] = 0;
    }
    free(cs);
    free(mark);
    return rc;
}
