/*
 * kxpu_aer_oracle.c -- CPU checker of kxpu_aer_health, kxpu_dra_slices_taints and kxpu_dra_slices_mdev_taints
 * (include/kxpu.h, ABI v12).
 *
 * kxo_aer_health reads every file front to back, line by line, and keeps the last line with the prefix: the GPU kernel
 * walks each file backward from its end, so the two share no search.  The _taints checkers write each slice with the
 * taint oracle's device writers and a taint list of their own; n_taints == 1 giving the _taint calls' bytes is then a
 * check against kxpu_dra_taint_oracle.c's put_taint, not an identity.
 *
 * TEST INFRASTRUCTURE ONLY, like kxpu_oracle.c.  Arguments and status codes are the product calls' without the context;
 * on KXPU_E_UNSUPPORTED *why names the first rule the first record outside the domain breaks (the record rules of the
 * layout, then "taint_since", then "taint_duplicate").
 *
 * This file is the root of the DRA oracles' one translation unit: it includes kxpu_dra_taint_oracle.c, which includes
 * kxpu_dra_mdev_oracle.c, which includes kxpu_dra_oracle.c, so the four share the static Buf writer and domain helpers.
 * oracle/Makefile compiles this file into libkxpu_oracle.so and not those three.
 */
#include "kxpu_dra_taint_oracle.c"

/* the count of one file, UINT64_MAX when unknown */
static uint64_t aer_count(const uint8_t *t, uint32_t len, const char *pfx) {
    const size_t pl = strlen(pfx);
    if (len == 0 || len > KXPU_AER_FILE_MAX) return UINT64_MAX;
    uint64_t count = UINT64_MAX;
    int seen = 0;
    for (uint32_t s = 0; s < len;) {
        uint32_t e = s;
        while (e < len && t[e] != '\n') e++;
        if (e - s >= pl && memcmp(t + s, pfx, pl) == 0) {  /* a later line replaces an earlier one, good or bad */
            seen = 1;
            const uint8_t *d = t + s + pl;
            const uint32_t nd = e - s - (uint32_t)pl;
            int ok = nd >= 1 && nd <= 20 && !(nd > 1 && d[0] == '0');
            unsigned __int128 v = 0;
            for (uint32_t k = 0; ok && k < nd; k++) {
                if (d[k] < '0' || d[k] > '9') ok = 0;
                else v = v * 10 + (d[k] - '0');
            }
            count = ok && v < (unsigned __int128)UINT64_MAX ? (uint64_t)v : UINT64_MAX;
        }
        s = e + 1;
    }
    return seen ? count : UINT64_MAX;
}

int32_t kxo_aer_health(const uint8_t *text, size_t text_len, const uint64_t *file_off, const uint32_t *file_len, size_t n,
                       uint64_t fatal_limit, uint64_t nonfatal_limit, const uint32_t *group_off,
                       const uint32_t *group_members, size_t n_groups, uint64_t *totals, uint8_t *group_aer) {
    if ((text_len && !text) || (n && (!file_off || !file_len)) || !group_off || (n_groups && !group_aer))
        return KXPU_E_INVALID;
    if (n >= (1ull << 28) || n_groups >= (1ull << 28)) return KXPU_E_UNSUPPORTED;
    for (size_t g = 0; g < n_groups; g++)
        if (group_off[g + 1] < group_off[g]) return KXPU_E_INVALID;
    if (group_off[n_groups] && !group_members) return KXPU_E_INVALID;
    for (size_t f = 0; f < 2 * n; f++)
        if (file_off[f] > text_len || file_len[f] > text_len - file_off[f]) return KXPU_E_INVALID;
    for (size_t m = group_off[0]; m < group_off[n_groups]; m++)
        if (group_members[m] >= n) return KXPU_E_INVALID;
    uint64_t *t = malloc((2 * n + 1) * sizeof(uint64_t));
    for (size_t f = 0; f < 2 * n; f++)
        t[f] = aer_count(text + file_off[f], file_len[f], (f & 1) ? "TOTAL_ERR_NONFATAL " : "TOTAL_ERR_FATAL ");
    for (size_t g = 0; g < n_groups; g++) {
        uint8_t bits = 0;
        for (uint32_t m = group_off[g]; m < group_off[g + 1]; m++) {
            const uint64_t tf = t[2 * group_members[m]], tn = t[2 * group_members[m] + 1];
            if (tf == UINT64_MAX || tn == UINT64_MAX) bits |= KXPU_AER_UNKNOWN;
            if (tf != UINT64_MAX && tf > fatal_limit) bits |= KXPU_AER_FATAL;
            if (tn != UINT64_MAX && tn > nonfatal_limit) bits |= KXPU_AER_NONFATAL;
        }
        group_aer[g] = bits;
    }
    if (totals) memcpy(totals, t, 2 * n * sizeof(uint64_t));
    free(t);
    return KXPU_OK;
}

/* "taints":[...] of one device, from its last attribute's closer on */
static void put_taints(Buf *b, const kxpu_dra_taint *tab, size_t nt, const int64_t *row) {
    struct tm tm;
    char ts[64];
    int first = 1;
    puts_(b, ",\"taints\":[");
    for (size_t t = 0; t < nt; t++) {
        if (row[t] < 0) continue;
        time_t tt = (time_t)row[t];
        gmtime_r(&tt, &tm);
        snprintf(ts, sizeof ts, "%04d-%02d-%02dT%02d:%02d:%02dZ", tm.tm_year + 1900, tm.tm_mon + 1, tm.tm_mday,
                 tm.tm_hour, tm.tm_min, tm.tm_sec);
        if (!first) puts_(b, ",");
        first = 0;
        puts_(b, "{\"key\":\""); puts_(b, tab[t].key); puts_(b, "\"");
        if (tab[t].value[0]) { puts_(b, ",\"value\":\""); puts_(b, tab[t].value); puts_(b, "\""); }
        puts_(b, ",\"effect\":\""); puts_(b, tab[t].effect); puts_(b, "\",\"timeAdded\":\""); puts_(b, ts); puts_(b, "\"}");
    }
    puts_(b, "]");
}

static int32_t taints_slices(int mdev, const char *driver, const char *pool, const char *node, uint64_t generation,
                             const void *devs, size_t n, const kxpu_dra_taint *tab, size_t nt, const int64_t *since,
                             uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off, size_t *n_slices, int32_t *why) {
    if (!since)  /* the untainted call: the taint oracle with no taint array gives it */
        return taint_slices(mdev, driver, pool, node, generation, devs, n, NULL, NULL, NULL, NULL, out, cap, len,
                            slice_off, n_slices, why);
    if (!len || !n_slices || (n && !devs)) return KXPU_E_INVALID;
    if (!subdomain_ok(driver, 63) || !subdomain_ok(pool, 253) || !subdomain_ok(node, 253) || generation >= (1ull << 63))
        return KXPU_E_INVALID;
    if (!tab || nt == 0 || nt > KXPU_DRA_MAX_TAINTS) return KXPU_E_INVALID;
    for (size_t t = 0; t < nt; t++)
        if (!taint_args_ok(tab[t].key, tab[t].value, tab[t].effect)) return KXPU_E_INVALID;
    if (n >= KXPU_DRA_MAX_DEVICES) return KXPU_E_UNSUPPORTED;
    const int n_rules = mdev ? 9 : 7;
    for (size_t i = 0; i < n; i++) {
        int w = mdev ? mdev_record_why((const kxpu_dramdev *)devs + i) : record_why((const kxpu_dradev *)devs + i);
        for (size_t t = 0; !w && t < nt; t++)
            if (since[i * nt + t] > KXPU_DRA_TAINT_SINCE_MAX) w = n_rules + 1;
        for (size_t t = 0; !w && t < nt; t++)
            for (size_t j = 0; !w && j < t; j++)
                if (since[i * nt + t] >= 0 && since[i * nt + j] >= 0 && strcmp(tab[t].key, tab[j].key) == 0 &&
                    strcmp(tab[t].effect, tab[j].effect) == 0)
                    w = n_rules + 2;
        if (w) {
            if (why) *why = w - 1;
            return KXPU_E_UNSUPPORTED;
        }
    }
    const size_t per = KXPU_DRA_TAINT_SLICE_DEVICES;
    size_t slices = n ? (n + per - 1) / per : 1;
    Buf b = {0, 0, 0};
    uint64_t *offs = malloc((slices + 1) * sizeof(uint64_t));
    char tmp[128];
    for (size_t s = 0; s < slices; s++) {
        offs[s] = b.n;
        puts_(&b, "{\"kind\":\"ResourceSlice\",\"apiVersion\":\"resource.k8s.io/v1\",\"metadata\":{\"generateName\":\"");
        puts_(&b, node); puts_(&b, "-"); puts_(&b, driver); puts_(&b, "-\"},\"spec\":{\"driver\":\"");
        puts_(&b, driver); puts_(&b, "\",\"pool\":{\"name\":\""); puts_(&b, pool);
        snprintf(tmp, sizeof tmp, "\",\"generation\":%llu,\"resourceSliceCount\":%zu},\"nodeName\":\"",
                 (unsigned long long)generation, slices);
        puts_(&b, tmp); puts_(&b, node); puts_(&b, "\",\"devices\":[");
        size_t end = (s + 1) * per < n ? (s + 1) * per : n;
        for (size_t i = s * per; i < end; i++) {
            if (i > s * per) puts_(&b, ",");
            if (mdev) put_mdev_device(&b, (const kxpu_dramdev *)devs + i);
            else put_pci_device(&b, (const kxpu_dradev *)devs + i);
            int any = 0;
            for (size_t t = 0; t < nt; t++) any |= since[i * nt + t] >= 0;
            if (any) put_taints(&b, tab, nt, since + i * nt);
            puts_(&b, "}");
        }
        puts_(&b, "]}}\n");
    }
    offs[slices] = b.n;
    *len = b.n;
    *n_slices = slices;
    int32_t rc = KXPU_OK;
    if (!out || cap < b.n) rc = KXPU_E_NOSPACE;
    else {
        memcpy(out, b.p, b.n);
        if (slice_off) memcpy(slice_off, offs, (slices + 1) * sizeof(uint64_t));
    }
    free(b.p);
    free(offs);
    return rc;
}

int32_t kxo_dra_slices_taints(const char *driver, const char *pool, const char *node, uint64_t generation,
                              const kxpu_dradev *devs, size_t n, const kxpu_dra_taint *taints, size_t n_taints,
                              const int64_t *taint_since, uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off,
                              size_t *n_slices, int32_t *why) {
    return taints_slices(0, driver, pool, node, generation, devs, n, taints, n_taints, taint_since, out, cap, len,
                         slice_off, n_slices, why);
}

int32_t kxo_dra_slices_mdev_taints(const char *driver, const char *pool, const char *node, uint64_t generation,
                                   const kxpu_dramdev *devs, size_t n, const kxpu_dra_taint *taints, size_t n_taints,
                                   const int64_t *taint_since, uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off,
                                   size_t *n_slices, int32_t *why) {
    return taints_slices(1, driver, pool, node, generation, devs, n, taints, n_taints, taint_since, out, cap, len,
                         slice_off, n_slices, why);
}
