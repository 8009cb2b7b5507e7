/*
 * dra_pcie_oracle.c -- CPU checker of kxpu_pcie_ports and kxpu_dra_slices_pcie (include/kxpu.h, additions to ABI v14),
 * the C statement next to the Python one (tests/pyref_dra_pcie.py).
 * TEST INFRASTRUCTURE ONLY: tests/dra_pcie_oracle.py compiles it into a temporary directory.  It builds on
 * dra_pf_oracle.c (included: its buffers, argument checks, record domain and taint writer).  Paths are parsed one
 * character at a time with no lanes or ballots, and each device's attributes are collected as (key, value) pairs and
 * sorted with qsort / strcmp, so no insertion position is computed.  kxd_dra_slices_pcie returns the product call's
 * status codes; on KXPU_E_UNSUPPORTED *why is the index of the first rule the first record outside the domain breaks:
 * kxd_dra_slices_pf's record rules, the two port rules, then taint_since, then a duplicate taint.
 */
#include "dra_pf_oracle.c"

#define MAXD KXPU_PCIE_MAX_DEPTH

static int hexv(char c) { return (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : -1; }

/* component s[0, l): 0 not a component, 1 function, 2 host bridge; *key its node key */
static int comp(const char *s, size_t l, uint64_t *key) {
    int hb = 0;
    if (l >= 3 && memcmp(s, "pci", 3) == 0) { hb = 1; s += 3; l -= 3; }
    size_t dl = 0;
    uint64_t dom = 0;
    while (dl < l && s[dl] != ':') {
        if (hexv(s[dl]) < 0 || dl == 8) return 0;
        dom = dom << 4 | (uint64_t)hexv(s[dl]);
        dl++;
    }
    if (!(dl == 4 || (dl >= 5 && dl <= 8 && s[0] != '0'))) return 0;
    const char *r = s + dl;
    const size_t rl = l - dl;
    if (hb) {
        if (rl != 3 || r[0] != ':' || hexv(r[1]) < 0 || hexv(r[2]) < 0) return 0;
        *key = 1ull << 63 | dom << 16 | (uint64_t)(hexv(r[1]) << 4 | hexv(r[2])) << 8;
        return 2;
    }
    if (rl != 8 || r[0] != ':' || r[3] != ':' || r[6] != '.') return 0;
    const int b0 = hexv(r[1]), b1 = hexv(r[2]), d0 = hexv(r[4]), d1 = hexv(r[5]), f = r[7] - '0';
    if (b0 < 0 || b1 < 0 || d0 < 0 || d1 < 0 || f < 0 || f > 7 || (d0 << 4 | d1) > 0x1f) return 0;
    *key = dom << 16 | (uint64_t)(b0 << 4 | b1) << 8 | (uint64_t)(d0 << 4 | d1) << 3 | (uint64_t)f;
    return 1;
}

/* the chain of record i into k; its length, 0 when the path is unknown */
static int chain_of(const kxpu_devrec *rec, const kxpu_pcipath *p, uint64_t *k) {
    const size_t len = p->len;
    if (len == 0 || len > 120) return 0;
    uint64_t keys[MAXD + 1];
    int nc = 0, kind = 0;
    size_t start = 0;
    for (size_t c = 0; c <= len; c++) {
        if (c < len && p->path[c] != '/') continue;
        if (nc == MAXD + 1) return 0;
        kind = comp(p->path + start, c - start, &keys[nc]);
        if (!kind || (nc == 0 && kind != 2)) return 0;
        if (c == len) {  /* the last: the function itself */
            const size_t bl = strnlen(rec->bdf, sizeof rec->bdf);
            if (c - start != bl || memcmp(p->path + start, rec->bdf, bl) != 0) return 0;
        }
        nc++;
        start = c + 1;
    }
    if (nc < 2) return 0;
    memcpy(k, keys, (size_t)(nc - 1) * sizeof(uint64_t));
    return nc - 1;
}

int32_t kxd_pcie_ports(const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n, const uint32_t *goff,
                       const uint32_t *gmem, size_t G, uint64_t *root_port, uint64_t *pcie_switch) {
    for (size_t g = 0; g < G; g++)
        if (goff[g + 1] < goff[g]) return KXPU_E_INVALID;
    for (size_t m = 0; m < (G ? goff[G] : 0); m++)
        if (gmem[m] >= n) return KXPU_E_INVALID;
    for (size_t g = 0; g < G; g++) {
        uint64_t pre[MAXD], k[MAXD];
        int L = -1;
        for (uint32_t m = goff[g]; m < goff[g + 1]; m++) {
            const int l = chain_of(&recs[gmem[m]], &paths[gmem[m]], k);
            if (!l) continue;
            if (L < 0) { memcpy(pre, k, sizeof k); L = l; continue; }
            int t = 0;
            while (t < L && t < l && pre[t] == k[t]) t++;
            L = t;
        }
        int hb = -1;
        for (int t = 0; t < L; t++)
            if (pre[t] >> 63) hb = t;
        const int nf = L > 0 ? L - hb - 1 : 0;  /* functions after the last host bridge */
        root_port[g] = nf >= 1 ? pre[hb + 1] : KXPU_PCIE_NO_KEY;
        int j = nf - 1;
        if (j % 2 == 0) j--;
        pcie_switch[g] = j >= 1 ? pre[hb + 1 + j] : KXPU_PCIE_NO_KEY;
    }
    return KXPU_OK;
}

static int domain_ok(const char *d) {
    if (!subdomain_ok(d, 63)) return 0;
    const size_t l = strlen(d);
    const char *reserved[2] = {"kubernetes.io", "k8s.io"};
    for (int r = 0; r < 2; r++) {
        const size_t rl = strlen(reserved[r]);
        if (strcmp(d, reserved[r]) == 0 || (l > rl && d[l - rl - 1] == '.' && strcmp(d + l - rl, reserved[r]) == 0)) return 0;
    }
    return 1;
}

static void address(char *o, uint64_t k) {
    const unsigned long long dom = k >> 16;
    snprintf(o, 24, dom <= 0xffff ? "%04llx:%02x:%02x.%u" : "%llx:%02x:%02x.%u", dom, (unsigned)(k >> 8 & 0xff),
             (unsigned)(k >> 3 & 0x1f), (unsigned)(k & 7));
}

typedef struct { char key[96]; char val[96]; } attr_t;
static int attr_cmp(const void *a, const void *b) { return strcmp(((const attr_t *)a)->key, ((const attr_t *)b)->key); }

static void str_attr(attr_t *a, const char *key, const char *v, size_t l) {
    snprintf(a->key, sizeof a->key, "%s", key);
    snprintf(a->val, sizeof a->val, "{\"string\":\"%.*s\"}", (int)l, v);
}

/* {"name":"vfio<g>","attributes":{...}  without the device's closing '}' */
static void put_device_pcie(buf_t *b, const kxpu_dradevpcie *r, const char *domain) {
    const kxpu_dradev *d = &r->pf.dev;
    attr_t a[11];
    int na = 0;
    char tmp[96];
    str_attr(&a[na++], "deviceID", d->device, strnlen(d->device, 8));
    snprintf(a[na].key, sizeof a[na].key, "iommuGroup");
    snprintf(a[na++].val, sizeof a[0].val, "{\"int\":%u}", d->iommu_group);
    if (d->numa_mask && !(d->numa_mask & (d->numa_mask - 1))) {
        snprintf(a[na].key, sizeof a[na].key, "numaNode");
        snprintf(a[na++].val, sizeof a[0].val, "{\"int\":%d}", __builtin_ctzll(d->numa_mask));
    }
    str_attr(&a[na++], "pciAddress", d->bdf, strnlen(d->bdf, 16));
    if (r->pf.physfn[0]) str_attr(&a[na++], "physfnAddress", r->pf.physfn, strnlen(r->pf.physfn, 16));
    if (r->pf.physfn_device[0]) str_attr(&a[na++], "physfnDeviceID", r->pf.physfn_device, strnlen(r->pf.physfn_device, 8));
    if (d->product_len) str_attr(&a[na++], "productName", (const char *)d->product, d->product_len);
    if (d->pcie_root[0]) str_attr(&a[na++], "resource.kubernetes.io/pcieRoot", d->pcie_root, strnlen(d->pcie_root, 16));
    str_attr(&a[na++], "vendorID", d->vendor, strnlen(d->vendor, 8));
    if (r->root_port != KXPU_PCIE_NO_KEY) {
        char key[96];
        address(tmp, r->root_port);
        snprintf(key, sizeof key, "%s/pcieRootPort", domain);
        str_attr(&a[na++], key, tmp, strlen(tmp));
    }
    if (r->pcie_switch != KXPU_PCIE_NO_KEY) {
        char key[96];
        address(tmp, r->pcie_switch);
        snprintf(key, sizeof key, "%s/pcieSwitch", domain);
        str_attr(&a[na++], key, tmp, strlen(tmp));
    }
    qsort(a, (size_t)na, sizeof a[0], attr_cmp);
    put(b, "{\"name\":\"vfio%u\",\"attributes\":{", d->iommu_group);
    for (int k = 0; k < na; k++) put(b, "%s\"%s\":%s", k ? "," : "", a[k].key, a[k].val);
    put(b, "}");
}

/* 0 = in the domain, else 1 + the index of the first failing rule */
static int record_why_pcie(const kxpu_dradevpcie *r) {
    const int w = record_why(&r->pf);
    if (w) return w;
    const uint64_t rp = r->root_port, sw = r->pcie_switch;
    if ((rp != KXPU_PCIE_NO_KEY && rp >> 48) || (sw != KXPU_PCIE_NO_KEY && sw >> 48)) return N_RULES + 1;
    if (sw != KXPU_PCIE_NO_KEY && rp == KXPU_PCIE_NO_KEY) return N_RULES + 2;
    return 0;
}
#define N_RULES_PCIE (N_RULES + 2)

int32_t kxd_dra_slices_pcie(const char *driver, const char *pool, const char *node, uint64_t generation, const char *domain,
                            const kxpu_dradevpcie *devs, size_t n, const kxpu_dra_taint *tab, size_t nt,
                            const int64_t *since, uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off,
                            size_t *n_slices, int32_t *why) {
    if (!len || !n_slices || (n && !devs)) return KXPU_E_INVALID;
    if (!subdomain_ok(driver, 63) || !subdomain_ok(pool, 253) || !subdomain_ok(node, 253) || generation >= (1ull << 63))
        return KXPU_E_INVALID;
    if (!domain || !domain_ok(domain)) return KXPU_E_INVALID;
    if (since) {
        if (!tab || nt == 0 || nt > KXPU_DRA_MAX_TAINTS) return KXPU_E_INVALID;
        for (size_t t = 0; t < nt; t++)
            if (!taint_ok(&tab[t])) return KXPU_E_INVALID;
    }
    if (n >= KXPU_DRA_MAX_DEVICES) return KXPU_E_UNSUPPORTED;
    for (size_t i = 0; i < n; i++) {
        int w = record_why_pcie(&devs[i]);
        for (size_t t = 0; since && !w && t < nt; t++)
            if (since[i * nt + t] > KXPU_DRA_TAINT_SINCE_MAX) w = N_RULES_PCIE + 1;
        for (size_t t = 0; since && !w && t < nt; t++)
            for (size_t j = 0; !w && j < t; j++)
                if (since[i * nt + t] >= 0 && since[i * nt + j] >= 0 && strcmp(tab[t].key, tab[j].key) == 0 &&
                    strcmp(tab[t].effect, tab[j].effect) == 0)
                    w = N_RULES_PCIE + 2;
        if (w) {
            if (why) *why = w - 1;
            return KXPU_E_UNSUPPORTED;
        }
    }
    const size_t per = since ? KXPU_DRA_TAINT_SLICE_DEVICES : KXPU_DRA_SLICE_DEVICES;
    const size_t slices = n ? (n + per - 1) / per : 1;
    buf_t b = {0, 0, 0};
    uint64_t *offs = malloc((slices + 1) * sizeof(uint64_t));
    if (!offs) abort();
    for (size_t s = 0; s < slices; s++) {
        offs[s] = b.len;
        put(&b, "{\"kind\":\"ResourceSlice\",\"apiVersion\":\"resource.k8s.io/v1\",\"metadata\":{\"generateName\":\"%s-%s-\"},",
            node, driver);
        put(&b, "\"spec\":{\"driver\":\"%s\",\"pool\":{\"name\":\"%s\",", driver, pool);
        put(&b, "\"generation\":%llu,\"resourceSliceCount\":%zu},\"nodeName\":\"%s\",\"devices\":[",
            (unsigned long long)generation, slices, node);
        const size_t end = (s + 1) * per < n ? (s + 1) * per : n;
        for (size_t i = s * per; i < end; i++) {
            if (i > s * per) put(&b, ",");
            put_device_pcie(&b, &devs[i], domain);
            int any = 0;
            for (size_t t = 0; since && t < nt; t++) any |= since[i * nt + t] >= 0;
            if (any) put_taints(&b, tab, nt, since + i * nt);
            put(&b, "}");
        }
        put(&b, "]}}\n");
    }
    offs[slices] = b.len;
    *len = b.len;
    *n_slices = slices;
    int32_t rc = KXPU_OK;
    if (!out || cap < b.len) rc = KXPU_E_NOSPACE;
    else {
        memcpy(out, b.p, b.len);
        if (slice_off) memcpy(slice_off, offs, (slices + 1) * sizeof(uint64_t));
    }
    free(b.p);
    free(offs);
    return rc;
}
