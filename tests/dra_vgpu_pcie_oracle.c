/*
 * dra_vgpu_pcie_oracle.c -- CPU checker of kxpu_pcie_ports_mdev, kxpu_dra_slices_mdev_pcie and
 * kxpu_dra_slices_vf_vgpu_pcie (include/kxpu.h, additions to ABI v14), the C statement next to the Python one
 * (tests/pyref_vgpu_pcie.py).
 * TEST INFRASTRUCTURE ONLY: tests/dra_vgpu_pcie_oracle.py compiles it twice into a temporary directory: on
 * mdev_pf_oracle.c (the mdev layout and the rule) and, with -DKXD_VF, on dra_vf_vgpu_oracle.c.  Each device is written by
 * the included checker, its attributes are cut into (key, value) pairs, the two port attributes are added and the pairs
 * are sorted with qsort / strcmp, so no insertion position is computed.  The mdev path is parsed one character at a time.
 * On KXPU_E_UNSUPPORTED *why is the index of the first rule the first record outside the domain breaks: the included
 * checker's record rules, the two port rules, then taint_since, then a duplicate taint.
 */
#ifdef KXD_VF
#include "dra_vf_vgpu_oracle.c"
typedef kxpu_dravfvgpupcie prec_t;
#define BASE(r) (&(r)->dev)
#else
#include "mdev_pf_oracle.c"
typedef kxpu_dramdevpcie prec_t;
#define BASE(r) (&(r)->pf)
#endif

#define MAXD KXPU_PCIE_MAX_DEPTH

#ifndef KXD_VF
static int hx(char c) { return (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : -1; }

/* component s[0, l): 0 not a component, 1 function, 2 host bridge; *key its node key */
static int comp(const char *s, size_t l, uint64_t *key) {
    int hb = 0;
    if (l >= 3 && memcmp(s, "pci", 3) == 0) { hb = 1; s += 3; l -= 3; }
    size_t dl = 0;
    uint64_t dom = 0;
    while (dl < l && s[dl] != ':') {
        if (hx(s[dl]) < 0 || dl == 8) return 0;
        dom = dom << 4 | (uint64_t)hx(s[dl]);
        dl++;
    }
    if (!(dl == 4 || (dl >= 5 && dl <= 8 && s[0] != '0'))) return 0;
    const char *r = s + dl;
    const size_t rl = l - dl;
    if (hb) {
        if (rl != 3 || r[0] != ':' || hx(r[1]) < 0 || hx(r[2]) < 0) return 0;
        *key = 1ull << 63 | dom << 16 | (uint64_t)(hx(r[1]) << 4 | hx(r[2])) << 8;
        return 2;
    }
    if (rl != 8 || r[0] != ':' || r[3] != ':' || r[6] != '.') return 0;
    const int b0 = hx(r[1]), b1 = hx(r[2]), d0 = hx(r[4]), d1 = hx(r[5]), f = r[7] - '0';
    if (b0 < 0 || b1 < 0 || d0 < 0 || d1 < 0 || f < 0 || f > 7 || (d0 << 4 | d1) > 0x1f) return 0;
    *key = dom << 16 | (uint64_t)(b0 << 4 | b1) << 8 | (uint64_t)(d0 << 4 | d1) << 3 | (uint64_t)f;
    return 1;
}

/* the parent chain of mdev record rec into k (its chain less the parent function); its length, 0 when unknown */
static int parent_chain(const kxpu_mdevrec *rec, const kxpu_pcipath *p, uint64_t *k) {
    const size_t len = p->len;
    if (len == 0 || len > 120) return 0;
    size_t cut = len;  /* the last '/': the UUID follows */
    while (cut > 0 && p->path[cut - 1] != '/') cut--;
    if (cut == 0 || len - cut != 36 || memcmp(p->path + cut, rec->uuid, 36) != 0) return 0;
    for (int c = 0; c < 36; c++) {
        const char ch = p->path[cut + c];
        if ((c == 8 || c == 13 || c == 18 || c == 23) ? ch != '-' : hx(ch) < 0) return 0;
    }
    uint64_t keys[MAXD + 1];
    int nc = 0, kind = 0;
    size_t start = 0, plen = 0;
    for (size_t c = 0; c < cut; c++) {
        if (p->path[c] != '/') continue;
        if (nc == MAXD) return 0;
        kind = comp(p->path + start, c - start, &keys[nc]);
        if (!kind || (nc == 0 && kind != 2)) return 0;
        plen = c - start;
        nc++;
        start = c + 1;
    }
    /* the parent function: the last component before the UUID, equal to rec->parent */
    const size_t pl = strnlen(rec->parent, sizeof rec->parent);
    if (nc < 2 || kind != 1 || plen != pl || memcmp(p->path + cut - 1 - plen, rec->parent, pl) != 0) return 0;
    memcpy(k, keys, (size_t)(nc - 1) * sizeof(uint64_t));
    return nc - 1;
}

int32_t kxd_pcie_ports_mdev(const kxpu_mdevrec *recs, const kxpu_pcipath *paths, size_t n, const uint32_t *goff,
                            const uint32_t *gmem, size_t G, uint64_t *root_port, uint64_t *pcie_switch) {
    for (size_t g = 0; g < G; g++)
        if (goff[g + 1] < goff[g]) return KXPU_E_INVALID;
    for (size_t m = 0; m < (G ? goff[G] : 0); m++)
        if (gmem[m] >= n) return KXPU_E_INVALID;
    for (size_t g = 0; g < G; g++) {
        uint64_t pre[MAXD], k[MAXD];
        int L = -1;
        for (uint32_t m = goff[g]; m < goff[g + 1]; m++) {
            const int l = parent_chain(&recs[gmem[m]], &paths[gmem[m]], k);
            if (!l) continue;
            if (L < 0) { memcpy(pre, k, sizeof k); L = l; continue; }
            int t = 0;
            while (t < L && t < l && pre[t] == k[t]) t++;
            L = t;
        }
        int hb = -1;
        for (int t = 0; t < L; t++)
            if (pre[t] >> 63) hb = t;
        const int nf = L > 0 ? L - hb - 1 : 0;
        root_port[g] = nf >= 1 ? pre[hb + 1] : KXPU_PCIE_NO_KEY;
        int j = nf - 1;
        if (j % 2 == 0) j--;
        pcie_switch[g] = j >= 1 ? pre[hb + 1 + j] : KXPU_PCIE_NO_KEY;
    }
    return KXPU_OK;
}
#endif

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

typedef struct { char key[96]; char val[128]; } attr_t;
static int attr_cmp(const void *a, const void *b) { return strcmp(((const attr_t *)a)->key, ((const attr_t *)b)->key); }

static void port_attr(attr_t *a, const char *domain, const char *what, uint64_t k) {
    const unsigned long long dom = k >> 16;
    snprintf(a->key, sizeof a->key, "%s/%s", domain, what);
    snprintf(a->val, sizeof a->val, dom <= 0xffff ? "{\"string\":\"%04llx:%02x:%02x.%u\"}" : "{\"string\":\"%llx:%02x:%02x.%u\"}",
             dom, (unsigned)(k >> 8 & 0xff), (unsigned)(k >> 3 & 0x1f), (unsigned)(k & 7));
}

/* the included checker's device, its attributes cut at the commas between them (no value holds a comma), the ports
 * added, the pairs sorted; without the device's closing '}' */
static void put_device_pcie(buf_t *b, const prec_t *r, const char *domain) {
    buf_t t = {0, 0, 0};
    put_device(&t, BASE(r));
    put(&t, "%c", '\0');
    const char *s = (const char *)t.p, *open = strstr(s, "\"attributes\":{");
    const char *body = open + strlen("\"attributes\":{");
    attr_t a[16];
    int na = 0, depth = 0;
    const char *start = body;
    for (const char *c = body;; c++) {
        const int end = *c == '}' && depth == 0;
        if ((*c == ',' && depth == 0) || end) {  /* one attribute: "key":value */
            const char *kq = strchr(start + 1, '"');
            snprintf(a[na].key, sizeof a[na].key, "%.*s", (int)(kq - start - 1), start + 1);
            snprintf(a[na].val, sizeof a[na].val, "%.*s", (int)(c - kq - 2), kq + 2);
            na++;
            start = c + 1;
            if (end) break;
            continue;
        }
        if (*c == '{') depth++;
        if (*c == '}') depth--;
    }
    if (r->root_port != KXPU_PCIE_NO_KEY) port_attr(&a[na++], domain, "pcieRootPort", r->root_port);
    if (r->pcie_switch != KXPU_PCIE_NO_KEY) port_attr(&a[na++], domain, "pcieSwitch", r->pcie_switch);
    qsort(a, (size_t)na, sizeof a[0], attr_cmp);
    putn(b, s, (size_t)(body - s));
    for (int k = 0; k < na; k++) put(b, "%s\"%s\":%s", k ? "," : "", a[k].key, a[k].val);
    put(b, "}");
    free(t.p);
}

static int record_why_pcie(const prec_t *r) {
    const int w = record_why(BASE(r));
    if (w) return w;
    const uint64_t rp = r->root_port, sw = r->pcie_switch;
    if ((rp != KXPU_PCIE_NO_KEY && rp >> 48) || (sw != KXPU_PCIE_NO_KEY && sw >> 48)) return N_RULES + 1;
    if (sw != KXPU_PCIE_NO_KEY && rp == KXPU_PCIE_NO_KEY) return N_RULES + 2;
    return 0;
}
#define N_RULES_PCIE (N_RULES + 2)

int32_t kxd_dra_slices_vgpu_pcie(const char *driver, const char *pool, const char *node, uint64_t generation,
                                 const char *domain, const prec_t *devs, size_t n, const kxpu_dra_taint *tab, size_t nt,
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
