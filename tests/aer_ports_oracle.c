/*
 * aer_ports_oracle.c -- CPU checker of kxpu_aer_ports and kxpu_aer_ports_mdev (include/kxpu.h, additions to ABI v14),
 * the C statement next to the Python restatement (tests/pyref_aer_ports.py).
 * TEST INFRASTRUCTURE ONLY: tests/aer_ports_oracle.py compiles it into a temporary directory.  It builds on
 * pcie_mdev_oracle.c (included: its component parse, the mdev path grammar and its hash).  Each path is scanned left to
 * right; the ports are numbered in one sequential pass, record by record, nearest first, through a key -> number map.
 */
#include "pcie_mdev_oracle.c"

/* the chain of a PCI record (kxpu_pcie_tree's grammar): its length (0 = unknown), keys in chain[0 .. len) */
static int chain_pci(const kxpu_devrec *rec, const kxpu_pcipath *p, uint64_t *chain) {
    const int len = p->len;
    if (len == 0 || len > 120) return 0;
    int comps = 1;
    for (int c = 0; c < len; c++) comps += p->path[c] == '/';
    if (comps < 2 || comps > MAXD + 1) return 0;
    int start = 0, k = 0;
    for (int c = 0; c <= len; c++) {
        if (c < len && p->path[c] != '/') continue;
        uint64_t key = 0;
        const int kind = component(p->path + start, c - start, &key);
        if (kind == 0 || (k == 0 && kind != 2)) return 0;
        if (k == comps - 1) { /* the function itself */
            const size_t bl = strnlen(rec->bdf, sizeof rec->bdf);
            if ((size_t)(c - start) != bl || memcmp(p->path + start, rec->bdf, bl)) return 0;
        } else {
            chain[k] = key;
        }
        k++;
        start = c + 1;
    }
    return comps - 1;
}

/* 0; the outputs as kxpu_aer_ports states them (mdev != 0: recs are kxpu_mdevrec, the chain less its parent) */
static int32_t ports(const void *recs, int mdev, const kxpu_pcipath *paths, size_t n, uint32_t *port_off,
                     uint32_t *port_of, uint64_t *port_key, uint32_t *n_ports) {
    uint32_t np = 0, nk = 0;
    size_t cap = 16;
    while (cap < 2 * (size_t)(MAXD - 1) * n + 16) cap <<= 1;
    uint32_t *num = malloc(cap * sizeof *num);  /* key -> its number + 1, 0 = free; port_key holds the keys */
    memset(num, 0, cap * sizeof *num);
    port_off[0] = 0;
    for (size_t i = 0; i < n; i++) {
        uint64_t chain[MAXD];
        int L = mdev ? kxo_pcie_parse_mdev((const kxpu_mdevrec *)recs + i, &paths[i], chain)
                     : chain_pci((const kxpu_devrec *)recs + i, &paths[i], chain);
        if (mdev && L > 0) L--;
        for (int t = L - 1; t >= 0; t--) {
            if (chain[t] >> 63) continue;
            size_t s = mixh(chain[t]) & (cap - 1);
            while (num[s] && port_key[num[s] - 1] != chain[t]) s = (s + 1) & (cap - 1);
            if (!num[s]) {
                port_key[nk] = chain[t];
                num[s] = ++nk;
            }
            port_of[np++] = num[s] - 1;
        }
        port_off[i + 1] = np;
    }
    *n_ports = nk;
    free(num);
    return 0;
}

int32_t kxa_aer_ports(const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n, uint32_t *port_off, uint32_t *port_of,
                      uint64_t *port_key, uint32_t *n_ports) {
    return ports(recs, 0, paths, n, port_off, port_of, port_key, n_ports);
}

int32_t kxa_aer_ports_mdev(const kxpu_mdevrec *recs, const kxpu_pcipath *paths, size_t n, uint32_t *port_off,
                           uint32_t *port_of, uint64_t *port_key, uint32_t *n_ports) {
    return ports(recs, 1, paths, n, port_off, port_of, port_key, n_ports);
}
