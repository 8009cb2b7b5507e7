/*
 * kxpu_dra_mdev_oracle.c -- CPU checker of kxpu_dra_slices_mdev (include/kxpu.h, ABI v10): the ResourceSlices of one
 * DRA pool of vGPUs as JSON Lines, written sequentially with snprintf from the rules stated in the header.
 *
 * TEST INFRASTRUCTURE ONLY, like kxpu_oracle.c.  The slices around the devices are kxpu_dra_slices' (the name, pool and
 * argument rules, the Buf writer), so this file includes kxpu_dra_oracle.c and builds on its helpers; it is compiled
 * as part of kxpu_aer_oracle.c's translation unit.  kxo_dra_slices_mdev takes kxpu_dra_slices_mdev's arguments without
 * the context and returns the same status codes; on KXPU_E_UNSUPPORTED *why names the first rule (the order of the
 * header's domain list) that the first record outside the domain breaks.
 */
#include "kxpu_dra_oracle.c"

static int name_byte(char c) {
    return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '_' || c == '.' || c == '-';
}

/* 0 = in the domain, else 1 + the index of the first failing rule: product, mdev_type, uuid, parent, pcie_root, vendor,
 * device, group, product_len */
static int mdev_record_why(const kxpu_dramdev *d) {
    if (d->product_len <= 64)
        for (size_t k = 0; k < d->product_len; k++)
            if (!name_byte((char)d->product[k])) return 1;
    size_t tl = field_len(d->mdev_type, 40);
    if (tl == 0) return 2;
    for (size_t k = 0; k < tl; k++)
        if (!name_byte(d->mdev_type[k])) return 2;
    for (size_t k = 0; k < 36; k++) {
        char c = d->uuid[k];
        if (k == 8 || k == 13 || k == 18 || k == 23 ? c != '-' : !is_hex(c)) return 3;
    }
    size_t bl = field_len(d->parent, 16);
    if (bl == 0) return 4;
    for (size_t k = 0; k < bl; k++)
        if (!is_hex(d->parent[k]) && d->parent[k] != ':' && d->parent[k] != '.') return 4;
    size_t rl = field_len(d->pcie_root, 16);
    if (rl) {
        if (rl < 4 || memcmp(d->pcie_root, "pci", 3) != 0) return 5;
        for (size_t k = 3; k < rl; k++)
            if (!is_hex(d->pcie_root[k]) && d->pcie_root[k] != ':') return 5;
    }
    size_t vl = field_len(d->vendor, 8), dl = field_len(d->device, 8);
    if (vl == 0 || vl > 6) return 6;
    for (size_t k = 0; k < vl; k++)
        if (!is_hex(d->vendor[k])) return 6;
    if (dl > 6) return 7;
    for (size_t k = 0; k < dl; k++)
        if (!is_hex(d->device[k])) return 7;
    if (d->iommu_group == 0xFFFFFFFFu) return 8;
    if (d->product_len > 64) return 9;
    return 0;
}

static void put_attr(Buf *b, const char *key, const char *val, size_t l) {
    puts_(b, ",\""); puts_(b, key); puts_(b, "\":{\"string\":\""); put(b, val, l); puts_(b, "\"}");
}

int32_t kxo_dra_slices_mdev(const char *driver, const char *pool, const char *node, uint64_t generation,
                            const kxpu_dramdev *devs, size_t n, uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off,
                            size_t *n_slices, int32_t *why) {
    if (!len || !n_slices || (n && !devs)) return KXPU_E_INVALID;
    if (!subdomain_ok(driver, 63) || !subdomain_ok(pool, 253) || !subdomain_ok(node, 253) || generation >= (1ull << 63))
        return KXPU_E_INVALID;
    if (n >= KXPU_DRA_MAX_DEVICES) return KXPU_E_UNSUPPORTED;
    for (size_t i = 0; i < n; i++) {
        int w = mdev_record_why(&devs[i]);
        if (w) {
            if (why) *why = w - 1;
            return KXPU_E_UNSUPPORTED;
        }
    }
    size_t slices = n ? (n + KXPU_DRA_SLICE_DEVICES - 1) / KXPU_DRA_SLICE_DEVICES : 1;
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
        size_t end = (s + 1) * KXPU_DRA_SLICE_DEVICES < n ? (s + 1) * KXPU_DRA_SLICE_DEVICES : n;
        for (size_t i = s * KXPU_DRA_SLICE_DEVICES; i < end; i++) {
            const kxpu_dramdev *d = &devs[i];
            if (i > s * KXPU_DRA_SLICE_DEVICES) puts_(&b, ",");
            snprintf(tmp, sizeof tmp, "{\"name\":\"vfio%u\",\"attributes\":{\"iommuGroup\":{\"int\":%u}", d->iommu_group,
                     d->iommu_group);
            puts_(&b, tmp);
            put_attr(&b, "mdevType", d->mdev_type, field_len(d->mdev_type, 40));
            if (d->numa_mask && !(d->numa_mask & (d->numa_mask - 1))) {
                int k = 0;
                while (!((d->numa_mask >> k) & 1)) k++;
                snprintf(tmp, sizeof tmp, ",\"numaNode\":{\"int\":%d}", k);
                puts_(&b, tmp);
            }
            put_attr(&b, "parentAddress", d->parent, field_len(d->parent, 16));
            if (d->device[0]) put_attr(&b, "parentDeviceID", d->device, field_len(d->device, 8));
            put_attr(&b, "parentVendorID", d->vendor, field_len(d->vendor, 8));
            if (d->product_len) put_attr(&b, "productName", (const char *)d->product, d->product_len);
            if (d->pcie_root[0]) put_attr(&b, "resource.kubernetes.io/pcieRoot", d->pcie_root, field_len(d->pcie_root, 16));
            put_attr(&b, "uuid", d->uuid, 36);
            puts_(&b, "}}");
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
