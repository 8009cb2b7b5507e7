/*
 * kxpu_dra_taint_oracle.c -- CPU checker of kxpu_dra_slices_taint and kxpu_dra_slices_mdev_taint (include/kxpu.h,
 * ABI v11): the ResourceSlices of one DRA pool with at most one taint per device, written sequentially with snprintf
 * from the rules stated in the header.  timeAdded comes from gmtime_r, so this checker shares no date arithmetic with
 * the GPU kernel.
 *
 * TEST INFRASTRUCTURE ONLY, like kxpu_oracle.c.  It builds on the passthrough and vGPU DRA oracles' helpers (names,
 * record domains, the Buf writer); the library it becomes also exports kxo_dra_slices and kxo_dra_slices_mdev.  The
 * devices are written here again rather than taken from those oracles, so that taint_since == NULL giving their bytes
 * is a check and not an identity.  Arguments and status codes are the product calls' without the context; on
 * KXPU_E_UNSUPPORTED *why names the first rule the first record outside the domain breaks (the record rules of the
 * layout, then "taint_since" as one more).
 */
#include <time.h>

#include "kxpu_dra_mdev_oracle.c"

/* [A-Za-z0-9] at both ends, [-A-Za-z0-9_.] between, 1..max bytes */
static int k8s_name(const char *s, size_t len, size_t max) {
    if (len == 0 || len > max) return 0;
    for (size_t i = 0; i < len; i++) {
        char c = s[i];
        int alnum = (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9');
        if (!alnum && ((i == 0 || i == len - 1) || (c != '-' && c != '_' && c != '.'))) return 0;
    }
    return 1;
}

static int taint_args_ok(const char *key, const char *value, const char *effect) {
    if (!key || !value || !effect) return 0;
    size_t kl = strnlen(key, 128);
    if (kl == 0 || kl > 127) return 0;
    const char *slash = memchr(key, '/', kl);
    if (slash) {
        char prefix[128];
        size_t pl = (size_t)(slash - key);
        memcpy(prefix, key, pl);
        prefix[pl] = 0;
        if (!subdomain_ok(prefix, 253) || !k8s_name(slash + 1, kl - pl - 1, 63)) return 0;
    } else if (!k8s_name(key, kl, 63)) {
        return 0;
    }
    size_t vl = strnlen(value, 64);
    if (vl && !k8s_name(value, vl, 63)) return 0;
    return strcmp(effect, "NoSchedule") == 0 || strcmp(effect, "NoExecute") == 0;
}

/* the taint member of one device, from its last attribute's closer on: "},"taints":[{...}]}" */
static void put_taint(Buf *b, const char *key, const char *value, const char *effect, int64_t since) {
    struct tm tm;
    time_t t = (time_t)since;
    gmtime_r(&t, &tm);
    char ts[64];
    snprintf(ts, sizeof ts, "%04d-%02d-%02dT%02d:%02d:%02dZ", tm.tm_year + 1900, tm.tm_mon + 1, tm.tm_mday, tm.tm_hour,
             tm.tm_min, tm.tm_sec);
    puts_(b, ",\"taints\":[{\"key\":\""); puts_(b, key); puts_(b, "\"");
    if (value[0]) { puts_(b, ",\"value\":\""); puts_(b, value); puts_(b, "\""); }
    puts_(b, ",\"effect\":\""); puts_(b, effect); puts_(b, "\",\"timeAdded\":\""); puts_(b, ts); puts_(b, "\"}]");
}

/* {"name":"vfio<g>","attributes":{...}  without the device's closing '}' */
static void put_pci_device(Buf *b, const kxpu_dradev *d) {
    char tmp[128];
    snprintf(tmp, sizeof tmp, "{\"name\":\"vfio%u\",\"attributes\":{\"deviceID\":{\"string\":\"", d->iommu_group);
    puts_(b, tmp); put(b, d->device, field_len(d->device, 8));
    snprintf(tmp, sizeof tmp, "\"},\"iommuGroup\":{\"int\":%u}", d->iommu_group);
    puts_(b, tmp);
    if (d->numa_mask && !(d->numa_mask & (d->numa_mask - 1))) {
        snprintf(tmp, sizeof tmp, ",\"numaNode\":{\"int\":%d}", __builtin_ctzll(d->numa_mask));
        puts_(b, tmp);
    }
    put_attr(b, "pciAddress", d->bdf, field_len(d->bdf, 16));
    if (d->product_len) put_attr(b, "productName", (const char *)d->product, d->product_len);
    if (d->pcie_root[0]) put_attr(b, "resource.kubernetes.io/pcieRoot", d->pcie_root, field_len(d->pcie_root, 16));
    put_attr(b, "vendorID", d->vendor, field_len(d->vendor, 8));
    puts_(b, "}");
}

static void put_mdev_device(Buf *b, const kxpu_dramdev *d) {
    char tmp[128];
    snprintf(tmp, sizeof tmp, "{\"name\":\"vfio%u\",\"attributes\":{\"iommuGroup\":{\"int\":%u}", d->iommu_group,
             d->iommu_group);
    puts_(b, tmp);
    put_attr(b, "mdevType", d->mdev_type, field_len(d->mdev_type, 40));
    if (d->numa_mask && !(d->numa_mask & (d->numa_mask - 1))) {
        snprintf(tmp, sizeof tmp, ",\"numaNode\":{\"int\":%d}", __builtin_ctzll(d->numa_mask));
        puts_(b, tmp);
    }
    put_attr(b, "parentAddress", d->parent, field_len(d->parent, 16));
    if (d->device[0]) put_attr(b, "parentDeviceID", d->device, field_len(d->device, 8));
    put_attr(b, "parentVendorID", d->vendor, field_len(d->vendor, 8));
    if (d->product_len) put_attr(b, "productName", (const char *)d->product, d->product_len);
    if (d->pcie_root[0]) put_attr(b, "resource.kubernetes.io/pcieRoot", d->pcie_root, field_len(d->pcie_root, 16));
    put_attr(b, "uuid", d->uuid, 36);
    puts_(b, "}");
}

static int32_t taint_slices(int mdev, const char *driver, const char *pool, const char *node, uint64_t generation,
                            const void *devs, size_t n, const char *key, const char *value, const char *effect,
                            const int64_t *since, uint8_t *out, size_t cap, size_t *len, uint64_t *slice_off,
                            size_t *n_slices, int32_t *why) {
    if (!len || !n_slices || (n && !devs)) return KXPU_E_INVALID;
    if (!subdomain_ok(driver, 63) || !subdomain_ok(pool, 253) || !subdomain_ok(node, 253) || generation >= (1ull << 63))
        return KXPU_E_INVALID;
    if (since && !taint_args_ok(key, value, effect)) return KXPU_E_INVALID;
    if (n >= KXPU_DRA_MAX_DEVICES) return KXPU_E_UNSUPPORTED;
    const int n_rules = mdev ? 9 : 7;
    for (size_t i = 0; i < n; i++) {
        int w = mdev ? mdev_record_why((const kxpu_dramdev *)devs + i) : record_why((const kxpu_dradev *)devs + i);
        if (!w && since && since[i] > KXPU_DRA_TAINT_SINCE_MAX) w = n_rules + 1;
        if (w) {
            if (why) *why = w - 1;
            return KXPU_E_UNSUPPORTED;
        }
    }
    const size_t per = since ? KXPU_DRA_TAINT_SLICE_DEVICES : KXPU_DRA_SLICE_DEVICES;
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
            if (since && since[i] >= 0) put_taint(&b, key, value, effect, since[i]);
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

int32_t kxo_dra_slices_taint(const char *driver, const char *pool, const char *node, uint64_t generation,
                             const kxpu_dradev *devs, size_t n, const char *taint_key, const char *taint_value,
                             const char *taint_effect, const int64_t *taint_since, uint8_t *out, size_t cap, size_t *len,
                             uint64_t *slice_off, size_t *n_slices, int32_t *why) {
    return taint_slices(0, driver, pool, node, generation, devs, n, taint_key, taint_value, taint_effect, taint_since, out,
                        cap, len, slice_off, n_slices, why);
}

int32_t kxo_dra_slices_mdev_taint(const char *driver, const char *pool, const char *node, uint64_t generation,
                                  const kxpu_dramdev *devs, size_t n, const char *taint_key, const char *taint_value,
                                  const char *taint_effect, const int64_t *taint_since, uint8_t *out, size_t cap,
                                  size_t *len, uint64_t *slice_off, size_t *n_slices, int32_t *why) {
    return taint_slices(1, driver, pool, node, generation, devs, n, taint_key, taint_value, taint_effect, taint_since, out,
                        cap, len, slice_off, n_slices, why);
}
