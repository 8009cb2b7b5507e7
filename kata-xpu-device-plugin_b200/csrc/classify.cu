// classify.cu -- K5: createIommuDeviceMap + device-list build over a flat record table.
//
// Reference: pkg/device_plugin/device_plugin.go:126-180 (walk, filter, group, index) and
// :91-98 (per-device-id group lists).  The sequential walk is restated as data-parallel
// primitives whose results equal the walk's:
//   candidate(i)  = !dir && vendor=="10de" && driver=="vfio-pci" && links readable   (:137-161)
//                   (kxpu_classify_rules: (vendor, driver) equals the pair of some rule r; the device-id key
//                   below becomes (rule of the group's first member, device id))
//   gfirst[g]     = min{ i : candidate(i), group(i)=g, device file readable }        (:162-170:
//                   a group only comes into existence at a record whose device read works)
//   accept(i)     = candidate(i) && gfirst[group(i)] <= i                            (:171-175)
//   busIndex(i)   = #accepted before i                       -> exclusive scan
//   group ordinal = rank of gfirst[g] among group-first records -> exclusive scan
//   iommuMap CSR  = accepted records stably sorted by group ordinal -> LSD radix sort
//   deviceMap     = groups keyed by the device id of their first member, ids ordered by
//                   first appearance; CSR by a second stable sort.
// kxpu_classify_mdev: the candidate kernel reads 128-byte mdev records and writes each candidate's type key; a
// name-intern pass maps every key to the first candidate carrying it (hash table, keys compared byte for byte);
// the device-id key becomes (rule << 48 | that record's index).  Everything from k_accept_scan on is shared.
// kxpu_classify_vf_vgpu: k_candidates_vf(_viable) reads the caller's key row of a record that matched a vGPU rule, k_intern_vf
// interns those rows as k_intern does the mdev keys, k_groups<MODE_VF(_VIAB)> keys such a group like an mdev group.
// kxpu_classify_viable: k_candidates_viable also folds the first blocker of every group into the group table's spare
// word, k_groups<MODE_VIAB> copies it out per ordinal (both on kxpu_classify_rules' launches).
// kxpu_classify_topo / _mdev_topo: k_pairs<true> also ORs each accepted record's NUMA node into its group ordinal's mask
// (zeroed by k_reset with the totals); same launches as the non-topology call.
// Launches: reset | candidates | accept + both scans (single pass, decoupled look-back) | per-group device ids | device-id
// first-seen scan over the groups | sort pairs + all digit histograms | <= 4 radix passes, each ONE
// kernel for both sorts (per-tile ranking + per-digit look-back, "onesweep") | CSR boundaries.
#include <algorithm>
#include <utility>

#include "common.cuh"
#include "mdev.cuh"
#include "scan.cuh"

namespace kxclass {

constexpr uint32_t EMPTY32 = 0xFFFFFFFFu;
constexpr unsigned long long EMPTY64 = 0xFFFFFFFFFFFFFFFFull;

// iommu group -> first good record, ordinal; pad: first blocker of the group (kxpu_classify_viable only)
struct __align__(16) GSlot { uint32_t key, first, ord, pad; };
struct __align__(16) DSlot { unsigned long long key; uint32_t first, ord; };  // device id string -> first group-first record, ordinal
struct __align__(16) ISlot { unsigned long long tag; uint32_t first, pad; };   // type key: hash << 32 | some record with it; first such record

constexpr int C_THREADS = 256;
constexpr int C_ITEMS = 8;
constexpr int C_TILE = C_THREADS * C_ITEMS;  // records per CTA of the scan kernels

// totals[] (device): 0 accepted, 1 groups, 2 device ids, 3 unsupported-input flag
struct Work {
    const kxpu_devrec *recs;
    uint32_t n;
    GSlot *gtab;
    DSlot *dtab;
    uint32_t gcap, gshift, dcap, dshift;
    uint32_t *gslot;      // [n] slot of the record's group (EMPTY32: not a candidate)
    uint32_t *grp_rec;    // [n_groups] first record of group ordinal o
    uint32_t *grp_dslot;  // [n_groups] device-id slot of group ordinal o
    uint32_t *totals;
    unsigned long long *st_acc, *st_gf, *st_df;  // look-back status words
    uint32_t ep_acc, ep_gf, ep_df;
    // sort buffers: members (group ordinal, record) / groups (device ordinal, group id)
    uint32_t *ak, *av, *bk, *bv;
    uint32_t *ghist;  // [2 sorts][4 passes][256]
    // outputs (device)
    uint32_t *accept_index, *group_ids, *group_off, *dev_off;
    unsigned long long *dev_ids;
    // kxpu_classify_rules only (NULL otherwise): rule of record i, rule of device-map entry d
    uint8_t *rrule, *dev_rule;
    // kxpu_classify_mdev only: the records, per-record type keys (48 bytes: 40 key bytes, zero padded, length in
    // byte 47), intern slot of each record (EMPTY32: no key to intern) and the intern table
    const kxpu_mdevrec *mrecs;
    uint4 *keybuf;
    union {
        uint32_t *islot;
        uint32_t *group_blocker;  // kxpu_classify_viable only (never mdev): [n] first blocker per group ordinal
    };
    ISlot *itab;
    uint32_t icap, ishift;
    // kxpu_classify_topo / _mdev_topo only: [n] NUMA mask per group ordinal (zeroed by k_reset)
    unsigned long long *group_numa;
};
enum { MODE_NV = 0, MODE_RULES = 1, MODE_MDEV = 2, MODE_VIAB = 3, MODE_VF = 4, MODE_VF_VIAB = 5, MODE_NAMED = 6, MODE_NAMED_VIAB = 7 };

// The rule list of kxpu_classify_rules as k_candidates compares it: per rule the vendor id bytes with the id
// length in bits 56-63 (the same packing as read_id's result), and the driver as two 64-bit words with
// masks that cover its bytes and the NUL behind it (strncmp over the 16-byte field).
struct RuleTable {
    unsigned long long vend[KXPU_MAX_RULES], d0[KXPU_MAX_RULES], d1[KXPU_MAX_RULES], m0[KXPU_MAX_RULES], m1[KXPU_MAX_RULES];
    uint32_t n;
    uint32_t vgpu_mask;  // kxpu_classify_vf_vgpu: bit r = rule r serves vGPU types (0 elsewhere; the struct's padding word)
};
// kxpu_classify_vf_vgpu keeps its key rows in keybuf and each record's intern slot (EMPTY32: no key to intern) in the
// member sort's key buffer `ak`, which nothing reads before k_pairs writes it: Work keeps its size and layout, so the
// existing kernels read their parameters where they always did.
__device__ __forceinline__ uint32_t *vf_islot(const Work &W) { return W.ak; }
// the device-id key carries the rule in bits 48-63: an id is at most 6 bytes after data[2:]
constexpr unsigned long long DEVID_MASK = 0x0000FFFFFFFFFFFFull;

// The name table of kxpu_classify_named as the candidate pass compares it: per exact entry the id packed like read_id's
// result with its length in bits 56-63, its rule and its slot; per rule the slot of its "*" entry (NO_STAR: none).
// A named candidate's key row is (slot, rule, 0..., NAME_ROW in byte 47): byte 47 of a type-key row is its length
// (at most 40), so the two kinds never intern together.  Its deviceMap key sets NAMED_KEY, which no id key and no
// type key carries, so a slotted entry never merges with an entry keyed by a device id of the same rule.
struct NameTable {
    unsigned long long id[KXPU_MAX_NAMES];
    uint8_t rule[KXPU_MAX_NAMES], slot[KXPU_MAX_NAMES];
    uint8_t star[KXPU_MAX_RULES];
    uint32_t n;
};
constexpr uint8_t NO_STAR = 0xFFu;
constexpr uint8_t NAME_ROW = 0xFFu;
constexpr unsigned long long NAMED_KEY = 1ull << 63;

// readIDFromFileFunc (device_plugin.go:183-191): data[2:] with '\n' trimmed at both ends.
// Returns false when the file is shorter than 2 bytes (the reference would panic) or longer
// than the 8 bytes the record carries.
__device__ __forceinline__ bool read_id(const uint8_t *txt, uint32_t flen, unsigned long long &id, uint32_t &len) {
    id = 0; len = 0;
    if (flen < 2u || flen > 8u) return false;
    int a = 2, b = (int)flen;
    while (a < b && txt[a] == (uint8_t)'\n') a++;
    while (b > a && txt[b - 1] == (uint8_t)'\n') b--;
    unsigned long long v = 0;
    for (int k = a; k < b; k++) v |= (unsigned long long)txt[k] << (8 * (k - a));
    id = v; len = (uint32_t)(b - a);
    return true;
}

__device__ __forceinline__ uint32_t hash32(uint32_t k) { return k * 0x9E3779B1u; }
__device__ __forceinline__ uint32_t hash64(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33;
    return (uint32_t)k * 0x9E3779B1u;
}

__device__ __forceinline__ uint32_t ginsert(const Work &W, uint32_t key) {
    uint32_t slot = hash32(key) >> W.gshift;
    for (;;) {
        uint32_t k = __ldcg(&W.gtab[slot].key);
        if (k == key) return slot;
        if (k == EMPTY32) {
            uint32_t old = atomicCAS(&W.gtab[slot].key, EMPTY32, key);
            if (old == EMPTY32 || old == key) return slot;
        }
        slot = (slot + 1) & (W.gcap - 1);
    }
}
// the device-id table starts small (real hosts see a few ids; a 4-hex id space holds 65 536): a probe
// run of 512 means it is too small -- flag it (totals[3] bit 1), the host runs again with dcap = gcap
__device__ __forceinline__ uint32_t dinsert(const Work &W, unsigned long long key) {
    uint32_t slot = hash64(key) >> W.dshift;
    for (uint32_t step = 0; step < 512u; step++) {
        unsigned long long k = __ldcg(&W.dtab[slot].key);
        if (k == key) return slot;
        if (k == EMPTY64) {
            unsigned long long old = atomicCAS(&W.dtab[slot].key, EMPTY64, key);
            if (old == EMPTY64 || old == key) return slot;
        }
        slot = (slot + 1) & (W.dcap - 1);
    }
    atomicOr(&W.totals[3], 2u);
    return 0u;
}

// pass 1: candidates, group table, gfirst.  RULES: the (vendor, driver) pair is matched against the rule list of
// kxpu_classify_rules and the matching rule is stored per record for k_groups; otherwise the NVIDIA constants.
// VIAB (kxpu_classify_viable): a blocker -- KXPU_REC_BLOCKS, not a directory, not a candidate -- inserts its group too
// and lowers the slot's pad word (all ones from k_reset) to its index.  Its slot never gets an ordinal: the scans
// read gslot[i], which stays EMPTY32 for a non-candidate.  Each record inserts at most one group, so gcap >= 2n holds.
// VF (kxpu_classify_vf_vgpu): a record of a rule in R.vgpu_mask is a candidate only with a non-empty key row, which also
// replaces its device read; its device file is not looked at.  Such a candidate's key goes to k_intern_vf (vf_islot).
// NAMED (kxpu_classify_named, always with VF): a candidate of any other rule whose device read works looks its id up in
// the name table, exact entry first, then its rule's "*"; with a slot it writes a name row and goes to k_intern_vf too.
template <bool RULES, bool VIAB = false, bool VF = false, bool NAMED = false>
__device__ __forceinline__ void candidates(const Work &W, const RuleTable &R, const NameTable *NT = nullptr) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W.n) return;
    // one 64-byte record per thread: three 16-byte vector loads (the bdf is not needed to classify)
    const uint4 *rp = reinterpret_cast<const uint4 *>(W.recs + i);
    uint4 q1 = rp[1], q2 = rp[2], q3 = rp[3];
    const uint8_t *vtxt = reinterpret_cast<const uint8_t *>(&q1);      // vendor_txt[8], device_txt[8]
    const uint8_t *dtxt = vtxt + 8;
    const unsigned long long drv0 = ((unsigned long long)q2.y << 32) | q2.x;  // driver[0..8)
    const uint32_t drv8 = q2.z & 0xffu;
    const uint32_t group = q3.x;
    const uint32_t vlen = q3.y & 0xffu, dlen = (q3.y >> 8) & 0xffu, fl = (q3.y >> 16) & 0xffu;
    unsigned long long vid, did;
    uint32_t vl, dl;
    bool vok = read_id(vtxt, vlen, vid, vl);
    bool match;
    uint32_t rule = 0;
    if (RULES) {
        const unsigned long long vkey = vid | ((unsigned long long)vl << 56);
        const unsigned long long drv1 = ((unsigned long long)q2.w << 32) | q2.z;  // driver[8..16)
        match = false;
#pragma unroll
        for (uint32_t r = 0; r < KXPU_MAX_RULES; r++) {  // constant indices: the table stays in the parameter bank
            if (r < R.n && vkey == R.vend[r] && (drv0 & R.m0[r]) == R.d0[r] && (drv1 & R.m1[r]) == R.d1[r]) {
                match = true;
                rule = r;
            }
        }
    } else {
        match = vl == 4u && vid == 0x65643031ull /* "10de" */ && drv0 == 0x6963702d6f696676ull /* "vfio-pci" */ && drv8 == 0u;
    }
    bool cand = !(fl & KXPU_REC_IS_DIR) && !(fl & KXPU_REC_VENDOR_ERR) && vok && match && !(fl & KXPU_REC_DRIVER_ERR) &&
                !(fl & KXPU_REC_IOMMU_ERR);
    bool dok = !(fl & KXPU_REC_DEVICE_ERR) && read_id(dtxt, dlen, did, dl);
    if (!(fl & (KXPU_REC_IS_DIR | KXPU_REC_VENDOR_ERR)) && vlen > 8u) atomicOr(&W.totals[3], 1u);
    bool vr = false;  // VF: the record matched a vGPU rule
    if (VF) {
        vr = match && ((R.vgpu_mask >> rule) & 1u);
        if (vr) {
            dok = reinterpret_cast<const uint8_t *>(W.keybuf + 3 * (size_t)i)[47] != 0u;  // the key length
            cand = cand && dok;
            if (cand && group == EMPTY32) atomicOr(&W.totals[3], 1u);
        }
        vf_islot(W)[i] = vr && cand ? 0u : EMPTY32;
    }
    if (NAMED && !vr && cand && dok) {
        const unsigned long long dkey = did | ((unsigned long long)dl << 56);
        uint32_t s = NO_STAR;
#pragma unroll
        for (uint32_t r = 0; r < KXPU_MAX_RULES; r++)
            if (r == rule) s = NT->star[r];
#pragma unroll
        for (uint32_t e = 0; e < KXPU_MAX_NAMES; e++)  // constant indices: the table stays in the parameter bank
            if (e < NT->n && NT->rule[e] == rule && NT->id[e] == dkey) s = NT->slot[e];
        if (s != NO_STAR) {
            uint4 *kb = W.keybuf + 3 * (size_t)i;
            kb[0] = make_uint4(s | (rule << 8), 0u, 0u, 0u);
            kb[1] = make_uint4(0u, 0u, 0u, 0u);
            kb[2] = make_uint4(0u, 0u, 0u, (uint32_t)NAME_ROW << 24);
            vf_islot(W)[i] = 0u;
        }
    }
    if (!vr && cand && (group == EMPTY32 || (dok && did == EMPTY64) || (!(fl & KXPU_REC_DEVICE_ERR) && dlen > 8u)))
        atomicOr(&W.totals[3], 1u);  // outside the supported domain
    uint32_t slot = EMPTY32;
    if (cand) {
        slot = ginsert(W, group);
        if (dok && i < __ldcg(&W.gtab[slot].first)) atomicMin(&W.gtab[slot].first, i);
    }
    if (VIAB && !cand && (fl & (KXPU_REC_BLOCKS | KXPU_REC_IS_DIR)) == KXPU_REC_BLOCKS) {
        if (group == EMPTY32) {
            atomicOr(&W.totals[3], 1u);  // outside the supported domain, as for a candidate
        } else {
            const uint32_t bs = ginsert(W, group);
            if (i < __ldcg(&W.gtab[bs].pad)) atomicMin(&W.gtab[bs].pad, i);
        }
    }
    W.gslot[i] = slot;
    if (RULES) W.rrule[i] = (uint8_t)rule;
}
__global__ void __launch_bounds__(256) k_candidates(const Work W) { candidates<false>(W, RuleTable{}); }
__global__ void __launch_bounds__(256) k_candidates_rules(const Work W, const __grid_constant__ RuleTable R) {
    candidates<true>(W, R);
}
__global__ void __launch_bounds__(256) k_candidates_viable(const Work W, const __grid_constant__ RuleTable R) {
    candidates<true, true>(W, R);
}
__global__ void __launch_bounds__(256) k_candidates_vf(const Work W, const __grid_constant__ RuleTable R) {
    candidates<true, false, true>(W, R);
}
__global__ void __launch_bounds__(256) k_candidates_vf_viable(const Work W, const __grid_constant__ RuleTable R) {
    candidates<true, true, true>(W, R);
}
__global__ void __launch_bounds__(256) k_candidates_named(const Work W, const __grid_constant__ RuleTable R,
                                                          const __grid_constant__ NameTable N) {
    candidates<true, false, true, true>(W, R, &N);
}
__global__ void __launch_bounds__(256) k_candidates_named_viable(const Work W, const __grid_constant__ RuleTable R,
                                                                 const __grid_constant__ NameTable N) {
    candidates<true, true, true, true>(W, R, &N);
}

// pass 1 of kxpu_classify_mdev: candidates, group table, gfirst (a group starts at a candidate with a non-empty type
// key), and the type key of every such candidate into keybuf for k_intern.  One 128-byte record per thread, eight
// vector loads; the key is assembled in this thread's 48-byte row of shared memory.
__global__ void __launch_bounds__(256) k_candidates_mdev(const Work W, const __grid_constant__ RuleTable R) {
    __shared__ __align__(16) uint8_t skey[256][48];
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W.n) return;
    const uint4 *rp = reinterpret_cast<const uint4 *>(W.mrecs + i);
    uint4 q[8];
#pragma unroll
    for (int k = 0; k < 8; k++) q[k] = rp[k];
    const uint32_t uw[9] = {q[0].x, q[0].y, q[0].z, q[0].w, q[1].x, q[1].y, q[1].z, q[1].w, q[2].x};  // uuid[36]
    const uint2 vtxt = make_uint2(q[3].y, q[3].z);                                 // parent_vendor_txt @52
    const unsigned long long drv0 = ((unsigned long long)q[4].x << 32) | q[3].w;   // driver @60
    const unsigned long long drv1 = ((unsigned long long)q[4].z << 32) | q[4].y;
    const uint32_t nw[10] = {q[4].w, q[5].x, q[5].y, q[5].z, q[5].w, q[6].x, q[6].y, q[6].z, q[6].w, q[7].x};  // type_name @76
    const uint32_t group = q[7].y;
    const uint32_t vlen = q[7].z & 0xffu, nlen = (q[7].z >> 8) & 0xffu, fl = (q[7].z >> 16) & 0xffu;
    unsigned long long vid;
    uint32_t vl;
    const bool vok = read_id(reinterpret_cast<const uint8_t *>(&vtxt), vlen, vid, vl);
    const unsigned long long vkey = vid | ((unsigned long long)vl << 56);
    bool match = false;
    uint32_t rule = 0;
#pragma unroll
    for (uint32_t r = 0; r < KXPU_MAX_RULES; r++) {
        if (r < R.n && vkey == R.vend[r] && (drv0 & R.m0[r]) == R.d0[r] && (drv1 & R.m1[r]) == R.d1[r]) {
            match = true;
            rule = r;
        }
    }
    const bool cand = !(fl & (KXPU_REC_IS_DIR | KXPU_REC_VENDOR_ERR | KXPU_REC_DRIVER_ERR | KXPU_REC_IOMMU_ERR)) && vok && match &&
                      group != EMPTY32 && kxmdev::uuid_ok(uw);
    uint8_t *row = skey[threadIdx.x];
    uint4 *row4 = reinterpret_cast<uint4 *>(row);
    row4[0] = row4[1] = row4[2] = make_uint4(0u, 0u, 0u, 0u);
    const bool nread = !(fl & KXPU_REC_NAME_ERR) && nlen <= kxmdev::NAME_MAX_BYTES;
    const uint32_t klen = nread ? kxmdev::type_key(nw, nlen, [&](uint32_t p, uint8_t c) { row[p] = c; }) : 0u;
    const bool nok = klen != 0u;
    uint32_t slot = EMPTY32;
    if (cand) {
        slot = ginsert(W, group);
        if (nok && i < __ldcg(&W.gtab[slot].first)) atomicMin(&W.gtab[slot].first, i);
    }
    W.gslot[i] = slot;
    W.rrule[i] = (uint8_t)rule;
    W.islot[i] = cand && nok ? 0u : EMPTY32;
    if (cand && nok) {
        row[47] = (uint8_t)klen;
        uint4 *kb = W.keybuf + 3 * (size_t)i;
        kb[0] = row4[0]; kb[1] = row4[1]; kb[2] = row4[2];
    }
}

__device__ __forceinline__ bool key_eq(const uint4 &a, const uint4 &b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }

// pass 1b of kxpu_classify_mdev: intern the type keys.  A slot holds (hash << 32 | some record with the key), claimed by
// CAS; a hash hit compares the 48 key bytes with that record's.  The slot's `first` is the lowest record with the key
// (atomicMin).  Like the device-id table the intern table starts small: a probe run of 512 flags it (totals[3] bit 2)
// and the host runs again with both tables at full size.  VF: the slots of kxpu_classify_vf_vgpu (vf_islot).
template <bool VF>
__device__ __forceinline__ void intern(const Work &W) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= W.n || (VF ? vf_islot(W)[i] : W.islot[i]) == EMPTY32) return;
    const uint4 *kp = W.keybuf + 3 * (size_t)i;
    const uint4 k0 = kp[0], k1 = kp[1], k2 = kp[2];
    unsigned long long hv = 0x9E3779B97F4A7C15ull;
    const uint32_t kw[12] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w, k2.x, k2.y, k2.z, k2.w};
#pragma unroll
    for (int k = 0; k < 12; k++) { hv = (hv ^ kw[k]) * 0xff51afd7ed558ccdull; hv ^= hv >> 29; }
    const uint32_t h = (uint32_t)(hv >> 32);
    const unsigned long long tag = ((unsigned long long)h << 32) | i;
    uint32_t slot = h >> W.ishift;
    for (uint32_t step = 0; step < 512u; step++) {
        unsigned long long t = __ldcg(&W.itab[slot].tag);
        if (t == EMPTY64) {
            t = atomicCAS(&W.itab[slot].tag, EMPTY64, tag);
            if (t == EMPTY64) t = tag;
        }
        if ((uint32_t)(t >> 32) == h) {
            const uint4 *op = W.keybuf + 3 * (size_t)(uint32_t)t;
            if (key_eq(op[0], k0) && key_eq(op[1], k1) && key_eq(op[2], k2)) {
                if (i < __ldcg(&W.itab[slot].first)) atomicMin(&W.itab[slot].first, i);
                (VF ? vf_islot(W)[i] : W.islot[i]) = slot;
                return;
            }
        }
        slot = (slot + 1) & (W.icap - 1);
    }
    atomicOr(&W.totals[3], 4u);
}
__global__ void __launch_bounds__(256) k_intern(const Work W) { intern<false>(W); }
__global__ void __launch_bounds__(256) k_intern_vf(const Work W) { intern<true>(W); }

// pass 2: accept / group-first flags of a 2048-record tile, both exclusive scans in the same kernel
// (two look-backs, warp 0 and warp 1), busIndex out, group ordinals out, device-id table insert.
__global__ void __launch_bounds__(C_THREADS) k_accept_scan(const Work W) {
    __shared__ uint32_t wsum[C_THREADS / 32];
    __shared__ uint32_t s_tot;
    __shared__ unsigned long long s_excl[2];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    const uint32_t base = blockIdx.x * C_TILE + tid * C_ITEMS;  // blocked: 16 consecutive records per thread
    uint32_t slot[C_ITEMS];
    if (base + C_ITEMS <= W.n) {
#pragma unroll
        for (int k = 0; k < C_ITEMS; k += 4) {
            const uint4 q = *reinterpret_cast<const uint4 *>(W.gslot + base + k);
            slot[k] = q.x; slot[k + 1] = q.y; slot[k + 2] = q.z; slot[k + 3] = q.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < C_ITEMS; k++) slot[k] = base + k < W.n ? W.gslot[base + k] : EMPTY32;
    }
    uint32_t accm = 0, gfm = 0;  // bit k: record base + k accepted / first of its group
    uint32_t first[C_ITEMS];
#pragma unroll
    for (int k = 0; k < C_ITEMS; k++) first[k] = W.gtab[slot[k] != EMPTY32 ? slot[k] : 0u].first;  // all loads in flight at once
#pragma unroll
    for (int k = 0; k < C_ITEMS; k++) {
        if (slot[k] != EMPTY32) {
            if (first[k] <= base + k) accm |= 1u << k;
            if (first[k] == base + k) gfm |= 1u << k;
        }
    }
    const uint32_t packed = (uint32_t)__popc(accm) | ((uint32_t)__popc(gfm) << 16);  // <= 2048 each per tile
    const uint32_t incl = kxscan::warp_incl(packed);
    if (lane == 31) wsum[w] = incl;
    __syncthreads();
    if (w == 0) {
        const uint32_t x = lane < C_THREADS / 32 ? wsum[lane] : 0u;
        const uint32_t xi = kxscan::warp_incl(x);
        if (lane < C_THREADS / 32) wsum[lane] = xi - x;
        if (lane == C_THREADS / 32 - 1) s_tot = xi;
    }
    __syncthreads();
    const uint32_t ex = wsum[w] + incl - packed;
    const uint32_t tot = s_tot;
    if (w < 2) {
        const unsigned long long agg = w == 0 ? (tot & 0xffffu) : (tot >> 16);
        const unsigned long long e = kxscan::lookback(w == 0 ? W.st_acc : W.st_gf, blockIdx.x, agg, w == 0 ? W.ep_acc : W.ep_gf);
        if (lane == 0) {
            s_excl[w] = e;
            if (blockIdx.x == gridDim.x - 1) W.totals[w] = (uint32_t)(e + agg);
        }
    }
    __syncthreads();
    uint32_t racc = (uint32_t)s_excl[0] + (ex & 0xffffu), rgf = (uint32_t)s_excl[1] + (ex >> 16);
    uint32_t outv[C_ITEMS];
#pragma unroll
    for (int k = 0; k < C_ITEMS; k++) {
        outv[k] = KXPU_REJECTED;
        if ((accm >> k) & 1u) outv[k] = racc++;
        if ((gfm >> k) & 1u) {
            const uint32_t ord = rgf++;
            W.gtab[slot[k]].ord = ord;
            W.grp_rec[ord] = base + k;  // the rest of the group's bookkeeping: k_groups, one thread per group
        }
    }
    if (base + C_ITEMS <= W.n) {
#pragma unroll
        for (int k = 0; k < C_ITEMS; k += 4)
            *reinterpret_cast<uint4 *>(W.accept_index + base + k) = make_uint4(outv[k], outv[k + 1], outv[k + 2], outv[k + 3]);
    } else {
#pragma unroll
        for (int k = 0; k < C_ITEMS; k++)
            if (base + k < W.n) W.accept_index[base + k] = outv[k];
    }
}

// pass 2b: one thread per group (ordinal order): the group id and the device id of its first member (the group is
// attributed to the device id of its FIRST member, device_plugin.go:162-170) -> device-id table, first-seen minimum.
// Kept out of k_accept_scan: there the chain record read -> table insert -> minimum ran serially per record in a
// divergent loop (6 % issue utilisation); here every group is an independent thread.
// MODE_RULES: the device-id key is (rule of the first member) << 48 | device id; MODE_MDEV: (rule of the first member)
// << 48 | first record with its type key.  MODE_VIAB: MODE_RULES plus the group's first blocker from its slot.
// MODE_VF / MODE_VF_VIAB: MODE_RULES / MODE_VIAB, except that a group whose first member matched a vGPU rule is keyed
// like MODE_MDEV's, by (rule, first record with its type key).  MODE_NAMED / MODE_NAMED_VIAB: MODE_VF / MODE_VF_VIAB,
// and a group whose first member has a slot is keyed NAMED_KEY | (rule, first record with that (rule, slot)).
template <int MODE>
__global__ void __launch_bounds__(256) k_groups(const Work W) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= W.totals[1]) return;
    const uint32_t i = W.grp_rec[o];
    if (MODE == MODE_MDEV) {
        W.group_ids[o] = reinterpret_cast<const uint32_t *>(W.mrecs + i)[29];  // iommu_group @116
        const unsigned long long key = ((unsigned long long)W.rrule[i] << 48) | W.itab[W.islot[i]].first;
        const uint32_t ds = dinsert(W, key);
        if (i < __ldcg(&W.dtab[ds].first)) atomicMin(&W.dtab[ds].first, i);
        W.grp_dslot[o] = ds;
        return;
    }
    const uint32_t *rw = reinterpret_cast<const uint32_t *>(W.recs + i);
    const uint2 dq = make_uint2(rw[6], rw[7]);  // device_txt
    const uint32_t dlen = (rw[13] >> 8) & 0xffu;
    W.group_ids[o] = rw[12];                    // iommu_group
    unsigned long long did;
    uint32_t dl;
    read_id(reinterpret_cast<const uint8_t *>(&dq), dlen, did, dl);
    if (MODE == MODE_RULES || MODE == MODE_VIAB || MODE == MODE_VF || MODE == MODE_VF_VIAB || MODE == MODE_NAMED ||
        MODE == MODE_NAMED_VIAB)
        did |= (unsigned long long)W.rrule[i] << 48;
    if ((MODE == MODE_VF || MODE == MODE_VF_VIAB) && vf_islot(W)[i] != EMPTY32)  // the first member matched a vGPU rule
        did = ((unsigned long long)W.rrule[i] << 48) | W.itab[vf_islot(W)[i]].first;
    if ((MODE == MODE_NAMED || MODE == MODE_NAMED_VIAB) && vf_islot(W)[i] != EMPTY32) {  // a vGPU rule or a slot
        const bool slotted = reinterpret_cast<const uint8_t *>(W.keybuf + 3 * (size_t)i)[47] == NAME_ROW;
        did = (slotted ? NAMED_KEY : 0ull) | ((unsigned long long)W.rrule[i] << 48) | W.itab[vf_islot(W)[i]].first;
    }
    if (MODE == MODE_VIAB || MODE == MODE_VF_VIAB || MODE == MODE_NAMED_VIAB) W.group_blocker[o] = W.gtab[W.gslot[i]].pad;
    const uint32_t ds = dinsert(W, did);
    // a few hot device ids own most groups: same-address atomics run at ~1 per ns, so only a group that can
    // still lower the minimum issues one
    if (i < __ldcg(&W.dtab[ds].first)) atomicMin(&W.dtab[ds].first, i);
    W.grp_dslot[o] = ds;
}

// pass 3: over the groups in ordinal order: is this the first group of its device id?  Scan -> device ordinals.
__global__ void __launch_bounds__(C_THREADS) k_devfirst_scan(const Work W) {
    __shared__ unsigned long long s_excl;
    const uint32_t ng = W.totals[1];
    const uint32_t base = blockIdx.x * C_TILE + threadIdx.x * C_ITEMS;
    uint32_t dfm = 0;
#pragma unroll
    for (int k = 0; k < C_ITEMS; k++) {
        const uint32_t o = base + k;
        if (o < ng && W.dtab[W.grp_dslot[o]].first == W.grp_rec[o]) dfm |= 1u << k;
    }
    uint32_t tot;
    const uint32_t ex = kxscan::block_excl((uint32_t)__popc(dfm), &tot);
    if (threadIdx.x < 32) {
        const unsigned long long e = kxscan::lookback(W.st_df, blockIdx.x, tot, W.ep_df);
        if (threadIdx.x == 0) {
            s_excl = e;
            if (blockIdx.x == gridDim.x - 1) W.totals[2] = (uint32_t)(e + tot);
        }
    }
    __syncthreads();
    uint32_t run = (uint32_t)s_excl + ex;
#pragma unroll
    for (int k = 0; k < C_ITEMS; k++) {
        if ((dfm >> k) & 1u) {
            DSlot &d = W.dtab[W.grp_dslot[base + k]];
            d.ord = run;
            W.dev_ids[run] = d.key & DEVID_MASK;
            if (W.dev_rule) W.dev_rule[run] = (uint8_t)(d.key >> 48);
            run++;
        }
    }
}

// pass 3b of kxpu_classify_named: one thread per group; the first group of each entry writes the entry's slot, from the
// name row of the record its key names, or KXPU_NO_SLOT.  A launch of its own keeps k_devfirst_scan as it is.
__global__ void __launch_bounds__(256) k_dev_slots(const Work W, uint32_t *dev_slot) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= W.totals[1]) return;
    const DSlot &d = W.dtab[W.grp_dslot[o]];
    if (d.first != W.grp_rec[o]) return;
    dev_slot[d.ord] = (d.key & NAMED_KEY) ? reinterpret_cast<const uint8_t *>(W.keybuf + 3 * (size_t)(uint32_t)d.key)[0]
                                           : KXPU_NO_SLOT;
}

// pass 4: sort inputs -- members (group ordinal, record) at busIndex, groups (device ordinal, group id)
// at group ordinal -- and the digit histograms of all radix passes of both sorts.
// TOPO (kxpu_classify_topo / _mdev_topo): this pass already holds every accepted record with its group ordinal, so it
// also ORs the record's NUMA node into group_numa[ordinal]: one more 4-byte load (the flags / numa_node word) and one
// 64-bit atomicOr per accepted record that carries a node.
template <bool TOPO>
__global__ void __launch_bounds__(256) k_pairs(const Work W, uint32_t passes) {
    __shared__ uint32_t h[2 * 4 * 256];
    for (uint32_t k = threadIdx.x; k < 2 * 4 * 256; k += 256) h[k] = 0u;
    __syncthreads();
    const uint32_t stride = gridDim.x * blockDim.x;
    const uint32_t ng = W.totals[1];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < W.n; i += stride) {
        const uint32_t b = W.accept_index[i];
        if (b != KXPU_REJECTED) {
            const uint32_t key = W.gtab[W.gslot[i]].ord;
            W.ak[b] = key;
            W.av[b] = i;
            if (TOPO) {
                // kxpu_devrec word 13 / kxpu_mdevrec word 30: [.., .., flags, numa_node]
                const uint32_t fw = W.mrecs ? reinterpret_cast<const uint32_t *>(W.mrecs + i)[30]
                                            : reinterpret_cast<const uint32_t *>(W.recs + i)[13];
                const uint32_t node = fw >> 24;
                if ((fw & (KXPU_REC_NUMA << 16)) && node < KXPU_MAX_NUMA_NODES) atomicOr(&W.group_numa[key], 1ull << node);
            }
            for (uint32_t p = 0; p < passes; p++) atomicAdd(&h[(0 * 4 + p) * 256 + ((key >> (8 * p)) & 255u)], 1u);
        }
        if (i < ng) {
            const uint32_t key = W.dtab[W.grp_dslot[i]].ord;
            W.bk[i] = key;
            W.bv[i] = W.group_ids[i];
            for (uint32_t p = 0; p < passes; p++) atomicAdd(&h[(1 * 4 + p) * 256 + ((key >> (8 * p)) & 255u)], 1u);
        }
    }
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < 2 * 4 * 256; k += 256) {
        const uint32_t v = h[k];
        if (v) atomicAdd(&W.ghist[k], v);
    }
}

// ---------------------------------------------------------------- stable LSD radix sort, one kernel per pass
// A CTA ranks a tile of 4096 pairs: every warp owns 256 consecutive items and counts digits in its
// own shared-memory counters (rank inside the warp by __match_any_sync), the warps' counts are
// scanned per digit, the tile's count of every digit is published and the digit's offset over the
// tiles in front comes from a look-back over those status words (one digit per thread), the
// pass-wide digit bases from the histogram k_pairs made.  Both sorts run in the same launch.
constexpr int OS_WARPS = 16;
constexpr int OS_THREADS = OS_WARPS * 32;
constexpr int OS_STEPS = 8;
constexpr int OS_TILE = OS_THREADS * OS_STEPS;  // 4096

struct SortJob {
    const uint32_t *kin, *vin;
    uint32_t *kout, *vout;
    const uint32_t *count;      // items (device)
    const uint32_t *ghist;      // [256] digit totals of this pass
    unsigned long long *state;  // [tiles][256]
};
struct SweepParams {
    SortJob job[2];
    uint32_t shift, epoch;
};

__global__ void __launch_bounds__(OS_THREADS) k_onesweep(const SweepParams P) {
    __shared__ uint32_t cnt[OS_WARPS][256];
    __shared__ uint32_t tbase[256];
    __shared__ uint32_t wsum[OS_THREADS / 32];
    const SortJob J = blockIdx.y ? P.job[1] : P.job[0];  // constant indices: the parameters stay in the constant bank
    const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
    const uint32_t n = *J.count;
    const uint32_t tile = blockIdx.x;
    const uint32_t wbase = tile * OS_TILE + w * (OS_TILE / OS_WARPS);
#pragma unroll
    for (int k = 0; k < 256 / 32; k++) cnt[w][lane + 32 * k] = 0u;
    __syncwarp();
    uint32_t key[OS_STEPS], val[OS_STEPS], rk[OS_STEPS];
    const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
    for (int s = 0; s < OS_STEPS; s++) {
        const uint32_t i = wbase + s * 32u + lane;
        const bool act = i < n;
        key[s] = act ? J.kin[i] : 0u;
        val[s] = act ? J.vin[i] : 0u;
        const uint32_t d = act ? ((key[s] >> P.shift) & 255u) : 256u;  // 256: inactive lanes match each other only
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t r = (uint32_t)__popc(peers & lt);
        uint32_t prev = 0;
        if (act) prev = cnt[w][d];
        __syncwarp();
        if (act && r == 0u) cnt[w][d] = prev + (uint32_t)__popc(peers);
        __syncwarp();
        rk[s] = prev + r;
    }
    __syncthreads();
    // per digit: exclusive scan over the warps, tile count
    uint32_t tot = 0;
    if (tid < 256) {
#pragma unroll
        for (int k = 0; k < OS_WARPS; k++) {
            const uint32_t x = cnt[k][tid];
            cnt[k][tid] = tot;
            tot += x;
        }
    }
    // pass-wide digit bases: exclusive scan of the 256 digit totals
    const uint32_t gh = tid < 256 ? J.ghist[tid] : 0u;
    const uint32_t gi = kxscan::warp_incl(gh);
    if (lane == 31) wsum[w] = gi;
    __syncthreads();
    if (w == 0) {
        const uint32_t x = lane < OS_THREADS / 32 ? wsum[lane] : 0u;
        const uint32_t xi = kxscan::warp_incl(x);
        if (lane < OS_THREADS / 32) wsum[lane] = xi - x;
    }
    __syncthreads();
    if (tid < 256) {
        const uint32_t gbase = wsum[w] + gi - gh;
        // look-back over the tiles in front, for this thread's digit
        const unsigned long long tag = (unsigned long long)(P.epoch & 0xffffffu) << kxscan::ST_EPOCH_SHIFT;
        unsigned long long *st = J.state + tid;
        *reinterpret_cast<volatile unsigned long long *>(st + (size_t)tile * 256) = tag | (tile == 0 ? kxscan::ST_PFX : kxscan::ST_AGG) | tot;
        uint32_t excl = 0;
        for (long long j = (long long)tile - 1; j >= 0;) {
            const unsigned long long v = kxscan::ld_state(st + (size_t)j * 256);
            if ((v >> kxscan::ST_EPOCH_SHIFT) != (tag >> kxscan::ST_EPOCH_SHIFT) || (v & kxscan::ST_FLAGS) == 0) continue;  // not published yet
            excl += (uint32_t)(v & kxscan::ST_VAL);
            if ((v & kxscan::ST_FLAGS) == kxscan::ST_PFX) break;
            j--;
        }
        if (tile != 0) *reinterpret_cast<volatile unsigned long long *>(st + (size_t)tile * 256) = tag | kxscan::ST_PFX | (unsigned long long)(excl + tot);
        tbase[tid] = gbase + excl;
    }
    __syncthreads();
#pragma unroll
    for (int s = 0; s < OS_STEPS; s++) {
        const uint32_t i = wbase + s * 32u + lane;
        if (i < n) {
            const uint32_t d = (key[s] >> P.shift) & 255u;
            const uint32_t pos = tbase[d] + cnt[w][d] + rk[s];
            J.kout[pos] = key[s];
            J.vout[pos] = val[s];
        }
    }
}

// off[key[j]] = j at every run start; off[n_ord] = count.  blockIdx.y: members / groups
struct BoundsParams {
    const uint32_t *keys[2], *count[2], *nord[2];
    uint32_t *off[2];
};
__global__ void __launch_bounds__(256) k_bounds(const BoundsParams B) {
    const uint32_t *keys = blockIdx.y ? B.keys[1] : B.keys[0];
    const uint32_t *nord = blockIdx.y ? B.nord[1] : B.nord[0];
    uint32_t *off = blockIdx.y ? B.off[1] : B.off[0];
    const uint32_t n = blockIdx.y ? *B.count[1] : *B.count[0];
    const uint32_t stride = gridDim.x * blockDim.x;
    const uint32_t j0 = blockIdx.x * blockDim.x + threadIdx.x;
    if (j0 == 0) off[*nord] = n;
    for (uint32_t j = j0; j < n; j += stride) {
        const uint32_t k = keys[j];
        if (j == 0 || k != keys[j - 1]) off[k] = j;
    }
}

// 0xff over the hash tables, 0 over totals + histograms: one launch
__global__ void __launch_bounds__(256) k_reset(uint4 *ff, size_t n_ff16, uint32_t *zero, uint32_t n_zero) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t k = i; k < n_ff16; k += stride) ff[k] = make_uint4(0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu);
    for (size_t k = i; k < n_zero; k += stride) zero[k] = 0u;
}

}  // namespace kxclass

using namespace kxclass;

static uint32_t bits_for(uint32_t n) {
    uint32_t b = 1;
    while (b < 32 && (1ull << b) < (unsigned long long)n + 1) b++;
    return b;
}

// R == nullptr: kxpu_classify (the NVIDIA constants); else the rule list of kxpu_classify_rules, or with mdev of
// kxpu_classify_mdev (recs then points at kxpu_mdevrec records)
// group_numa != nullptr: the _topo calls (NUMA mask per group); group_blocker != nullptr: kxpu_classify_viable
// vgpu_mask != 0: kxpu_classify_vf_vgpu (keys: its key rows)
static int32_t classify_once(kxpu_ctx *ctx, const void *recs, size_t n, kxpu_classify_out *out, const RuleTable *R,
                             bool mdev, uint8_t *dev_rule, uint64_t *group_numa, uint32_t *group_blocker, uint32_t vgpu_mask,
                             const kxpu_vgpukey *keys, const NameTable *NT, uint32_t *dev_slot, bool small_dtab, bool *retry);

static int32_t classify_run(kxpu_ctx *ctx, const void *recs, size_t n, kxpu_classify_out *out, const RuleTable *R, bool mdev,
                            uint8_t *dev_rule, uint64_t *group_numa = nullptr, uint32_t *group_blocker = nullptr,
                            uint32_t vgpu_mask = 0, const kxpu_vgpukey *keys = nullptr, const NameTable *NT = nullptr,
                            uint32_t *dev_slot = nullptr) {
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    bool retry = false;
    int32_t rc = classify_once(ctx, recs, n, out, R, mdev, dev_rule, group_numa, group_blocker, vgpu_mask, keys, NT, dev_slot, true,
                               &retry);
    // more distinct device ids (or type keys) than the small tables hold; the rerun resets every table, blockers included
    if (retry)
        rc = classify_once(ctx, recs, n, out, R, mdev, dev_rule, group_numa, group_blocker, vgpu_mask, keys, NT, dev_slot, false,
                           &retry);
    return rc;
}

extern "C" int32_t kxpu_classify(kxpu_ctx *ctx, const kxpu_devrec *recs, size_t n, kxpu_classify_out *out) {
    if (!ctx || !out || (n && !recs)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    return classify_run(ctx, recs, n, out, nullptr, false, nullptr);
}

// a NUL-padded field: length of the text before the first NUL, -1 when a non-NUL byte follows that NUL
static int field_len(const char *f, int cap) {
    int l = 0;
    while (l < cap && f[l]) l++;
    for (int k = l; k < cap; k++)
        if (f[k]) return -1;
    return l;
}

// the rule list of kxpu_classify_rules / kxpu_classify_mdev -> R; KXPU_E_INVALID with a message when it is invalid
static int32_t rule_table(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, RuleTable &R) {
    memset(&R, 0, sizeof R);
    R.n = (uint32_t)n_rules;
    for (size_t r = 0; r < n_rules; r++) {
        const kxpu_xpu_rule &u = rules[r];
        const int vl = field_len(u.vendor, (int)sizeof u.vendor), dl = field_len(u.driver, (int)sizeof u.driver);
        if (vl < 1 || vl > 6 || memchr(u.vendor, '\n', (size_t)vl)) {
            KX_SET_ERR(ctx, "classify_rules: rule %zu: vendor must be 1-6 bytes without '\\n', NUL padded", r);
            return KXPU_E_INVALID;
        }
        if (dl < 1 || dl > 15 || memchr(u.driver, '/', (size_t)dl)) {
            KX_SET_ERR(ctx, "classify_rules: rule %zu: driver must be 1-15 bytes without '/', NUL padded", r);
            return KXPU_E_INVALID;
        }
        for (size_t q = 0; q < r; q++) {
            if (memcmp(rules[q].vendor, u.vendor, sizeof u.vendor) == 0 && memcmp(rules[q].driver, u.driver, sizeof u.driver) == 0) {
                KX_SET_ERR(ctx, "classify_rules: rules %zu and %zu are the same (vendor, driver) pair", q, r);
                return KXPU_E_INVALID;
            }
        }
        unsigned long long v = 0, d[2] = {0, 0}, m[2] = {0, 0};
        memcpy(&v, u.vendor, (size_t)vl);
        R.vend[r] = v | ((unsigned long long)vl << 56);
        memcpy(d, u.driver, sizeof u.driver);
        for (int k = 0; k <= dl; k++) m[k >> 3] |= 0xffull << (8 * (k & 7));  // the driver's bytes and its NUL
        R.d0[r] = d[0]; R.d1[r] = d[1]; R.m0[r] = m[0]; R.m1[r] = m[1];
    }
    return KXPU_OK;
}

extern "C" int32_t kxpu_classify_rules(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                                       size_t n, kxpu_classify_out *out, uint8_t *dev_rule) {
    if (!ctx || !out || (n && !recs) || !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    return classify_run(ctx, recs, n, out, &R, false, dev_rule);
}

extern "C" int32_t kxpu_classify_mdev(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs,
                                      size_t n, kxpu_classify_out *out, uint8_t *dev_rule) {
    static_assert(sizeof(kxpu_mdevrec) == 128 && offsetof(kxpu_mdevrec, iommu_group) == 116, "kxpu_mdevrec layout");
    if (!ctx || !out || (n && !recs) || !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    return classify_run(ctx, recs, n, out, &R, true, dev_rule);
}

extern "C" int32_t kxpu_classify_topo(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                                      size_t n, kxpu_classify_out *out, uint8_t *dev_rule, uint64_t *group_numa) {
    if (!ctx || !out || (n && (!recs || !group_numa)) || !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    return classify_run(ctx, recs, n, out, &R, false, dev_rule, group_numa);
}

extern "C" int32_t kxpu_classify_mdev_topo(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_mdevrec *recs,
                                           size_t n, kxpu_classify_out *out, uint8_t *dev_rule, uint64_t *group_numa) {
    if (!ctx || !out || (n && (!recs || !group_numa)) || !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    return classify_run(ctx, recs, n, out, &R, true, dev_rule, group_numa);
}

extern "C" int32_t kxpu_classify_viable(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, const kxpu_devrec *recs,
                                        size_t n, kxpu_classify_out *out, uint8_t *dev_rule, uint64_t *group_numa,
                                        uint32_t *group_blocker) {
    if (!ctx || !out || (n && (!recs || !group_blocker)) || !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES)
        return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    return classify_run(ctx, recs, n, out, &R, false, dev_rule, group_numa, group_blocker);
}

extern "C" int32_t kxpu_classify_vf_vgpu(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, uint32_t vgpu_rules,
                                         const kxpu_devrec *recs, size_t n, const kxpu_vgpukey *keys, kxpu_classify_out *out,
                                         uint8_t *dev_rule, uint64_t *group_numa, uint32_t *group_blocker) {
    if (!ctx || !out || (n && !recs) || !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    if ((vgpu_rules >> n_rules) || (vgpu_rules && !keys)) return KXPU_E_INVALID;
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    return classify_run(ctx, recs, n, out, &R, false, dev_rule, group_numa, group_blocker, vgpu_rules, keys);
}

extern "C" int32_t kxpu_classify_named(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, uint32_t vgpu_rules,
                                       const kxpu_devrec *recs, size_t n, const kxpu_vgpukey *keys, const kxpu_name_entry *names,
                                       size_t n_names, kxpu_classify_out *out, uint8_t *dev_rule, uint32_t *dev_slot,
                                       uint64_t *group_numa, uint32_t *group_blocker) {
    static_assert(sizeof(kxpu_name_entry) == 16, "kxpu_name_entry layout");
    if (!ctx || !out || (n && !recs) || !rules || n_rules == 0 || n_rules > KXPU_MAX_RULES) return KXPU_E_INVALID;
    if ((vgpu_rules >> n_rules) || (vgpu_rules && !keys)) return KXPU_E_INVALID;
    if (n_names > KXPU_MAX_NAMES || (n_names && (!names || (n && !dev_slot)))) return KXPU_E_INVALID;
    if (n_names == 0)  // kxpu_classify_vf_vgpu's call, byte for byte
        return kxpu_classify_vf_vgpu(ctx, rules, n_rules, vgpu_rules, recs, n, keys, out, dev_rule, group_numa, group_blocker);
    NameTable NT;
    memset(&NT, 0, sizeof NT);
    memset(NT.star, NO_STAR, sizeof NT.star);
    for (size_t e = 0; e < n_names; e++) {
        const kxpu_name_entry &u = names[e];
        const int il = field_len(u.device, (int)sizeof u.device);
        const bool star = il == 1 && u.device[0] == '*';
        bool hex = il == 4;
        for (int k = 0; hex && k < 4; k++) hex = (u.device[k] >= '0' && u.device[k] <= '9') || (u.device[k] >= 'a' && u.device[k] <= 'f');
        if (u.rule >= n_rules || ((vgpu_rules >> u.rule) & 1u)) {
            KX_SET_ERR(ctx, "classify_named: name %zu: rule %u is not a passthrough rule of the list", e, u.rule);
            return KXPU_E_INVALID;
        }
        if (!star && !hex) {
            KX_SET_ERR(ctx, "classify_named: name %zu: device must be 4 lowercase hex digits or \"*\", NUL padded", e);
            return KXPU_E_INVALID;
        }
        if (u.slot >= n_names) {
            KX_SET_ERR(ctx, "classify_named: name %zu: slot %u is not below n_names (%zu)", e, u.slot, n_names);
            return KXPU_E_INVALID;
        }
        for (size_t q = 0; q < e; q++) {
            if (names[q].rule == u.rule && memcmp(names[q].device, u.device, sizeof u.device) == 0) {
                KX_SET_ERR(ctx, "classify_named: names %zu and %zu are the same (rule, device) pair", q, e);
                return KXPU_E_INVALID;
            }
        }
        if (star) {
            NT.star[u.rule] = (uint8_t)u.slot;
        } else {
            unsigned long long v = 0;
            memcpy(&v, u.device, 4);
            NT.id[NT.n] = v | (4ull << 56);
            NT.rule[NT.n] = (uint8_t)u.rule;
            NT.slot[NT.n] = (uint8_t)u.slot;
            NT.n++;
        }
    }
    if (n >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    return classify_run(ctx, recs, n, out, &R, false, dev_rule, group_numa, group_blocker, vgpu_rules, keys, &NT, dev_slot);
}

int32_t kx_rule_drivers(kxpu_ctx *ctx, const kxpu_xpu_rule *rules, size_t n_rules, unsigned long long drv[][4]) {
    RuleTable R;
    const int32_t rc = rule_table(ctx, rules, n_rules, R);
    if (rc != KXPU_OK) return rc;
    for (size_t r = 0; r < n_rules; r++) {
        drv[r][0] = R.d0[r]; drv[r][1] = R.d1[r]; drv[r][2] = R.m0[r]; drv[r][3] = R.m1[r];
    }
    return KXPU_OK;
}

static int32_t classify_once(kxpu_ctx *ctx, const void *recs, size_t n, kxpu_classify_out *out, const RuleTable *R,
                             bool mdev, uint8_t *dev_rule, uint64_t *group_numa, uint32_t *group_blocker, uint32_t vgpu_mask,
                             const kxpu_vgpukey *keys, const NameTable *NT, uint32_t *dev_slot, bool small_dtab, bool *retry) {
    *retry = false;
    out->n_accepted = out->n_groups = out->n_devids = 0;
    if (n == 0) {
        if (out->group_off) out->group_off[0] = 0;
        if (out->dev_off) out->dev_off[0] = 0;
        return KXPU_OK;
    }
    if (!out->accept_index || !out->group_ids || !out->group_off || !out->group_members || !out->dev_ids ||
        !out->dev_off || !out->dev_groups)
        return KXPU_E_INVALID;

    const uint32_t N = (uint32_t)n;
    uint32_t gcap = 1024;
    while (gcap < 2 * N) gcap <<= 1;
    uint32_t lg = 0;
    while ((1u << lg) < gcap) lg++;
    const uint32_t dcap = small_dtab ? std::min<uint32_t>(gcap, 1u << 17) : gcap;
    uint32_t dlg = 0;
    while ((1u << dlg) < dcap) dlg++;
    const uint32_t c_tiles = (N + C_TILE - 1) / C_TILE;
    const uint32_t s_tiles = (N + OS_TILE - 1) / OS_TILE;
    const uint32_t passes = (bits_for(N) + 7) / 8;

    // one arena; [ff-region | zero-region | rest]
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const bool interns = mdev || vgpu_mask || NT;
    const uint32_t icap = interns ? dcap : 0u;  // the intern table grows with the device-id table
    const size_t o_gtab = take((size_t)gcap * sizeof(GSlot)), o_dtab = take((size_t)dcap * sizeof(DSlot));
    const size_t o_itab = interns ? take((size_t)icap * sizeof(ISlot)) : 0;
    const size_t ff_bytes = off;
    const size_t o_totals = take(16), o_ghist = take(2 * 4 * 256 * 4);
    const size_t o_gnuma = group_numa ? take(n * 8) : 0;  // zeroed with the totals: one reset launch either way
    const size_t zero_words = (off - ff_bytes) / 4;
    const size_t rec_bytes = mdev ? sizeof(kxpu_mdevrec) : sizeof(kxpu_devrec);
    const size_t o_recs = take(n * rec_bytes);
    const size_t o_gslot = take(n * 4 + 64), o_grec = take(n * 4), o_gds = take(n * 4);
    const size_t o_ak = take(n * 4), o_av = take(n * 4), o_ak2 = take(n * 4), o_av2 = take(n * 4);
    const size_t o_bk = take(n * 4), o_bv = take(n * 4), o_bk2 = take(n * 4), o_bv2 = take(n * 4);
    const size_t o_acc_idx = take(n * 4 + 64), o_gids = take(n * 4), o_goff = take((n + 1) * 4);
    const size_t o_dids = take(n * 8), o_doff = take((n + 1) * 4);
    const size_t o_rrule = R ? take(n) : 0, o_drule = R ? take(n) : 0;
    const size_t o_keys = mdev ? take(n * 48) : 0, o_islot = mdev ? take(n * 4) : 0;
    const size_t o_gblk = group_blocker ? take(n * 4) : 0;  // every ordinal is written by k_groups: no reset
    const size_t o_vkeys = vgpu_mask || NT ? take(n * 48) : 0;  // NT: the name rows of the slotted candidates
    const size_t o_dslot = NT ? take(n * 4) : 0;
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    // look-back status words: three scans + the two sorts' per-digit words
    const size_t st_words = 3 * (size_t)c_tiles + 2 * (size_t)s_tiles * 256;
    unsigned long long *st = kx_scan_state(ctx, st_words);
    if (!st) return KXPU_E_NOMEM;

    Work W;
    memset(&W, 0, sizeof W);
    W.recs = (const kxpu_devrec *)(b + o_recs); W.n = N;
    W.gtab = (GSlot *)(b + o_gtab); W.dtab = (DSlot *)(b + o_dtab); W.gcap = gcap; W.gshift = 32 - lg; W.dcap = dcap; W.dshift = 32 - dlg;
    W.gslot = (uint32_t *)(b + o_gslot); W.grp_rec = (uint32_t *)(b + o_grec); W.grp_dslot = (uint32_t *)(b + o_gds);
    W.totals = (uint32_t *)(b + o_totals); W.ghist = (uint32_t *)(b + o_ghist);
    W.st_acc = st; W.st_gf = st + c_tiles; W.st_df = st + 2 * (size_t)c_tiles;
    W.ep_acc = kx_next_epoch(ctx); W.ep_gf = kx_next_epoch(ctx); W.ep_df = kx_next_epoch(ctx);
    W.ak = (uint32_t *)(b + o_ak); W.av = (uint32_t *)(b + o_av); W.bk = (uint32_t *)(b + o_bk); W.bv = (uint32_t *)(b + o_bv);
    W.accept_index = (uint32_t *)(b + o_acc_idx); W.group_ids = (uint32_t *)(b + o_gids);
    W.group_off = (uint32_t *)(b + o_goff); W.dev_ids = (unsigned long long *)(b + o_dids); W.dev_off = (uint32_t *)(b + o_doff);
    if (R) { W.rrule = b + o_rrule; W.dev_rule = b + o_drule; }
    if (group_numa) W.group_numa = (unsigned long long *)(b + o_gnuma);
    if (group_blocker) W.group_blocker = (uint32_t *)(b + o_gblk);
    if (mdev) {
        W.mrecs = (const kxpu_mdevrec *)(b + o_recs);
        W.keybuf = (uint4 *)(b + o_keys); W.islot = (uint32_t *)(b + o_islot);
        W.itab = (ISlot *)(b + o_itab); W.icap = icap; W.ishift = 32 - dlg;
    }
    if (vgpu_mask || NT) {
        W.keybuf = (uint4 *)(b + o_vkeys);
        W.itab = (ISlot *)(b + o_itab); W.icap = icap; W.ishift = 32 - dlg;
        if (vgpu_mask) cudaMemcpyAsync(W.keybuf, keys, n * 48, cudaMemcpyHostToDevice, ctx->stream);
    }

    cudaMemcpyAsync(b + o_recs, recs, n * rec_bytes, cudaMemcpyHostToDevice, ctx->stream);
    const unsigned g = (N + 255) / 256;
    uint32_t *ak = W.ak, *av = W.av, *ak2 = (uint32_t *)(b + o_ak2), *av2 = (uint32_t *)(b + o_av2);
    uint32_t *bk = W.bk, *bv = W.bv, *bk2 = (uint32_t *)(b + o_bk2), *bv2 = (uint32_t *)(b + o_bv2);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        k_reset<<<std::min<unsigned>((unsigned)((ff_bytes / 16 + 255) / 256), 8u * ctx->sm_count), 256, 0, ctx->stream>>>(
            (uint4 *)b, ff_bytes / 16, W.totals, (uint32_t)zero_words);
        if (mdev) {
            k_candidates_mdev<<<g, 256, 0, ctx->stream>>>(W, *R);
            k_intern<<<g, 256, 0, ctx->stream>>>(W);
            ctx->launches++;
        } else if (NT) {
            RuleTable RV = *R;
            RV.vgpu_mask = vgpu_mask;
            if (group_blocker) k_candidates_named_viable<<<g, 256, 0, ctx->stream>>>(W, RV, *NT);
            else k_candidates_named<<<g, 256, 0, ctx->stream>>>(W, RV, *NT);
            k_intern_vf<<<g, 256, 0, ctx->stream>>>(W);
            ctx->launches++;
        } else if (vgpu_mask) {
            RuleTable RV = *R;
            RV.vgpu_mask = vgpu_mask;
            if (group_blocker) k_candidates_vf_viable<<<g, 256, 0, ctx->stream>>>(W, RV);
            else k_candidates_vf<<<g, 256, 0, ctx->stream>>>(W, RV);
            k_intern_vf<<<g, 256, 0, ctx->stream>>>(W);
            ctx->launches++;
        } else if (group_blocker) k_candidates_viable<<<g, 256, 0, ctx->stream>>>(W, *R);
        else if (R) k_candidates_rules<<<g, 256, 0, ctx->stream>>>(W, *R);
        else k_candidates<<<g, 256, 0, ctx->stream>>>(W);
        k_accept_scan<<<c_tiles, C_THREADS, 0, ctx->stream>>>(W);
        if (mdev) k_groups<MODE_MDEV><<<g, 256, 0, ctx->stream>>>(W);
        else if (NT && group_blocker) k_groups<MODE_NAMED_VIAB><<<g, 256, 0, ctx->stream>>>(W);
        else if (NT) k_groups<MODE_NAMED><<<g, 256, 0, ctx->stream>>>(W);
        else if (vgpu_mask && group_blocker) k_groups<MODE_VF_VIAB><<<g, 256, 0, ctx->stream>>>(W);
        else if (vgpu_mask) k_groups<MODE_VF><<<g, 256, 0, ctx->stream>>>(W);
        else if (group_blocker) k_groups<MODE_VIAB><<<g, 256, 0, ctx->stream>>>(W);
        else if (R) k_groups<MODE_RULES><<<g, 256, 0, ctx->stream>>>(W);
        else k_groups<MODE_NV><<<g, 256, 0, ctx->stream>>>(W);
        k_devfirst_scan<<<c_tiles, C_THREADS, 0, ctx->stream>>>(W);
        if (NT) {
            k_dev_slots<<<g, 256, 0, ctx->stream>>>(W, (uint32_t *)(b + o_dslot));
            ctx->launches++;
        }
        if (group_numa) k_pairs<true><<<std::min<unsigned>(g, 4u * ctx->sm_count), 256, 0, ctx->stream>>>(W, passes);
        else k_pairs<false><<<std::min<unsigned>(g, 4u * ctx->sm_count), 256, 0, ctx->stream>>>(W, passes);
        ctx->launches += 6;
        for (uint32_t p = 0; p < passes; p++) {
            SweepParams S;
            S.shift = 8 * p;
            S.epoch = kx_next_epoch(ctx);
            S.job[0] = SortJob{ak, av, ak2, av2, W.totals + 0, W.ghist + (0 * 4 + p) * 256, st + 3 * (size_t)c_tiles};
            S.job[1] = SortJob{bk, bv, bk2, bv2, W.totals + 1, W.ghist + (1 * 4 + p) * 256, st + 3 * (size_t)c_tiles + (size_t)s_tiles * 256};
            k_onesweep<<<dim3(s_tiles, 2), OS_THREADS, 0, ctx->stream>>>(S);
            ctx->launches++;
            std::swap(ak, ak2); std::swap(av, av2); std::swap(bk, bk2); std::swap(bv, bv2);
        }
        BoundsParams B;
        B.keys[0] = ak; B.count[0] = W.totals + 0; B.nord[0] = W.totals + 1; B.off[0] = W.group_off;
        B.keys[1] = bk; B.count[1] = W.totals + 1; B.nord[1] = W.totals + 2; B.off[1] = W.dev_off;
        k_bounds<<<dim3(std::min<unsigned>(g, 2u * ctx->sm_count), 2), 256, 0, ctx->stream>>>(B);
        ctx->launches++;
    }
    // results: sorted values are the CSR payloads
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, W.totals, 16, cudaMemcpyDeviceToHost, ctx->stream);
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    int32_t rc = KXPU_OK;
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "classify failed: %s", cudaGetErrorString(e)); rc = KXPU_E_CUDA; }
    else if ((h[3] & 6u) && small_dtab) { *retry = true; return KXPU_E_CAPACITY; }
    else if (h[3] & 1u) { KX_SET_ERR(ctx, "classify: record outside the supported domain (group 0xffffffff or id file > 8 bytes)"); rc = KXPU_E_UNSUPPORTED; }
    else if (h[3] & 6u) { KX_SET_ERR(ctx, "classify: device-id or type-key table overflow"); rc = KXPU_E_CAPACITY; }
    if (rc == KXPU_OK) {
        const uint32_t na = h[0], ng = h[1], nd = h[2];
        out->n_accepted = na; out->n_groups = ng; out->n_devids = nd;
        cudaMemcpyAsync(out->accept_index, W.accept_index, n * 4, cudaMemcpyDeviceToHost, ctx->stream);
        cudaMemcpyAsync(out->group_ids, W.group_ids, (size_t)ng * 4, cudaMemcpyDeviceToHost, ctx->stream);
        cudaMemcpyAsync(out->group_off, W.group_off, ((size_t)ng + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream);
        cudaMemcpyAsync(out->group_members, av, (size_t)na * 4, cudaMemcpyDeviceToHost, ctx->stream);
        cudaMemcpyAsync(out->dev_ids, W.dev_ids, (size_t)nd * 8, cudaMemcpyDeviceToHost, ctx->stream);
        cudaMemcpyAsync(out->dev_off, W.dev_off, ((size_t)nd + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream);
        cudaMemcpyAsync(out->dev_groups, bv, (size_t)ng * 4, cudaMemcpyDeviceToHost, ctx->stream);
        if (dev_rule && nd) cudaMemcpyAsync(dev_rule, W.dev_rule, nd, cudaMemcpyDeviceToHost, ctx->stream);
        if (group_numa && ng) cudaMemcpyAsync(group_numa, W.group_numa, (size_t)ng * 8, cudaMemcpyDeviceToHost, ctx->stream);
        if (group_blocker && ng) cudaMemcpyAsync(group_blocker, W.group_blocker, (size_t)ng * 4, cudaMemcpyDeviceToHost, ctx->stream);
        if (NT && nd) cudaMemcpyAsync(dev_slot, b + o_dslot, (size_t)nd * 4, cudaMemcpyDeviceToHost, ctx->stream);
        e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) { KX_SET_ERR(ctx, "classify D2H failed: %s", cudaGetErrorString(e)); rc = KXPU_E_CUDA; }
        if (ng == 0) out->group_off[0] = 0;
        if (nd == 0) out->dev_off[0] = 0;
    }
    return rc;
}
