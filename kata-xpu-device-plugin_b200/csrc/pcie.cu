// pcie.cu -- K10: the PCIe forest of a walk (kxpu_pcie_tree).  include/kxpu.h states the path grammar and the tree.
//
// Five kernels and one scan:
//   - k_parse: 16 lanes per 128-byte kxpu_pcipath (two records per warp).  Eight lanes load the record with one 16-byte
//     vector load each; lane j then finds and parses component j of the path (at most 9 components: 8 of chain, the
//     function itself), a ballot over the 16 lanes decides "known", and lane j stores key j of the record's chain.
//   - k_lcp: one thread per group: the longest common prefix of its members' chains (member indices checked).
//   - k_insert: one thread per group inserts each prefix of its chain into an open-addressing table of u64 slots
//     (group << 3 | depth).  A slot is claimed by CAS; a hit compares the two prefixes key by key through the groups'
//     chains and then takes the atomic min, so every slot ends up naming the FIRST group with that prefix.  A slot's
//     group only ever changes to another group with the same prefix, so the comparison stays valid throughout.
//   - k_count: a group's prefixes whose first group is itself are its new nodes: always a suffix of its chain.
//   - the single-pass scan (scan.cuh) of the new-node counts gives each group's first ordinal; the total is n_nodes.
//   - k_emit: ordinal of prefix (g, t) = base[f] + t - (len(f) - new(f)), f its first group; a group writes key,
//     parent and depth of its own new nodes and its group_node.
// kxpu_pcie_tree_sriov runs the same launches with k_parse<kxpu_devrec, true> (which also stores each record's own key)
// and k_lcp<true> (which reads a VF's chain through its PF); the <kxpu_devrec, false> / <false> instantiations are
// kxpu_pcie_tree's kernels.  kxpu_pcie_tree_mdev runs k_parse<kxpu_mdevrec, false>, whose leaf is the record's UUID
// below its parent function (lanes 8..11 stage the record's UUID and parent next to the path), and kxpu_pcie_tree's
// other kernels.  kxpu_pcie_ports runs kxpu_pcie_tree's parse, then k_ports: the LCP pass (group_lcp<false>, shared
// with k_lcp) writing each group's root port and switch instead of its prefix.  kxpu_pcie_ports_mdev runs
// k_parse<kxpu_mdevrec, false>, then k_ports_mdev: the same pass over each member's chain one key short (its parent
// chain).  kxpu_aer_ports[_mdev] run the same two parses, then one thread per record in each of: k_port_count (the
// function keys of its chain, for the mdev variant less the parent), the single-pass scan (port_off), k_port_insert
// (each port into an open-addressing table of u32 position codes, atomic min: a key's first position), k_port_first
// (each position's slot and whether it is its key's first, counted per record), the scan of those counts (each
// record's first ordinal; the total is n_ports), k_port_key (port_key, and the ordinal into the slot) and k_port_of.
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "scan.cuh"

namespace kxpcie {

constexpr uint32_t NO_NODE = KXPU_PCIE_NO_NODE;
constexpr int MAXD = KXPU_PCIE_MAX_DEPTH;
constexpr int PATH_LANES = 16;
constexpr int PARSE_THREADS = 256;
constexpr int PARSE_RECS = PARSE_THREADS / PATH_LANES;
constexpr unsigned long long HOST_BRIDGE = 1ull << 63;
constexpr unsigned long long EMPTY = ~0ull;

__device__ __forceinline__ int hexv(char c) {
    return (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : -1;
}

// component t[s, e): 0 = not a component, 1 = function, 2 = host bridge; *key its node key
__device__ int parse_comp(const char *t, int s, int e, unsigned long long *key) {
    bool hb = false;
    if (e - s >= 3 && t[s] == 'p' && t[s + 1] == 'c' && t[s + 2] == 'i') { hb = true; s += 3; }
    int c = s;
    unsigned long long dom = 0;
    while (c < e && c - s < 9 && t[c] != ':') {
        const int v = hexv(t[c]);
        if (v < 0) return 0;
        dom = dom << 4 | (unsigned)v;
        c++;
    }
    const int dl = c - s;
    if (!(dl == 4 || (dl >= 5 && dl <= 8 && t[s] != '0'))) return 0;
    if (c >= e || t[c] != ':' || e - c < 3) return 0;
    const int b0 = hexv(t[c + 1]), b1 = hexv(t[c + 2]);
    if (b0 < 0 || b1 < 0) return 0;
    const unsigned long long bus = (unsigned)(b0 << 4 | b1);
    c += 3;
    if (hb) {
        if (c != e) return 0;
        *key = HOST_BRIDGE | dom << 16 | bus << 8;
        return 2;
    }
    if (e - c != 5 || t[c] != ':' || t[c + 3] != '.') return 0;
    const int d0 = hexv(t[c + 1]), d1 = hexv(t[c + 2]), f = t[c + 4] - '0';
    if (d0 < 0 || d1 < 0 || f < 0 || f > 7 || (d0 << 4 | d1) > 0x1f) return 0;
    *key = dom << 16 | bus << 8 | (unsigned long long)(d0 << 4 | d1) << 3 | (unsigned)f;
    return 1;
}

// component t[s, e) equals the name b[0 .. 16) up to its first NUL
__device__ __forceinline__ bool same_name(const char *t, int s, int e, const char *b) {
    int bl = 0;
    while (bl < 16 && b[bl]) bl++;
    bool same = e - s == bl;
    for (int k = 0; same && k < bl; k++) same = t[s + k] == b[k];
    return same;
}

// component t[s, e) is a canonical lowercase UUID (8-4-4-4-12) equal to uuid[0 .. 36)
__device__ __forceinline__ bool uuid_leaf(const char *t, int s, int e, const char *uuid) {
    bool same = e - s == 36;
    for (int k = 0; same && k < 36; k++) {
        const char c = t[s + k];
        same = c == uuid[k] && ((k == 8 || k == 13 || k == 18 || k == 23) ? c == '-' : hexv(c) >= 0);
    }
    return same;
}

// chain[i * MAXD + t] = key of component t of record i, clen[i] = chain length (0: unknown path).  SR
// (kxpu_pcie_tree_sriov): self[i] = the key of the record's own component when its path is known.  Rec = kxpu_mdevrec
// (kxpu_pcie_tree_mdev): the last component is the record's UUID and the one before it its parent function, which
// ends the chain.
template <typename Rec, bool SR>
__global__ void __launch_bounds__(PARSE_THREADS) k_parse(const Rec *__restrict__ recs, const kxpu_pcipath *__restrict__ paths,
                                                         uint32_t n, unsigned long long *__restrict__ chain, uint8_t *__restrict__ clen,
                                                         unsigned long long *__restrict__ self) {
    constexpr bool MD = std::is_same<Rec, kxpu_mdevrec>::value;
    static_assert(!(MD && SR), "the SR-IOV forest reads kxpu_devrec records");
    __shared__ __align__(16) char txt[PARSE_RECS][128];
    const uint32_t lane = threadIdx.x & (PATH_LANES - 1), slot = threadIdx.x / PATH_LANES;
    const uint32_t i = blockIdx.x * PARSE_RECS + slot;
    const bool have = i < n;
    if (have && lane < 8) reinterpret_cast<uint4 *>(txt[slot])[lane] = reinterpret_cast<const uint4 *>(paths + i)[lane];
    const char *own = nullptr;  // MD: the record's first 64 bytes (uuid at 0, parent at 36), staged by lanes 8..11
    if constexpr (MD) {
        __shared__ __align__(16) char head[PARSE_RECS][64];
        if (have && lane >= 8 && lane < 12)
            reinterpret_cast<uint4 *>(head[slot])[lane - 8] = reinterpret_cast<const uint4 *>(recs + i)[lane - 8];
        own = head[slot];
    }
    __syncwarp();
    const char *t = txt[slot];
    const int len = have ? (uint8_t)t[120] : 0;
    bool ok = len > 0 && len <= 120;
    // component `lane`: [s, e); n_comp = slashes + 1
    int s = 0, e = len, slashes = 0;
    if (ok) {
        for (int c = 0; c < len; c++) {
            if (t[c] != '/') continue;
            if (slashes == (int)lane - 1) s = c + 1;
            if (slashes == (int)lane) e = c;
            slashes++;
        }
    }
    const int ncomp = slashes + 1;
    ok = ok && ncomp >= 2 && ncomp <= MAXD + 1;
    bool mine = true;
    unsigned long long key = 0;
    if (ok && (int)lane < ncomp) {
        if constexpr (MD) {
            if ((int)lane == ncomp - 1) {  // the mdev itself: its UUID
                mine = uuid_leaf(t, s, e, own + offsetof(kxpu_mdevrec, uuid));
            } else {
                const int kind = parse_comp(t, s, e, &key);
                if (lane == 0) mine = kind == 2;
                else mine = kind != 0;
                // its parent: a function equal to the record's parent (a host bridge there is unknown, also at lane 0)
                if ((int)lane == ncomp - 2) mine = mine && kind == 1 && same_name(t, s, e, own + offsetof(kxpu_mdevrec, parent));
            }
        } else {
            const int kind = parse_comp(t, s, e, &key);
            if (lane == 0) mine = kind == 2;
            else mine = kind != 0;
            if ((int)lane == ncomp - 1 && mine) mine = same_name(t, s, e, recs[i].bdf);  // the function itself
        }
    }
    const uint32_t half = (threadIdx.x & 31u) & ~(uint32_t)(PATH_LANES - 1);
    const uint32_t bad = (__ballot_sync(0xffffffffu, !mine) >> half) & 0xffffu;
    ok = ok && bad == 0;
    if (!have) return;
    if (ok && (int)lane < ncomp - 1) chain[(size_t)i * MAXD + lane] = key;
    if constexpr (SR) {
        if (ok && (int)lane == ncomp - 1) self[i] = key;
    }
    if (lane == 0) clen[i] = ok ? (uint8_t)(ncomp - 1) : 0;
}

struct Tree {
    const uint32_t *goff, *gmem;
    uint32_t n, G;
    const unsigned long long *chain;
    const uint8_t *clen;
    unsigned long long *gchain;  // [G * MAXD]
    uint8_t *glen;               // [G]
    unsigned long long *slots;   // [mask + 1]
    uint32_t mask;
    uint32_t *first;             // [G * MAXD] first group of prefix (g, t)
    uint32_t *cnt, *base;        // [G] new nodes of g, their first ordinal
    uint32_t *group_node, *parent;
    unsigned long long *key;
    uint8_t *depth;
    uint32_t *err;               // [0] = 1: a member index >= n
    // kxpu_pcie_tree_sriov only: the PF of every record (each < n or NO_PF) and every record's own key
    const uint32_t *pf_of;
    const unsigned long long *self;
};

// the longest common prefix of group g's member chains into k[0 .. return value); *bad: a member index >= n.  SR: a
// member whose PF has a known chain shorter than MAXD reads the PF's chain followed by the PF's own key.  PARENT
// (kxpu_pcie_ports_mdev): a member reads its known chain less its last key, the parent function
template <bool SR, bool PARENT = false>
__device__ __forceinline__ int group_lcp(const Tree &T, uint32_t g, unsigned long long (&k)[MAXD], bool &bad) {
    static_assert(!(SR && PARENT), "the parent chain is read from mdev chains");
    int L = -1;
    for (uint32_t m = T.goff[g]; m < T.goff[g + 1]; m++) {
        const uint32_t i = T.gmem[m];
        if (i >= T.n) { bad = true; continue; }
        int l = T.clen[i];
        if constexpr (PARENT) l = max(l - 1, 0);  // a known mdev chain has 2..MAXD keys
        const unsigned long long *c = T.chain + (size_t)i * MAXD;
        unsigned long long tail = 0;  // SR, through the PF (via): the key at position l - 1
        bool via = false;
        if constexpr (SR) {
            const uint32_t p = T.pf_of[i];
            const int pl = p == KXPU_NO_PF ? 0 : T.clen[p];
            if (pl > 0 && pl < MAXD) {
                c = T.chain + (size_t)p * MAXD;
                l = pl + 1;
                tail = T.self[p];
                via = true;
            }
        }
        if (!l) continue;
        int nl = L < 0 ? l : min(L, l);
#pragma unroll
        for (int t = 0; t < MAXD; t++) {
            if (t >= nl) continue;
            const unsigned long long x = SR && via && t == l - 1 ? tail : c[t];
            if (L < 0) k[t] = x;
            else if (x != k[t]) nl = min(nl, t);
        }
        L = nl;
    }
    return max(L, 0);
}

template <bool SR>
__global__ void __launch_bounds__(256) k_lcp(const Tree T) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= T.G) return;
    unsigned long long k[MAXD];
    bool bad = false;
    const int L = group_lcp<SR>(T, g, k, bad);
    if (bad) atomicOr(T.err, 1u);
#pragma unroll
    for (int t = 0; t < MAXD; t++)
        if (t < L) T.gchain[(size_t)g * MAXD + t] = k[t];
    T.glen[g] = (uint8_t)L;
}

// the LCP pass of kxpu_pcie_tree (plain chains; PARENT: the mdevs' parent chains), then the rule of include/kxpu.h on
// the prefix: the functions after its last host bridge are f0, f1, ...; the root port is f0, the switch f_j for the
// greatest odd j
template <bool PARENT>
__device__ __forceinline__ void group_ports(const Tree &T, unsigned long long *__restrict__ root_port,
                                            unsigned long long *__restrict__ pcie_switch) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= T.G) return;
    unsigned long long k[MAXD];
    bool bad = false;
    const int L = group_lcp<false, PARENT>(T, g, k, bad);
    if (bad) atomicOr(T.err, 1u);
    // one pass root to leaf: a host bridge starts the function list again, f0 is the root port, each odd f_j the switch
    unsigned long long rp = KXPU_PCIE_NO_KEY, sw = KXPU_PCIE_NO_KEY;
    uint32_t j = 0;
#pragma unroll
    for (int t = 0; t < MAXD; t++) {
        if (t >= L) continue;
        if (k[t] & HOST_BRIDGE) {
            rp = sw = KXPU_PCIE_NO_KEY;
            j = 0;
            continue;
        }
        if (j == 0) rp = k[t];
        else if (j & 1u) sw = k[t];
        j++;
    }
    root_port[g] = rp;
    pcie_switch[g] = sw;
}

// kxpu_pcie_ports
__global__ void __launch_bounds__(256) k_ports(const Tree T, unsigned long long *__restrict__ root_port,
                                               unsigned long long *__restrict__ pcie_switch) {
    group_ports<false>(T, root_port, pcie_switch);
}

// kxpu_pcie_ports_mdev
__global__ void __launch_bounds__(256) k_ports_mdev(const Tree T, unsigned long long *__restrict__ root_port,
                                                    unsigned long long *__restrict__ pcie_switch) {
    group_ports<true>(T, root_port, pcie_switch);
}

__device__ __forceinline__ unsigned long long mix(unsigned long long h, unsigned long long x) {
    h = (h ^ x) * 0x9E3779B97F4A7C15ull;
    return h ^ (h >> 29);
}

// slot of prefix (g, t) (the prefix has been inserted when insert = false).  The table has at least two slots per
// prefix, so a probe sequence always ends; the bound only guarantees that it does (err[1] set, ~0u returned).
__device__ __forceinline__ uint32_t find_slot(const Tree &T, uint32_t g, int t, unsigned long long h, bool insert) {
    const unsigned long long *mine = T.gchain + (size_t)g * MAXD;
    const unsigned long long me = (unsigned long long)g << 3 | (unsigned)t;
    uint32_t s = (uint32_t)h & T.mask;
    for (uint32_t probes = 0; probes <= T.mask; probes++, s = (s + 1) & T.mask) {
        unsigned long long v = *reinterpret_cast<volatile unsigned long long *>(T.slots + s);
        if (v == EMPTY) {
            if (!insert) break;
            v = atomicCAS(T.slots + s, EMPTY, me);
            if (v == EMPTY) return s;
        }
        if ((int)(v & 7u) != t) continue;
        const unsigned long long *other = T.gchain + (size_t)(v >> 3) * MAXD;
        bool same = true;
        for (int u = t; u >= 0 && same; u--) same = other[u] == mine[u];
        if (!same) continue;
        if (insert) atomicMin(T.slots + s, me);
        return s;
    }
    atomicOr(T.err + 1, 1u);
    return ~0u;
}

__global__ void __launch_bounds__(256) k_insert(const Tree T) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= T.G) return;
    unsigned long long h = 0x243F6A8885A308D3ull;
    for (int t = 0; t < T.glen[g]; t++) {
        h = mix(h, T.gchain[(size_t)g * MAXD + t]);
        find_slot(T, g, t, h, true);
    }
}

__global__ void __launch_bounds__(256) k_count(const Tree T) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= T.G) return;
    unsigned long long h = 0x243F6A8885A308D3ull;
    uint32_t fresh = 0;
    for (int t = 0; t < T.glen[g]; t++) {
        h = mix(h, T.gchain[(size_t)g * MAXD + t]);
        const uint32_t s = find_slot(T, g, t, h, false);
        const uint32_t f = s == ~0u ? g : (uint32_t)(T.slots[s] >> 3);
        T.first[(size_t)g * MAXD + t] = f;
        fresh += f == g;
    }
    T.cnt[g] = fresh;
}

__global__ void __launch_bounds__(256) k_emit(const Tree T) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= T.G) return;
    const int L = T.glen[g];
    uint32_t prev = NO_NODE;
    for (int t = 0; t < L; t++) {
        const uint32_t f = T.first[(size_t)g * MAXD + t];
        const uint32_t v = T.base[f] + (uint32_t)t - ((uint32_t)T.glen[f] - T.cnt[f]);
        if (f == g) {
            T.key[v] = T.gchain[(size_t)g * MAXD + t];
            T.parent[v] = prev;
            T.depth[v] = (uint8_t)t;
        }
        prev = v;
    }
    T.group_node[g] = prev;
}

// kxpu_aer_ports[_mdev].  A record's ports are the function keys of its chain (MD: the chain less its last key, the
// parent function), nearest first; position (i, t) of chain key t sorts as i << 3 | (MAXD - 1 - t).  One thread per
// record in every pass.
constexpr uint32_t EMPTY32 = ~0u;
constexpr int PORTS_MAX = MAXD - 1;  // a known chain starts with a host bridge

struct Ports {
    uint32_t n;
    const unsigned long long *chain;
    const uint8_t *clen;
    uint32_t *cnt, *off;     // [n] ports of record i, its first position
    uint32_t *fcnt, *fbase;  // [n] positions of record i that are their key's first, their first ordinal
    uint32_t *slots;         // [mask + 1]: the least position code of a key; after k_port_key, that key's ordinal
    uint32_t mask;
    uint32_t *pslot;         // [PORTS_MAX * n] slot of position p
    uint8_t *pfirst;         // [PORTS_MAX * n] position p is its key's first
    uint32_t *port_of;
    unsigned long long *port_key;
    uint32_t *err;           // [0] = 1: table overflow
};

template <bool MD>
__device__ __forceinline__ int port_chain_len(const Ports &P, uint32_t i) {
    const int l = P.clen[i];
    return MD ? max(l - 1, 0) : l;
}

template <bool MD>
__global__ void __launch_bounds__(256) k_port_count(const Ports P) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const unsigned long long *c = P.chain + (size_t)i * MAXD;
    const int L = port_chain_len<MD>(P, i);
    uint32_t k = 0;
    for (int t = 0; t < L; t++) k += !(c[t] & HOST_BRIDGE);
    P.cnt[i] = k;
}

// slot of a port key (insert: of position code me, the atomic min of the codes; else the key has been inserted).  A slot
// holds a code whose key is read back from the chains, written by the parse, so the comparison stays valid while the
// slot's code falls to another position of the same key.  At least two slots per position: the bound only guarantees
// that a probe sequence ends (err[0] set, ~0u returned).
__device__ __forceinline__ uint32_t port_slot(const Ports &P, unsigned long long key, uint32_t me, bool insert) {
    uint32_t s = (uint32_t)mix(0x243F6A8885A308D3ull, key) & P.mask;
    for (unsigned long long probes = 0; probes <= P.mask; probes++, s = (s + 1) & P.mask) {
        uint32_t v = *reinterpret_cast<volatile uint32_t *>(P.slots + s);
        if (v == EMPTY32) {
            if (!insert) break;
            v = atomicCAS(P.slots + s, EMPTY32, me);
            if (v == EMPTY32) return s;
        }
        if (P.chain[(size_t)(v >> 3) * MAXD + (MAXD - 1 - (v & 7u))] != key) continue;
        if (insert && me < v) atomicMin(P.slots + s, me);  // a shared port: most records see a smaller code already
        return s;
    }
    atomicOr(P.err, 1u);
    return ~0u;
}

template <bool MD>
__global__ void __launch_bounds__(256) k_port_insert(const Ports P) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const unsigned long long *c = P.chain + (size_t)i * MAXD;
    for (int t = port_chain_len<MD>(P, i) - 1; t >= 0; t--)
        if (!(c[t] & HOST_BRIDGE)) port_slot(P, c[t], i << 3 | (uint32_t)(MAXD - 1 - t), true);
}

template <bool MD>
__global__ void __launch_bounds__(256) k_port_first(const Ports P) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const unsigned long long *c = P.chain + (size_t)i * MAXD;
    uint32_t p = P.off[i], f = 0;
    for (int t = port_chain_len<MD>(P, i) - 1; t >= 0; t--) {
        if (c[t] & HOST_BRIDGE) continue;
        const uint32_t me = i << 3 | (uint32_t)(MAXD - 1 - t);
        const uint32_t s = port_slot(P, c[t], me, false);
        const bool first = s != ~0u && P.slots[s] == me;
        P.pslot[p] = s;
        P.pfirst[p] = first;
        f += first;
        p++;
    }
    P.fcnt[i] = f;
}

// a first position names its key: port_key[ordinal], and the ordinal replaces the code in its slot
template <bool MD>
__global__ void __launch_bounds__(256) k_port_key(const Ports P) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    const unsigned long long *c = P.chain + (size_t)i * MAXD;
    uint32_t p = P.off[i], o = P.fbase[i];
    for (int t = port_chain_len<MD>(P, i) - 1; t >= 0; t--) {
        if (c[t] & HOST_BRIDGE) continue;
        if (P.pfirst[p]) {
            P.port_key[o] = c[t];
            P.slots[P.pslot[p]] = o++;
        }
        p++;
    }
}

__global__ void __launch_bounds__(256) k_port_of(const Ports P) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P.n) return;
    for (uint32_t p = P.off[i], e = p + P.cnt[i]; p < e; p++) {
        const uint32_t s = P.pslot[p];  // ~0u only after a table overflow, which the call reports
        P.port_of[p] = s == ~0u ? ~0u : P.slots[s];
    }
}

}  // namespace kxpcie

using namespace kxpcie;

void kx_pcie_parse(cudaStream_t st, const kxpu_devrec *recs, const kxpu_pcipath *paths, uint32_t n, unsigned long long *chain,
                   uint8_t *clen) {
    k_parse<kxpu_devrec, false><<<(n + PARSE_RECS - 1) / PARSE_RECS, PARSE_THREADS, 0, st>>>(recs, paths, n, chain, clen, nullptr);
}

// Rec = kxpu_devrec: pf_of == nullptr: kxpu_pcie_tree; else kxpu_pcie_tree_sriov (pf_of checked by the caller).
// Rec = kxpu_mdevrec: kxpu_pcie_tree_mdev (pf_of == nullptr).
template <typename Rec>
static int32_t pcie_tree(kxpu_ctx *ctx, const Rec *recs, const kxpu_pcipath *paths, size_t n, const uint32_t *group_off,
                         const uint32_t *group_members, size_t n_groups, uint32_t *group_node, uint64_t *key, uint32_t *parent,
                         uint8_t *depth, uint32_t *n_nodes, const uint32_t *pf_of) {
    static_assert(sizeof(kxpu_pcipath) == 128 && offsetof(kxpu_pcipath, len) == 120, "kxpu_pcipath layout");
    if (!ctx || !n_nodes || (n && (!recs || !paths)) || !group_off) return KXPU_E_INVALID;
    if (n >= (1ull << 28) || n_groups >= (1ull << 28)) return KXPU_E_UNSUPPORTED;
    *n_nodes = 0;
    for (size_t g = 0; g < n_groups; g++)
        if (group_off[g + 1] < group_off[g]) { KX_SET_ERR(ctx, "pcie_tree: group %zu: offsets decrease", g); return KXPU_E_INVALID; }
    const size_t nm = group_off[n_groups];
    if ((nm && !group_members) || (n_groups && (!group_node || !key || !parent || !depth))) return KXPU_E_INVALID;
    if (n_groups == 0) return KXPU_OK;
    if (nm >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    const size_t G = n_groups, GD = G * MAXD;
    uint32_t slots = 1;
    while (slots < 2 * GD) slots <<= 1;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_recs = take(n * sizeof(Rec)), o_paths = take(n * sizeof(kxpu_pcipath));
    const size_t o_goff = take((G + 1) * 4), o_gmem = take(nm * 4), o_chain = take(n * MAXD * 8), o_clen = take(n);
    const size_t o_gchain = take(GD * 8), o_glen = take(G), o_slots = take((size_t)slots * 8), o_first = take(GD * 4);
    const size_t o_cnt = take(G * 4), o_base = take(G * 4), o_gnode = take(G * 4), o_parent = take(GD * 4);
    const size_t o_key = take(GD * 8), o_depth = take(GD), o_err = take(8 + 8);
    const size_t o_pf = pf_of ? take(n * 4) : 0, o_self = pf_of ? take(n * 8) : 0;
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_recs, recs, n * sizeof(Rec)); up(o_paths, paths, n * sizeof(kxpu_pcipath));
    up(o_goff, group_off, (G + 1) * 4); up(o_gmem, group_members, nm * 4);
    if (pf_of) up(o_pf, pf_of, n * 4);
    cudaMemsetAsync(b + o_slots, 0xFF, (size_t)slots * 8, st);
    cudaMemsetAsync(b + o_err, 0, 16, st);
    Tree T;
    T.goff = (const uint32_t *)(b + o_goff); T.gmem = (const uint32_t *)(b + o_gmem);
    T.n = (uint32_t)n; T.G = (uint32_t)G;
    T.chain = (const unsigned long long *)(b + o_chain); T.clen = (const uint8_t *)(b + o_clen);
    T.gchain = (unsigned long long *)(b + o_gchain); T.glen = b + o_glen;
    T.slots = (unsigned long long *)(b + o_slots); T.mask = slots - 1;
    T.first = (uint32_t *)(b + o_first); T.cnt = (uint32_t *)(b + o_cnt); T.base = (uint32_t *)(b + o_base);
    T.group_node = (uint32_t *)(b + o_gnode); T.parent = (uint32_t *)(b + o_parent);
    T.key = (unsigned long long *)(b + o_key); T.depth = b + o_depth; T.err = (uint32_t *)(b + o_err);
    T.pf_of = pf_of ? (const uint32_t *)(b + o_pf) : nullptr;
    T.self = pf_of ? (const unsigned long long *)(b + o_self) : nullptr;
    unsigned long long *d_total = (unsigned long long *)(b + o_err + 8);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        if (n) {
            auto *parse = k_parse<Rec, false>;
            if constexpr (std::is_same<Rec, kxpu_devrec>::value) if (pf_of) parse = k_parse<Rec, true>;
            parse<<<(unsigned)((n + PARSE_RECS - 1) / PARSE_RECS), PARSE_THREADS, 0, st>>>(
                (const Rec *)(b + o_recs), (const kxpu_pcipath *)(b + o_paths), (uint32_t)n,
                (unsigned long long *)(b + o_chain), b + o_clen, (unsigned long long *)(b + o_self));
            ctx->launches++;
        }
        const unsigned gb = (unsigned)((G + 255) / 256);
        (pf_of ? k_lcp<true> : k_lcp<false>)<<<gb, 256, 0, st>>>(T);
        k_insert<<<gb, 256, 0, st>>>(T);
        k_count<<<gb, 256, 0, st>>>(T);
        ctx->launches += 3;
        const int32_t rc = kxscan::exclusive_scan(ctx, T.cnt, G, T.base, d_total);
        if (rc != KXPU_OK) return rc;
        k_emit<<<gb, 256, 0, st>>>(T);
        ctx->launches++;
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, T.err, 16, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "pcie_tree failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) { KX_SET_ERR(ctx, "pcie_tree: a group member index is >= n"); return KXPU_E_INVALID; }
    if (h[1]) { KX_SET_ERR(ctx, "pcie_tree: prefix table overflow"); return KXPU_E_CAPACITY; }
    const uint32_t nn = h[2];
    cudaMemcpyAsync(group_node, T.group_node, G * 4, cudaMemcpyDeviceToHost, st);
    if (nn) {
        cudaMemcpyAsync(key, T.key, (size_t)nn * 8, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(parent, T.parent, (size_t)nn * 4, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(depth, T.depth, nn, cudaMemcpyDeviceToHost, st);
    }
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "pcie_tree D2H failed: %s", cudaGetErrorString(e)); return KXPU_E_CUDA; }
    *n_nodes = nn;
    return KXPU_OK;
}

extern "C" int32_t kxpu_pcie_tree(kxpu_ctx *ctx, const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n,
                                  const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                  uint32_t *group_node, uint64_t *key, uint32_t *parent, uint8_t *depth, uint32_t *n_nodes) {
    return pcie_tree(ctx, recs, paths, n, group_off, group_members, n_groups, group_node, key, parent, depth, n_nodes, nullptr);
}

extern "C" int32_t kxpu_pcie_tree_sriov(kxpu_ctx *ctx, const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n,
                                        const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                        uint32_t *group_node, uint64_t *key, uint32_t *parent, uint8_t *depth,
                                        uint32_t *n_nodes, const uint32_t *pf_of) {
    if (!ctx || (n && !pf_of)) return KXPU_E_INVALID;
    if (n >= (1ull << 28)) return KXPU_E_UNSUPPORTED;
    for (size_t i = 0; i < n; i++)
        if (pf_of[i] != KXPU_NO_PF && pf_of[i] >= n) {
            KX_SET_ERR(ctx, "pcie_tree_sriov: pf_of[%zu] = %u is >= n", i, pf_of[i]);
            return KXPU_E_INVALID;
        }
    static const uint32_t none = KXPU_NO_PF;  // n == 0: nothing to upload, but still the variant
    return pcie_tree(ctx, recs, paths, n, group_off, group_members, n_groups, group_node, key, parent, depth, n_nodes,
                     n ? pf_of : &none);
}

extern "C" int32_t kxpu_pcie_tree_mdev(kxpu_ctx *ctx, const kxpu_mdevrec *recs, const kxpu_pcipath *paths, size_t n,
                                       const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                       uint32_t *group_node, uint64_t *key, uint32_t *parent, uint8_t *depth, uint32_t *n_nodes) {
    static_assert(sizeof(kxpu_mdevrec) == 128 && offsetof(kxpu_mdevrec, parent) + 16 <= 64, "kxpu_mdevrec layout");
    return pcie_tree(ctx, recs, paths, n, group_off, group_members, n_groups, group_node, key, parent, depth, n_nodes, nullptr);
}

// Rec = kxpu_devrec: kxpu_pcie_ports; Rec = kxpu_mdevrec: kxpu_pcie_ports_mdev
template <typename Rec>
static int32_t pcie_ports(kxpu_ctx *ctx, const char *what, const Rec *recs, const kxpu_pcipath *paths, size_t n,
                          const uint32_t *group_off, const uint32_t *group_members, size_t n_groups, uint64_t *root_port,
                          uint64_t *pcie_switch) {
    constexpr bool MD = std::is_same<Rec, kxpu_mdevrec>::value;
    static_assert(sizeof(unsigned long long) == sizeof(uint64_t), "keys");
    if (!ctx || (n && (!recs || !paths)) || !group_off) return KXPU_E_INVALID;
    if (n >= (1ull << 28) || n_groups >= (1ull << 28)) return KXPU_E_UNSUPPORTED;
    for (size_t g = 0; g < n_groups; g++)
        if (group_off[g + 1] < group_off[g]) { KX_SET_ERR(ctx, "%s: group %zu: offsets decrease", what, g); return KXPU_E_INVALID; }
    const size_t nm = group_off[n_groups];
    if ((nm && !group_members) || (n_groups && (!root_port || !pcie_switch))) return KXPU_E_INVALID;
    if (n_groups == 0) return KXPU_OK;
    if (nm >= 0x7FFFFFFFull) return KXPU_E_UNSUPPORTED;

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    const size_t G = n_groups;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_recs = take(n * sizeof(Rec)), o_paths = take(n * sizeof(kxpu_pcipath));
    const size_t o_goff = take((G + 1) * 4), o_gmem = take(nm * 4), o_chain = take(n * MAXD * 8), o_clen = take(n);
    const size_t o_rp = take(G * 8), o_sw = take(G * 8), o_err = take(16);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    auto up = [&](size_t o, const void *h, size_t bytes) { if (bytes) cudaMemcpyAsync(b + o, h, bytes, cudaMemcpyHostToDevice, st); };
    up(o_recs, recs, n * sizeof(Rec)); up(o_paths, paths, n * sizeof(kxpu_pcipath));
    up(o_goff, group_off, (G + 1) * 4); up(o_gmem, group_members, nm * 4);
    cudaMemsetAsync(b + o_err, 0, 16, st);
    Tree T;
    memset(&T, 0, sizeof T);  // k_ports reads goff, gmem, n, G, chain, clen and err only
    T.goff = (const uint32_t *)(b + o_goff); T.gmem = (const uint32_t *)(b + o_gmem);
    T.n = (uint32_t)n; T.G = (uint32_t)G;
    T.chain = (const unsigned long long *)(b + o_chain); T.clen = (const uint8_t *)(b + o_clen);
    T.err = (uint32_t *)(b + o_err);
    unsigned long long *d_rp = (unsigned long long *)(b + o_rp), *d_sw = (unsigned long long *)(b + o_sw);
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        if (n) {
            k_parse<Rec, false><<<(unsigned)((n + PARSE_RECS - 1) / PARSE_RECS), PARSE_THREADS, 0, st>>>(
                (const Rec *)(b + o_recs), (const kxpu_pcipath *)(b + o_paths), (uint32_t)n,
                (unsigned long long *)(b + o_chain), b + o_clen, nullptr);
            ctx->launches++;
        }
        (MD ? k_ports_mdev : k_ports)<<<(unsigned)((G + 255) / 256), 256, 0, st>>>(T, d_rp, d_sw);
        ctx->launches++;
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, T.err, 4, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) { KX_SET_ERR(ctx, "%s: a group member index is >= n", what); return KXPU_E_INVALID; }
    cudaMemcpyAsync(root_port, d_rp, G * 8, cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(pcie_switch, d_sw, G * 8, cudaMemcpyDeviceToHost, st);
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s D2H failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    return KXPU_OK;
}

extern "C" int32_t kxpu_pcie_ports(kxpu_ctx *ctx, const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n,
                                   const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                   uint64_t *root_port, uint64_t *pcie_switch) {
    return pcie_ports(ctx, "pcie_ports", recs, paths, n, group_off, group_members, n_groups, root_port, pcie_switch);
}

extern "C" int32_t kxpu_pcie_ports_mdev(kxpu_ctx *ctx, const kxpu_mdevrec *recs, const kxpu_pcipath *paths, size_t n,
                                        const uint32_t *group_off, const uint32_t *group_members, size_t n_groups,
                                        uint64_t *root_port, uint64_t *pcie_switch) {
    return pcie_ports(ctx, "pcie_ports_mdev", recs, paths, n, group_off, group_members, n_groups, root_port, pcie_switch);
}

// Rec = kxpu_devrec: kxpu_aer_ports; Rec = kxpu_mdevrec: kxpu_aer_ports_mdev
template <typename Rec>
static int32_t aer_ports(kxpu_ctx *ctx, const char *what, const Rec *recs, const kxpu_pcipath *paths, size_t n,
                         uint32_t *port_off, uint32_t *port_of, uint64_t *port_key, uint32_t *n_ports) {
    constexpr bool MD = std::is_same<Rec, kxpu_mdevrec>::value;
    if (!ctx || (n && (!recs || !paths)) || !port_off || (n && (!port_of || !port_key || !n_ports))) return KXPU_E_INVALID;
    if (n >= (1ull << 28)) return KXPU_E_UNSUPPORTED;
    if (n == 0) {
        port_off[0] = 0;
        if (n_ports) *n_ports = 0;
        return KXPU_OK;
    }

    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    kx_clear_timings(ctx);
    const size_t NP = (size_t)PORTS_MAX * n;  // bounds the positions
    uint32_t slots = 1;
    while (slots < 2 * NP) slots <<= 1;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) / 256 * 256; return o; };
    const size_t o_recs = take(n * sizeof(Rec)), o_paths = take(n * sizeof(kxpu_pcipath));
    const size_t o_chain = take(n * MAXD * 8), o_clen = take(n);
    const size_t o_cnt = take(n * 4), o_off = take(n * 4), o_fcnt = take(n * 4), o_fbase = take(n * 4);
    const size_t o_slots = take((size_t)slots * 4), o_pslot = take(NP * 4), o_pfirst = take(NP);
    const size_t o_of = take(NP * 4), o_key = take(NP * 8), o_err = take(32);
    KxScratch sc(ctx);
    uint8_t *b = nullptr;
    KX_CUDA(ctx, sc.alloc((void **)&b, off));
    cudaStream_t st = ctx->stream;
    cudaMemcpyAsync(b + o_recs, recs, n * sizeof(Rec), cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(b + o_paths, paths, n * sizeof(kxpu_pcipath), cudaMemcpyHostToDevice, st);
    cudaMemsetAsync(b + o_slots, 0xFF, (size_t)slots * 4, st);
    cudaMemsetAsync(b + o_err, 0, 32, st);
    Ports P;
    P.n = (uint32_t)n;
    P.chain = (const unsigned long long *)(b + o_chain); P.clen = b + o_clen;
    P.cnt = (uint32_t *)(b + o_cnt); P.off = (uint32_t *)(b + o_off);
    P.fcnt = (uint32_t *)(b + o_fcnt); P.fbase = (uint32_t *)(b + o_fbase);
    P.slots = (uint32_t *)(b + o_slots); P.mask = slots - 1;
    P.pslot = (uint32_t *)(b + o_pslot); P.pfirst = b + o_pfirst;
    P.port_of = (uint32_t *)(b + o_of); P.port_key = (unsigned long long *)(b + o_key);
    P.err = (uint32_t *)(b + o_err);
    unsigned long long *d_totals = (unsigned long long *)(b + o_err + 16);  // positions, distinct ports
    {
        KxTimer tm(ctx, KXPU_T_CLASSIFY);
        k_parse<Rec, false><<<(unsigned)((n + PARSE_RECS - 1) / PARSE_RECS), PARSE_THREADS, 0, st>>>(
            (const Rec *)(b + o_recs), (const kxpu_pcipath *)(b + o_paths), (uint32_t)n,
            (unsigned long long *)(b + o_chain), b + o_clen, nullptr);
        const unsigned nb = (unsigned)((n + 255) / 256);
        k_port_count<MD><<<nb, 256, 0, st>>>(P);
        ctx->launches += 2;
        int32_t rc = kxscan::exclusive_scan(ctx, P.cnt, n, P.off, d_totals);
        if (rc != KXPU_OK) return rc;
        k_port_insert<MD><<<nb, 256, 0, st>>>(P);
        k_port_first<MD><<<nb, 256, 0, st>>>(P);
        ctx->launches += 2;
        rc = kxscan::exclusive_scan(ctx, P.fcnt, n, P.fbase, d_totals + 1);
        if (rc != KXPU_OK) return rc;
        k_port_key<MD><<<nb, 256, 0, st>>>(P);
        k_port_of<<<nb, 256, 0, st>>>(P);
        ctx->launches += 2;
    }
    uint32_t *h = ctx->h_ctl;
    cudaMemcpyAsync(h, P.err, 32, cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    if (h[0]) { KX_SET_ERR(ctx, "%s: port table overflow", what); return KXPU_E_CAPACITY; }
    const uint32_t np = h[4], nk = h[6];  // the two totals' low words (each below 2^31)
    cudaMemcpyAsync(port_off, P.off, n * 4, cudaMemcpyDeviceToHost, st);
    if (np) cudaMemcpyAsync(port_of, P.port_of, (size_t)np * 4, cudaMemcpyDeviceToHost, st);
    if (nk) cudaMemcpyAsync(port_key, P.port_key, (size_t)nk * 8, cudaMemcpyDeviceToHost, st);
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { KX_SET_ERR(ctx, "%s D2H failed: %s", what, cudaGetErrorString(e)); return KXPU_E_CUDA; }
    port_off[n] = np;
    *n_ports = nk;
    return KXPU_OK;
}

extern "C" int32_t kxpu_aer_ports(kxpu_ctx *ctx, const kxpu_devrec *recs, const kxpu_pcipath *paths, size_t n,
                                  uint32_t *port_off, uint32_t *port_of, uint64_t *port_key, uint32_t *n_ports) {
    return aer_ports(ctx, "aer_ports", recs, paths, n, port_off, port_of, port_key, n_ports);
}

extern "C" int32_t kxpu_aer_ports_mdev(kxpu_ctx *ctx, const kxpu_mdevrec *recs, const kxpu_pcipath *paths, size_t n,
                                       uint32_t *port_off, uint32_t *port_of, uint64_t *port_key, uint32_t *n_ports) {
    return aer_ports(ctx, "aer_ports_mdev", recs, paths, n, port_off, port_of, port_key, n_ports);
}
