"""Synthetic inputs for BASELINE.json configs[0..4] (SURVEY.md 8(d)).  Pure numpy, seeded;
shared by tests/ and bench.py.  Nothing here is on the product path."""
import gzip
import os

import numpy as np

from .binding import (CDIDEV_DTYPE, DEVREC_DTYPE, MDEVREC_DTYPE, REC_DRIVER_ERR, REC_IOMMU_ERR, REC_NAME_ERR,
                      REC_VENDOR_ERR)

_REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PCI_IDS_GZ = os.path.join(_REPO, "tests", "golden", "pci.ids.gz")
PCI_IDS_SHA256 = "33bd4fd9762e99556748bb7f85a81912c7f742c6226eccf3861d60f4b0ea4d6e"


def load_pci_ids() -> bytes:
    """The reference's bundled utils/pci.ids (v2024.06.23), from the committed fixture."""
    with gzip.open(PCI_IDS_GZ, "rb") as f:
        return f.read()


def make_queries(present_keys, n, seed, hit_frac=0.75):
    """cfg2/cfg4 key mix: hit_frac hits drawn uniformly from the present pairs, the rest
    misses -- half with a present vendor and an absent device, half with an absent vendor (when one exists)."""
    rng = np.random.default_rng(seed)
    present_keys = np.asarray(present_keys, dtype=np.uint32)
    pset = set(int(k) for k in present_keys)
    vendors = np.unique(present_keys >> 16)
    vset = set(int(v) for v in vendors)
    n_hit = int(round(n * hit_frac))
    n_m1 = (n - n_hit) // 2
    n_m2 = n - n_hit - n_m1
    if len(vset) == 65536:  # every vendor id is present (a text of all 65 536 vendors): every miss has an absent device
        n_m1, n_m2 = n - n_hit, 0
    hits = present_keys[rng.integers(0, len(present_keys), n_hit)]
    m1 = np.empty(n_m1, np.uint32)
    i = 0
    while i < n_m1:  # present vendor, absent device
        v = int(vendors[rng.integers(0, len(vendors))])
        d = int(rng.integers(0, 65536))
        k = (v << 16) | d
        if k not in pset:
            m1[i] = k
            i += 1
    m2 = np.empty(n_m2, np.uint32)
    i = 0
    while i < n_m2:  # absent vendor
        v = int(rng.integers(0, 65536))
        if v not in vset:
            m2[i] = (v << 16) | int(rng.integers(0, 65536))
            i += 1
    keys = np.concatenate([hits, m1, m2]).astype(np.uint32)
    rng.shuffle(keys)
    return keys


def cfg2_queries(present_keys):
    return make_queries(present_keys, 1024, 0xC0FFEE)


def cfg4_queries(present_keys, n=1 << 20):
    return make_queries(present_keys, n, 2)


def enumerate_bdfs(n, start=0):
    """First n PCI addresses dddd:bb:dd.f in lexical (= filepath.Walk) order."""
    i = np.arange(start, start + n, dtype=np.int64)
    fn, dev, bus, dom = i & 7, (i >> 3) & 31, (i >> 8) & 255, i >> 16
    hexd = np.frombuffer(b"0123456789abcdef", dtype=np.uint8)
    out = np.zeros((n, 16), np.uint8)
    out[:, 0] = hexd[(dom >> 12) & 15]; out[:, 1] = hexd[(dom >> 8) & 15]
    out[:, 2] = hexd[(dom >> 4) & 15]; out[:, 3] = hexd[dom & 15]
    out[:, 4] = ord(":")
    out[:, 5] = hexd[(bus >> 4) & 15]; out[:, 6] = hexd[bus & 15]
    out[:, 7] = ord(":")
    out[:, 8] = hexd[(dev >> 4) & 15]; out[:, 9] = hexd[dev & 15]
    out[:, 10] = ord(".")
    out[:, 11] = hexd[fn]
    return out


def _id_text(ids):
    """'0x%04x\\n' for an array of 16-bit ids -> (n,8) uint8 (7 bytes used)."""
    ids = np.asarray(ids, dtype=np.int64)
    hexd = np.frombuffer(b"0123456789abcdef", dtype=np.uint8)
    out = np.zeros((len(ids), 8), np.uint8)
    out[:, 0] = ord("0"); out[:, 1] = ord("x")
    for k in range(4):
        out[:, 2 + k] = hexd[(ids >> (12 - 4 * k)) & 15]
    out[:, 6] = ord("\n")
    return out


def cfg3_records(present_keys, n=1 << 20, seed=1):
    """n synthetic sysfs records (SURVEY.md 8(d) cfg3): 50% vendor 10de (device ids Zipf-ish
    over the NVIDIA ids), 50% from {8086,1002,15b3,1d0f}; driver 80% vfio-pci, 10% nvidia,
    10% unreadable link; iommu group = bdf>>3 (all functions of a slot share a group)."""
    rng = np.random.default_rng(seed)
    present_keys = np.asarray(present_keys, dtype=np.uint32)
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    recs["bdf"] = enumerate_bdfs(n).view("S16").reshape(n)
    nv_ids = (present_keys[(present_keys >> 16) == 0x10de] & 0xFFFF).astype(np.int64)
    is_nv = rng.random(n) < 0.5
    # Zipf-ish: 70% of NVIDIA devices come from 16 hot ids
    hot = nv_ids[rng.permutation(len(nv_ids))[:16]]
    pick_hot = rng.random(n) < 0.7
    dev = np.where(pick_hot, hot[rng.integers(0, 16, n)], nv_ids[rng.integers(0, len(nv_ids), n)])
    others = np.array([0x8086, 0x1002, 0x15b3, 0x1d0f], dtype=np.int64)
    ov = others[rng.integers(0, 4, n)]
    vendor = np.where(is_nv, 0x10de, ov)
    for v in others:
        ids = (present_keys[(present_keys >> 16) == v] & 0xFFFF).astype(np.int64)
        sel = (~is_nv) & (ov == v)
        dev[sel] = ids[rng.integers(0, len(ids), int(sel.sum()))]
    recs["vendor_txt"] = _id_text(vendor)
    recs["device_txt"] = _id_text(dev)
    recs["vendor_len"] = 7
    recs["device_len"] = 7
    r = rng.random(n)
    drv = np.where(r < 0.8, b"vfio-pci", np.where(r < 0.9, b"nvidia", b"")).astype("S16")
    recs["driver"] = drv
    recs["flags"] = np.where(r >= 0.9, REC_DRIVER_ERR, 0).astype(np.uint8)
    recs["iommu_group"] = (np.arange(n, dtype=np.int64) >> 3).astype(np.uint32)
    return recs


XPU_VENDORS = (0x10de, 0x1002, 0x8086, 0x15b3, 0x1d0f)


def xpu_records(present_keys, n=1 << 20, seed=4):
    """cfg3's shape for a node with accelerators of several vendors: vendor uniform over XPU_VENDORS, each drawing
    device ids from its own pci.ids rows; 2% of the records of 10de and 1002 take a device id that both vendors
    list (the same id string under two vendors); driver 60% vfio-pci, 10% nvidia, 10% amdgpu, 20% unbound
    (unreadable link); iommu group = bdf>>3, so one group can hold functions of different vendors."""
    rng = np.random.default_rng(seed)
    present_keys = np.asarray(present_keys, dtype=np.uint32)
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    recs["bdf"] = enumerate_bdfs(n).view("S16").reshape(n)
    vendors = np.array(XPU_VENDORS, dtype=np.int64)
    vendor = vendors[rng.integers(0, len(vendors), n)]
    dev = np.zeros(n, np.int64)
    ids = {}
    for v in XPU_VENDORS:
        ids[v] = (present_keys[(present_keys >> 16) == v] & 0xFFFF).astype(np.int64)
        sel = vendor == v
        dev[sel] = ids[v][rng.integers(0, len(ids[v]), int(sel.sum()))]
    shared = np.intersect1d(ids[0x10de], ids[0x1002])
    assert len(shared), "pci.ids lists no device id under both 10de and 1002"
    both = ((vendor == 0x10de) | (vendor == 0x1002)) & (rng.random(n) < 0.02)
    dev[both] = shared[0]
    recs["vendor_txt"] = _id_text(vendor)
    recs["device_txt"] = _id_text(dev)
    recs["vendor_len"] = 7
    recs["device_len"] = 7
    r = rng.random(n)
    drv = np.where(r < 0.6, b"vfio-pci", np.where(r < 0.7, b"nvidia", np.where(r < 0.8, b"amdgpu", b""))).astype("S16")
    recs["driver"] = drv
    recs["flags"] = np.where(r >= 0.8, REC_DRIVER_ERR, 0).astype(np.uint8)
    recs["iommu_group"] = (np.arange(n, dtype=np.int64) >> 3).astype(np.uint32)
    return recs


XPU_RULES = [(b"10de", b"vfio-pci"), (b"1002", b"vfio-pci"), (b"8086", b"vfio-pci"), (b"15b3", b"vfio-pci"),
             (b"1d0f", b"vfio-pci")]


def cfg1_record():
    """One mocked VFIO NVIDIA GPU (SURVEY.md 8(d) cfg1)."""
    recs = np.zeros(1, dtype=DEVREC_DTYPE)
    recs["bdf"] = b"0000:c1:00.0"
    recs["vendor_txt"] = np.frombuffer(b"0x10de\n\0", np.uint8)
    recs["device_txt"] = np.frombuffer(b"0x2330\n\0", np.uint8)
    recs["vendor_len"] = 7
    recs["device_len"] = 7
    recs["driver"] = b"vfio-pci"
    recs["iommu_group"] = 214
    return recs


def cfg5_devices(n=65536):
    """index 0..n-1, group = 1000 + index//2, bdf enumerated as in cfg3 (quoted and plain
    YAML forms both occur)."""
    devs = np.zeros(n, dtype=CDIDEV_DTYPE)
    devs["bdf"] = enumerate_bdfs(n).view("S16").reshape(n)
    devs["iommu_group"] = (1000 + np.arange(n) // 2).astype(np.uint32)
    devs["index"] = np.arange(n, dtype=np.uint64)
    return devs


def synthetic_pci_ids(n_vendors, devs_per_vendor, subs_per_dev=1, seed=7, copies=1):
    """pci.ids-shaped synthetic text WITHOUT replication (north_star's "pci.ids-shaped synthetic text"):
    n_vendors distinct vendor ids (<= 65536), each with devs_per_vendor distinct device ids and
    subs_per_dev subsystem lines per device -- every vendor block is a first occurrence, so the parse
    cannot skip anything ("all-alive" text).  Fixed-width lines (vendor 29 B, device 42 B, subsystem
    38 B: close to the 38 B mean of the real file).  numpy only; returns a uint8 array."""
    assert 0 < n_vendors <= 65536 and 0 < devs_per_vendor <= 65536
    hexd = np.frombuffer(b"0123456789abcdef", np.uint8)
    rng = np.random.default_rng(seed)
    v_ids = rng.permutation(65536)[:n_vendors].astype(np.int64)
    v_ids.sort()  # the real file is sorted by vendor id

    def put_hex4(arr, col, vals):
        for k in range(4):
            arr[..., col + k] = hexd[(vals >> (12 - 4 * k)) & 15]

    def put_dec(arr, col, vals, width):
        for k in range(width):
            arr[..., col + width - 1 - k] = ord("0") + (vals // 10 ** k) % 10

    vline = np.frombuffer(b"vvvv  Vendor Corp. Nr 00000\n", np.uint8)
    dline = np.frombuffer(b"\tdddd  Device / Model 00000 [Rev. 000000]\n", np.uint8)
    sline = np.frombuffer(b"\t\tvvvv dddd  Subsystem board 00000\n", np.uint8)
    block = len(vline) + devs_per_vendor * (len(dline) + subs_per_dev * len(sline))
    out = np.empty((n_vendors, block), np.uint8)
    out[:, :len(vline)] = vline
    put_hex4(out, 0, v_ids)
    put_dec(out, 22, v_ids, 5)
    body = out[:, len(vline):].reshape(n_vendors, devs_per_vendor, len(dline) + subs_per_dev * len(sline))
    # distinct device ids per vendor: an odd stride walks all 65536 values
    start = rng.integers(0, 65536, n_vendors)[:, None]
    stride = (rng.integers(0, 32768, n_vendors)[:, None] * 2 + 1)
    d_ids = (start + stride * np.arange(devs_per_vendor)[None, :]) & 0xFFFF
    body[:, :, :len(dline)] = dline
    put_hex4(body, 1, d_ids)
    put_dec(body, 22, d_ids, 5)
    put_dec(body, 34, (d_ids * 7919) % 1000000, 6)
    for s in range(subs_per_dev):
        o = len(dline) + s * len(sline)
        body[:, :, o:o + len(sline)] = sline
        put_hex4(body, o + 2, np.broadcast_to(v_ids[:, None], d_ids.shape))
        put_hex4(body, o + 7, (d_ids + s + 1) & 0xFFFF)
        put_dec(body, o + 29, d_ids, 5)
    flat = out.reshape(-1)
    return np.tile(flat, copies) if copies > 1 else flat


MDEV_RULES = [(b"10de", b"nvidia-vgpu"), (b"10de", b"vfio_mdev"), (b"8086", b"vfio_mdev"), (b"1002", b"vfio_mdev")]
MDEV_TYPE_NAMES = [b"GRID T4-1Q\n", b"GRID T4-2B\n", b"GRID V100-8Q", b"NVIDIA A100-4C\n", b"NVIDIA  A100-4C",
                   b"GRID A40-24Q (x)\n", b"i915-GVTg_V5_4", b"  GRID\tT4-1Q \n\n", b"\n", b"MxGPU+/vf 2"]


def uuids(n, seed=0):
    """n distinct random canonical lowercase UUIDs in lexical order, as an (n, 36) uint8 array."""
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 16, (n, 32), dtype=np.uint8)
    raw[:, 0] = (np.arange(n, dtype=np.int64) * 16 // max(n, 1)).astype(np.uint8)  # spread, then sort
    hexd = np.frombuffer(b"0123456789abcdef", np.uint8)
    out = np.full((n, 36), ord("-"), np.uint8)
    cols = [c for c in range(36) if c not in (8, 13, 18, 23)]
    out[:, cols] = hexd[raw]
    s = np.unique(out.view("S36").reshape(n))  # sorted, distinct
    if len(s) < n:  # astronomically unlikely; keep n rows
        s = np.concatenate([s, s[:n - len(s)]])
    return s.view(np.uint8).reshape(n, 36)


def mdev_records(n=1 << 20, seed=5):
    """n synthetic /sys/bus/mdev/devices records (kxpu_mdevrec), entries in lexical UUID order.  Parent vendors
    10de (60 %), 8086, 1002 and 1af4; mdev drivers nvidia-vgpu, vfio_mdev and others; type names from a few
    realistic ones (inner runs of spaces, trailing newlines, bytes the type key deletes, a name that is only white
    space) plus about 6 000 generated ones; groups shared by two mdevs each; 10 % read errors over the vendor,
    driver, iommu_group and name reads.  Every rule of MDEV_RULES matches part of the records."""
    rng = np.random.default_rng(seed)
    recs = np.zeros(n, dtype=MDEVREC_DTYPE)
    recs["uuid"] = uuids(n, seed).view("S36").reshape(n)
    recs["parent"] = enumerate_bdfs(n >> 4 or 1)[np.arange(n) >> 4].view("S16").reshape(n)
    vend = np.array([0x10de, 0x8086, 0x1002, 0x1af4], np.int64)[np.searchsorted([0.6, 0.75, 0.9], rng.random(n), side="right")]
    recs["parent_vendor_txt"] = _id_text(vend)
    recs["vendor_len"] = 7
    r = rng.random(n)
    recs["driver"] = np.where(r < 0.5, b"nvidia-vgpu", np.where(r < 0.9, b"vfio_mdev", b"i915")).astype("S16")
    gen = [b"NVIDIA L40S-%dQ%s" % (k, b"\n" if k & 1 else b"") for k in range(6000)]
    pool = MDEV_TYPE_NAMES + gen
    pa = np.zeros((len(pool), 40), np.uint8)
    pl = np.zeros(len(pool), np.uint8)
    for i, nm in enumerate(pool):
        pa[i, :len(nm)] = np.frombuffer(nm, np.uint8)
        pl[i] = len(nm)
    pick = np.where(rng.random(n) < 0.7, rng.integers(0, len(MDEV_TYPE_NAMES), n), rng.integers(0, len(pool), n))
    recs["type_name"] = pa[pick]
    recs["name_len"] = pl[pick]
    recs["iommu_group"] = (np.arange(n, dtype=np.int64) >> 1).astype(np.uint32) + 100
    e = rng.random(n)
    flags = np.zeros(n, np.uint8)
    flags[e < 0.025] = REC_VENDOR_ERR
    flags[(e >= 0.025) & (e < 0.05)] = REC_DRIVER_ERR
    flags[(e >= 0.05) & (e < 0.075)] = REC_IOMMU_ERR
    flags[(e >= 0.075) & (e < 0.1)] = REC_NAME_ERR
    recs["flags"] = flags
    return recs


def mdev_devices(n=65536, seed=6):
    """n kxpu_mdevcdi entries: index 0..n-1, one group each, parents enumerated as in cfg3 (quoted and plain YAML
    forms both occur)."""
    from .binding import MDEVCDI_DTYPE
    devs = np.zeros(n, dtype=MDEVCDI_DTYPE)
    devs["uuid"] = uuids(n, seed).view("S36").reshape(n)
    devs["parent"] = enumerate_bdfs(n).view("S16").reshape(n)
    devs["iommu_group"] = (2000 + np.arange(n)).astype(np.uint32)
    devs["index"] = np.arange(n, dtype=np.uint64)
    return devs


# ---------------------------------------------------------------- NUMA topology (ABI v5)
def _numa_assign(recs, bus, nodes, rng):
    """numa_node / KXPU_REC_NUMA by bus range over `nodes` nodes, 3 % unknown (no flag), and about 1 % of the records
    moved to another node (some groups then span two nodes)."""
    from .binding import NUMA_FIELD, REC_NUMA
    n = len(recs)
    node = bus * nodes // (int(bus.max()) + 1 if n else 1)  # contiguous bus ranges, one per node
    moved = rng.random(n) < 0.01
    node = np.where(moved, (node + 1 + rng.integers(0, max(nodes - 1, 1), n)) % nodes, node)
    known = rng.random(n) >= 0.03
    recs[NUMA_FIELD] = np.where(known, node, 0).astype(np.uint8)
    recs["flags"] = recs["flags"] | np.where(known, REC_NUMA, 0).astype(np.uint8)
    return recs


def topo_records(present_keys, n=1 << 20, nodes=2, seed=1):
    """cfg3_records(present_keys, n, seed) plus a NUMA assignment by PCI bus range over `nodes` nodes (2 or 4):
    3 % unknown nodes and a few functions on another node than the rest of their slot (multi-node groups)."""
    recs = cfg3_records(present_keys, n, seed)
    bus = np.arange(n, dtype=np.int64) >> 8  # domain:bus of the walk position
    return _numa_assign(recs, bus, nodes, np.random.default_rng(seed + 100))


def topo_mdev_records(n=1 << 20, nodes=2, seed=5):
    """mdev_records(n, seed) with the parents' NUMA nodes assigned like topo_records (by the parent's bus)."""
    recs = mdev_records(n, seed)
    bus = (np.arange(n, dtype=np.int64) >> 4) >> 8  # domain:bus of the parent
    return _numa_assign(recs, bus, nodes, np.random.default_rng(seed + 100))


def topo_requests(dev_numa, n_req=4096, avail=16, size=8, must_max=2, seed=9):
    """n_req GetPreferredAllocation container requests over a device list with masks dev_numa: each offers `avail`
    distinct random positions, must-include 0..must_max of them, and asks for `size`.  avail = len(dev_numa) with
    n_req = 1 is the one-request-over-everything case."""
    rng = np.random.default_rng(seed)
    n = len(dev_numa)
    reqs = []
    for _ in range(n_req):
        av = rng.permutation(n)[:avail] if avail < n else rng.permutation(n)
        nm = int(rng.integers(0, must_max + 1))
        mu = av[rng.permutation(len(av))[:nm]]
        reqs.append((av.astype(np.uint32), mu.astype(np.uint32), size))
    return reqs


def topo_dev_numa(n, nodes=4, seed=11):
    """NUMA masks of n devices: by position range over `nodes` nodes, 5 % unknown (0), 2 % on two nodes."""
    rng = np.random.default_rng(seed)
    node = (np.arange(n, dtype=np.int64) * nodes // max(n, 1))
    m = (np.uint64(1) << node.astype(np.uint64))
    two = rng.random(n) < 0.02
    m = np.where(two, m | (np.uint64(1) << ((node + 1) % nodes).astype(np.uint64)), m)
    return np.where(rng.random(n) < 0.05, np.uint64(0), m).astype(np.uint64)


# ---------------------------------------------------------------- PCIe topology (ABI v7)
def _pcie_prefix(dom, bus, dev, kind):
    """Components above the function at dom:bus:dev.  An HGX-like board: a host bridge per 64 buses, 8 root ports
    under it, a switch per bus, a down port per slot.  kind 1: a VMD domain between the root port and the switch;
    2: 4 more bridge levels (a chain of exactly 8); 3: 5 more (9: unknown); 4: upper-case hex (unknown)."""
    hb = bus & 0xC0
    comps = ["pci%04x:%02x" % (dom, hb), "%04x:%02x:%02x.0" % (dom, hb, ((bus >> 3) & 7) + 1)]
    if kind == 1:
        comps += ["%04x:%02x:00.5" % (dom, hb), "pci10000:e0", "10000:e0:%02x.0" % (bus & 0x1F)]
    if kind in (2, 3):
        comps += ["%04x:%02x:%02x.0" % (dom, (bus + 1 + k) & 0xFF, k) for k in range(4 if kind == 2 else 5)]
    comps += ["%04x:%02x:00.0" % (dom, bus), "%04x:%02x:%02x.0" % (dom, bus, dev)]
    if kind == 4:
        comps[1] = comps[1].upper().replace("X", "x")
    return "/".join(comps) + "/"


def pcie_walk(n=1 << 20, seed=21, group_max=4):
    """n records (DEVREC_DTYPE, bdfs in walk order) with their kxpu_pcipath side records and a group CSR over them
    (groups of 1..group_max consecutive records, 4 % of the records in no group).  Per bus: 2 % behind a VMD domain,
    1 % with a chain of exactly 8, 1 % with 9 (unknown), 1 % with upper-case hex (unknown); per record: 3 % unknown
    (len 0), 0.5 % with a trailing '/'.  A group may straddle two slots or buses, so its chain is the common prefix.
    Returns (recs, paths, group_off, group_members)."""
    from .binding import PCIPATH_DTYPE
    rng = np.random.default_rng(seed)
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    bdfs = enumerate_bdfs(n)
    recs["bdf"] = bdfs.view("S16").reshape(n)
    recs["driver"] = b"vfio-pci"
    recs["vendor_txt"] = _id_text(np.full(n, 0x10DE))
    recs["device_txt"] = _id_text(np.full(n, 0x2330))
    recs["vendor_len"] = recs["device_len"] = 7
    i = np.arange(n, dtype=np.int64)
    dom, bus, dev = i >> 16, (i >> 8) & 255, (i >> 3) & 31
    n_bus = int((n + 255) >> 8)
    bus_kind = rng.choice(5, size=n_bus, p=[0.95, 0.02, 0.01, 0.01, 0.01])
    texts = []
    cache = {}
    for k in range(n):
        slot = int(k >> 3)
        pre = cache.get(slot)
        if pre is None:
            pre = cache[slot] = _pcie_prefix(int(dom[k]), int(bus[k]), int(dev[k]), int(bus_kind[k >> 8]))
        texts.append(pre + bytes(bdfs[k][:12]).decode())
    paths = np.zeros(n, dtype=PCIPATH_DTYPE)
    paths["path"] = np.array([t.encode() for t in texts], dtype="S120")
    paths["len"] = np.array([len(t) for t in texts], np.uint8)
    r = rng.random(n)
    paths["len"][r < 0.03] = 0
    trail = (r >= 0.03) & (r < 0.035)
    for k in np.nonzero(trail)[0]:
        t = texts[k] + "/"
        paths["path"][k], paths["len"][k] = t.encode(), len(t)
    sizes = rng.integers(1, group_max + 1, n)
    starts = np.cumsum(sizes) - sizes
    starts = starts[starts < n]
    keep = rng.random(n) >= 0.04
    members, off = [], [0]
    for g, s in enumerate(starts):
        e = min(int(s) + int(sizes[g]), n)
        m = [x for x in range(int(s), e) if keep[x]]
        if not m:
            continue
        members.extend(m)
        off.append(len(members))
    recs["iommu_group"] = np.repeat(np.arange(len(starts), dtype=np.uint32), np.diff(np.append(starts, n)))
    return recs, paths, np.array(off, np.uint32), np.array(members, np.uint32)


def pcie_mdev_walk(n=1 << 20, seed=23, per_gpu=32):
    """n mdev records (MDEVREC_DTYPE, UUIDs in lexical order, one group each) with the kxpu_pcipath of each entry's link,
    and a PCI twin with the same forest shape.  per_gpu vGPUs per parent GPU, the parents scattered over the walk order
    (lexical UUID order says nothing about the hardware).  Per domain: a host bridge, 8 root ports, a switch under each
    with one down port per GPU; 3 % of the paths unknown (len 0), 1 % with an upper-case UUID (unknown).  The twin's
    record k is a PCI function whose path is the same chain followed by its own bdf, so kxpu_pcie_tree gives it the
    chain of mdev k.  Returns (recs, paths, group_off, group_members, twin_recs, twin_paths)."""
    from .binding import PCIPATH_DTYPE
    rng = np.random.default_rng(seed)
    n_gpu = max((n + per_gpu - 1) // per_gpu, 1)
    g = np.arange(n_gpu, dtype=np.int64)
    dom, bus = g >> 8, g & 255
    pre, gpu = [], []
    for d, b in zip(dom.tolist(), bus.tolist()):
        gb = "%04x:%02x:00.0" % (d, b)
        pre.append("pci%04x:00/%04x:00:%02x.0/%04x:%02x:00.0/%04x:%02x:%02x.0/%s"
                   % (d, d, 1 + (b >> 5), d, 0xE0 | (b >> 5), d, 0xE8 | (b >> 5), b & 31, gb))
        gpu.append(gb)
    pre, gpu = np.array(pre, dtype="S96"), np.array(gpu, dtype="S16")
    gpu_of = rng.permutation(n) // per_gpu
    recs = np.zeros(n, dtype=MDEVREC_DTYPE)
    u = uuids(n, seed).view("S36").reshape(n)
    recs["uuid"] = u
    recs["parent"] = gpu[gpu_of]
    recs["parent_vendor_txt"] = _id_text(np.full(n, 0x10DE))
    recs["vendor_len"] = 7
    recs["driver"] = b"nvidia-vgpu"
    recs["iommu_group"] = np.arange(n, dtype=np.uint32) + 100
    r = rng.random(n)
    leaf = np.where((r >= 0.03) & (r < 0.04), np.char.upper(u), u)
    text = np.char.add(np.char.add(pre[gpu_of], b"/"), leaf)
    paths = np.zeros(n, dtype=PCIPATH_DTYPE)
    paths["path"] = text.astype("S120")
    paths["len"] = np.where(r < 0.03, 0, np.char.str_len(text)).astype(np.uint8)
    twin = np.zeros(n, dtype=DEVREC_DTYPE)
    bdfs = enumerate_bdfs(n).view("S16").reshape(n)
    twin["bdf"] = bdfs
    twin_text = np.char.add(np.char.add(pre[gpu_of], b"/"), bdfs)
    twin_paths = np.zeros(n, dtype=PCIPATH_DTYPE)
    twin_paths["path"] = twin_text.astype("S120")
    twin_paths["len"] = np.where(r < 0.04, 0, np.char.str_len(twin_text)).astype(np.uint8)
    off = np.arange(n + 1, dtype=np.uint32)
    return recs, paths, off, np.arange(n, dtype=np.uint32), twin, twin_paths


# ---------------------------------------------------------------- runtime rediscovery (ABI v6)
def fnv1a64(data: bytes) -> int:
    """64-bit FNV-1a: the snapshot tag of an mdev (over its type key)."""
    h = 0xCBF29CE484222325
    for c in data:
        h = ((h ^ c) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


def pack_id_text(txt: bytes) -> int:
    """An id string (e.g. b"2330") packed little-endian into a u64, NUL padded: what kxpu_classify's dev_ids holds and
    the snapshot tag of a PCI function."""
    return int.from_bytes(txt[:8].ljust(8, b"\0"), "little")


def snapshot_of_records(recs, accept_index):
    """The snapshot (SNAPREC_DTYPE) of a PCI walk: one entry per accepted record in walk order, key = bdf, group,
    klass 0, tag = the packed device id text, index = busIndex."""
    from .binding import SNAPREC_DTYPE
    acc = np.nonzero(np.asarray(accept_index) != 0xFFFFFFFF)[0]
    snap = np.zeros(len(acc), SNAPREC_DTYPE)
    snap["key"] = recs["bdf"][acc]
    snap["iommu_group"] = recs["iommu_group"][acc]
    dl = recs["device_len"][acc].astype(np.int64)
    txt = recs["device_txt"][acc].copy()
    txt[:, :6] = txt[:, 2:8]  # readIDFromFile: data[2:], '\n' trimmed
    txt[:, 6:] = 0
    pos = np.arange(8)[None, :]
    keep = pos < np.maximum(dl - 2, 0)[:, None]
    keep &= np.cumsum(txt == ord("\n"), axis=1) == 0
    snap["tag"] = np.where(keep, txt, 0).astype(np.uint8).view("<u8").reshape(-1)
    snap["index"] = np.asarray(accept_index)[acc]
    return snap


def reconcile_pair(seed=3, n=1 << 20, mdev=False):
    """(prev, cur, next_index) of a rediscovery.  prev: an n-entry accepted snapshot (PCI addresses, or UUIDs with
    mdev=True) in lexical walk order, indices 0..n-1, next_index = n.  cur: the next walk, with 5 % of prev removed,
    5 % new keys interleaved in lexical order, and 1 % each with a changed group, a changed class and a changed tag.
    Tags: packed device id texts (PCI) or FNV-1a 64 of type keys (mdev), a few distinct values."""
    from .binding import SNAPREC_DTYPE
    rng = np.random.default_rng(seed)
    m = n + n // 20
    if mdev:
        keys = uuids(m, seed).view("S36").reshape(m)
        tags = np.array([fnv1a64(b"GRID_T4-%dQ" % k) for k in (1, 2, 4, 8, 16)], np.uint64)
    else:
        keys = enumerate_bdfs(m).view("S16").reshape(m)
        tags = np.array([pack_id_text(b"%04x" % d) for d in (0x2330, 0x2331, 0x20b5, 0x26b9, 0x1db6)], np.uint64)
    is_new = np.zeros(m, bool)
    is_new[rng.permutation(m)[:m - n]] = True
    group = (np.arange(m, dtype=np.int64) >> 1).astype(np.uint32) + 7
    klass = rng.integers(0, 3, m).astype(np.uint32)
    tag = tags[rng.integers(0, len(tags), m)]
    prev = np.zeros(n, SNAPREC_DTYPE)
    pi = np.nonzero(~is_new)[0]
    prev["key"], prev["iommu_group"], prev["klass"], prev["tag"] = keys[pi], group[pi], klass[pi], tag[pi]
    prev["index"] = np.arange(n, dtype=np.uint64)
    removed = np.zeros(m, bool)
    removed[pi[rng.permutation(n)[:n // 20]]] = True
    ci = np.nonzero(~removed)[0]
    cur = np.zeros(len(ci), SNAPREC_DTYPE)
    cur["key"], cur["iommu_group"], cur["klass"], cur["tag"] = keys[ci], group[ci], klass[ci], tag[ci]
    cur["index"] = rng.integers(0, 1 << 62, len(ci), dtype=np.uint64)  # ignored by the call
    survivors = np.nonzero(~is_new[ci])[0]
    pick = rng.permutation(len(survivors))[:3 * (n // 100)]
    g_, k_, t_ = np.array_split(survivors[pick], 3)
    cur["iommu_group"][g_] += np.uint32(1 << 20)
    cur["klass"][k_] = (cur["klass"][k_] + 1) % 3
    tag_pos = {int(v): i for i, v in enumerate(tags)}
    cur["tag"][t_] = tags[[(tag_pos[int(v)] + 1) % len(tags) for v in cur["tag"][t_]]]
    return prev, cur, n


# ---------------------------------------------------------------- IOMMU group viability (ABI v8)
VIAB_RULES = [(b"10de", b"vfio-pci")]


def viab_records(n=1 << 20, seed=31):
    """n records in HGX-like IOMMU groups for kxpu_classify_viable, one 8-function slot per group.  Slot kinds:
      - 55 % GPU: a 10de:2330 GPU on vfio-pci and its 10de:22a3 HD-audio function behind it (40 % on snd_hda_intel, a
        blocker; 40 % on vfio-pci, a member; 20 % unbound).  In a fifth of these slots function 0 is a NIC on ixgbe (a
        blocker in front of the GPU) and the GPU moves to function 1.  The other functions: 30 % switch ports on
        pcieport, 10 % on a host driver (blockers behind the members), the rest unbound;
      - 15 % switch: every function on pcieport;
      - 15 % host: NVMe drives and NICs on their host drivers, every one a blocker (blocker-only groups);
      - 15 % empty: every function unbound.
    A tenth of the slots share the group of the slot before them (no ACS between them), so some groups hold several
    blockers and a blocker may sit far behind the group's first member.  Blockers carry KXPU_REC_BLOCKS and their
    group, as the host stores them; unbound functions carry KXPU_REC_DRIVER_ERR."""
    from .binding import REC_BLOCKS
    rng = np.random.default_rng(seed)
    i = np.arange(n, dtype=np.int64)
    slot, fn = i >> 3, i & 7
    n_slots = int(slot[-1]) + 1 if n else 0
    kind = rng.choice(4, n_slots, p=[0.55, 0.15, 0.15, 0.15])[slot]
    shift = (rng.random(n_slots) < 0.2)[slot]  # GPU slots: a blocker in front of the GPU
    audio = rng.choice(3, n_slots, p=[0.4, 0.4, 0.2])[slot]
    merged = rng.random(n_slots) < 0.1
    merged[:1] = False
    group = np.arange(n_slots, dtype=np.int64)
    for s in np.flatnonzero(merged):
        group[s] = group[s - 1]
    r = rng.random(n)
    vendor = np.full(n, 0x8086, np.int64)
    dev = np.full(n, 0x1533, np.int64)
    drv = np.full(n, b"", "S16")
    blocks = np.zeros(n, bool)
    gpu_fn = np.where(shift, 1, 0)
    is_gpu = (kind == 0) & (fn == gpu_fn)
    is_audio = (kind == 0) & (fn == gpu_fn + 1)
    front = (kind == 0) & shift & (fn == 0)
    rest = (kind == 0) & ~is_gpu & ~is_audio & ~front
    vendor[is_gpu | is_audio] = 0x10de
    dev[is_gpu] = 0x2330
    dev[is_audio] = 0x22a3
    drv[is_gpu] = b"vfio-pci"
    drv[is_audio & (audio == 0)] = b"snd_hda_intel"
    drv[is_audio & (audio == 1)] = b"vfio-pci"
    blocks |= is_audio & (audio == 0)
    drv[front] = b"ixgbe"
    blocks |= front
    port = (rest & (r < 0.3)) | (kind == 1)
    vendor[port], dev[port], drv[port] = 0x10b5, 0xc010, b"pcieport"
    host = (rest & (r >= 0.3) & (r < 0.4)) | (kind == 2)
    hsel = rng.integers(0, 3, n)
    vendor[host] = np.array([0x144d, 0x15b3, 0x8086])[hsel[host]]
    dev[host] = np.array([0xa80a, 0x1021, 0x10fb])[hsel[host]]
    drv[host] = np.array([b"nvme", b"mlx5_core", b"ixgbe"], "S16")[hsel[host]]
    blocks |= host
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    recs["bdf"] = enumerate_bdfs(n).view("S16").reshape(n)
    recs["vendor_txt"] = _id_text(vendor)
    recs["device_txt"] = _id_text(dev)
    recs["vendor_len"] = 7
    recs["device_len"] = 7
    recs["driver"] = drv
    recs["flags"] = np.where(drv == b"", REC_DRIVER_ERR, 0).astype(np.uint8) | np.where(blocks, REC_BLOCKS, 0).astype(np.uint8)
    recs["iommu_group"] = group[slot].astype(np.uint32)
    return recs


# ---------------------------------------------------------------- DRA ResourceSlices (ABI v9)
def dra_devices(n=1 << 16, seed=41):
    """n published devices with every optional attribute present and the longest fields the host produces: a 64-byte
    product name, a 12-byte PCI address, a 10-byte PCIe root, 4-digit ids, one NUMA node, 9-digit groups"""
    from .binding import DRADEV_DTYPE
    rng = np.random.default_rng(seed)
    d = np.zeros(n, DRADEV_DTYPE)
    alnum = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_", np.uint8)
    d["product"] = alnum[rng.integers(0, len(alnum), (n, 64))]
    d["product_len"] = 64
    i = np.arange(n)
    d["bdf"] = [b"%04x:%02x:%02x.%d" % (k >> 13, (k >> 5) & 0xff, (k >> 3) & 0x1f, k & 7) for k in range(n)]
    d["pcie_root"] = [b"pci%04x:%02x" % (k >> 13, (k >> 5) & 0xff) for k in range(n)]
    d["vendor"], d["device"] = b"10de", b"2330"
    d["numa_mask"] = np.left_shift(np.uint64(1), (i % 8).astype(np.uint64))
    d["iommu_group"] = 100000000 + i
    return d


def dra_pf_devices(n=1 << 16, vf_every=8, seed=41):
    """kxpu_dra_slices_pf's input: dra_devices(n), one in vf_every of them a VF that names its PF -- the function 0 of
    its bus, a 12-byte address -- and the PF's 4-digit device id; the others are no VF (both fields empty)"""
    from .binding import DRADEVPF_DTYPE
    d = np.zeros(n, DRADEVPF_DTYPE)
    d["dev"] = dra_devices(n, seed)
    vf = np.arange(n) % vf_every == 0
    pf = np.array([b"%04x:%02x:00.0" % (k >> 13, (k >> 5) & 0xff) for k in range(n)], "S16")
    d["physfn"] = np.where(vf, pf, b"")
    d["physfn_device"] = np.where(vf, b"2330", b"")
    return d


def dra_pcie_devices(n=1 << 16, vf_every=8, seed=41):
    """kxpu_dra_slices_pcie's input: dra_pf_devices(n, vf_every) with a root port on every device and a switch on three
    in four: 4-digit domains, 12-byte addresses"""
    from .binding import DRADEVPCIE_DTYPE, PCIE_NO_KEY
    d = np.zeros(n, DRADEVPCIE_DTYPE)
    d["pf"] = dra_pf_devices(n, vf_every, seed)
    k = np.arange(n, dtype=np.uint64)
    d["root_port"] = (k >> np.uint64(6) & np.uint64(0xff)) << np.uint64(8) | np.uint64(8)
    d["pcie_switch"] = np.where(k % 4 != 3, d["root_port"] + np.uint64(0x100), np.uint64(PCIE_NO_KEY))
    return d


def pcie_ports_walk(n=1 << 20, vf_every=8):
    """kxpu_pcie_ports' and kxpu_pcie_tree's input: n functions, one group each, two sockets of four root ports, a switch
    below each root port and 256 down ports below each switch; one in vf_every functions is a VF beside function 0 of
    its bus"""
    from .binding import DEVREC_DTYPE, PCIPATH_DTYPE
    recs = np.zeros(n, DEVREC_DTYPE)
    paths = np.zeros(n, PCIPATH_DTYPE)
    bdfs, ps = [], []
    for i in range(n):
        sock, rp, dp, fn = i >> 19 & 1, i >> 17 & 3, i >> 9 & 0xff, i & 0x1ff
        hb = 0x80 * sock
        bus = 0x10 + (dp & 0x3f)
        bdf = "%04x:%02x:%02x.%d" % (1 + (i >> 15), bus, fn >> 4 & 0x1f, (fn & 7) if i % vf_every == 0 else 0)
        bdfs.append(bdf.encode())
        ps.append(("pci0000:%02x/0000:%02x:%02x.0/0000:%02x:00.0/0000:%02x:%02x.0/%s" %
                   (hb, hb, 1 + rp, hb + 1 + rp, hb + 8, dp & 0x1f, bdf)).encode())
    recs["bdf"] = bdfs
    paths["path"] = ps
    paths["len"] = [len(p) for p in ps]
    return recs, paths, np.arange(n + 1, dtype=np.uint32), np.arange(n, dtype=np.uint32)


def pcie_ports_mdev_walk(n=1 << 20, vf_every=4, seed=23):
    """kxpu_pcie_ports_mdev's and kxpu_pcie_tree_mdev's input: pcie_mdev_walk(n) (parent GPUs below root ports and
    switches, one group per mdev), with the mdevs of one parent GPU in vf_every on a VF (function 4 beside the GPU, its
    link beside the PF's).  Returns (recs, paths, group_off, group_members)."""
    recs, paths, off, mem, _, _ = pcie_mdev_walk(n, seed)
    par = recs["parent"]
    vf = (np.char.str_len(par) > 0) & (np.frombuffer(par.tobytes(), np.uint8).reshape(n, 16)[:, 5] % vf_every == 0) \
        if n else np.zeros(0, bool)
    vfpar = np.char.replace(par, b":00.0", b":00.4")
    text = paths["path"]
    paths["path"] = np.where(vf, np.char.replace(text, np.char.add(par, b"/"), np.char.add(vfpar, b"/")), text)
    recs["parent"] = np.where(vf, vfpar, par)
    return recs, paths, off, mem


def aer_port_walk(n=1 << 20, depth=2, fanout=8, seed=53, mixed=False):
    """kxpu_aer_ports' input: n functions (DEVREC_DTYPE) below complete switch trees.  Each root port has a PCI domain of
    its own (pci<dom>:00, then <dom>:00:01.0) and `depth` switch levels below it (0..3: a chain of at most 8 keys), each
    switch an upstream port and `fanout` downstream ports (1..32), one function per downstream port of the last level,
    so fanout**depth functions share a root port.  mixed: record i's chain stops after 1 + i % (2 * depth + 2) keys (a
    function below the host bridge, the root port, a switch upstream or downstream port), at the same key counts for
    every seed.  seed: the order of the records (a permutation of the leaves).  Returns (recs, paths)."""
    from .binding import DEVREC_DTYPE, PCIPATH_DTYPE
    assert 0 <= depth <= 3 and 1 <= fanout <= 32
    rng = np.random.default_rng(seed)
    leaves = fanout ** depth
    first_bus = [1 + 2 * sum(fanout ** m for m in range(k)) for k in range(depth + 1)]  # level k's upstream buses
    recs = np.zeros(n, DEVREC_DTYPE)
    paths = np.zeros(n, PCIPATH_DTYPE)
    bdfs, texts = [], []
    for slot, i in enumerate(rng.permutation(n).tolist()):
        dom, leaf = i // leaves, i % leaves
        comps = ["pci%04x:00" % dom, "%04x:00:01.0" % dom]
        j = 0  # the switch's index within its level
        for k in range(depth):
            d = leaf // fanout ** (depth - 1 - k) % fanout
            up = first_bus[k] + 2 * j
            comps += ["%04x:%02x:00.0" % (dom, up), "%04x:%02x:%02x.0" % (dom, up + 1, d)]
            j = j * fanout + d
        if mixed:
            comps = comps[:1 + slot % (2 * depth + 2)]
        bdf = "%04x:%02x:00.0" % (dom, 0x80 + leaf % 0x80)
        bdfs.append(bdf.encode())
        texts.append(("/".join(comps) + "/" + bdf).encode())
    recs["bdf"] = bdfs
    paths["path"] = texts
    paths["len"] = [len(t) for t in texts]
    return recs, paths


def dra_mdev_pcie_devices(n=1 << 16, vf_every=8, seed=43):
    """kxpu_dra_slices_mdev_pcie's input: dra_mdev_devices(n), one in vf_every on a VF with its PF's address and device
    id, a root port on every device and a switch on three in four: 4-digit domains, 12-byte addresses"""
    from .binding import DRAMDEVPCIE_DTYPE, PCIE_NO_KEY
    d = np.zeros(n, DRAMDEVPCIE_DTYPE)
    d["pf"]["dev"] = dra_mdev_devices(n, seed)
    vf = np.arange(n) % vf_every == 0
    d["pf"]["physfn"] = np.where(vf, b"0000:41:00.0", b"")
    d["pf"]["physfn_device"] = np.where(vf, b"2330", b"")
    _ports(d, n, PCIE_NO_KEY)
    return d


def dra_vf_vgpu_pcie_devices(n=1 << 16, seed=47):
    """kxpu_dra_slices_vf_vgpu_pcie's input: dra_vf_vgpu_devices(n) with dra_mdev_pcie_devices' ports"""
    from .binding import DRAVFVGPUPCIE_DTYPE, PCIE_NO_KEY
    d = np.zeros(n, DRAVFVGPUPCIE_DTYPE)
    d["dev"] = dra_vf_vgpu_devices(n, seed)
    _ports(d, n, PCIE_NO_KEY)
    return d


def _ports(d, n, no_key):
    k = np.arange(n, dtype=np.uint64)
    d["root_port"] = (k >> np.uint64(6) & np.uint64(0xff)) << np.uint64(8) | np.uint64(8)
    d["pcie_switch"] = np.where(k % 4 != 3, d["root_port"] + np.uint64(0x100), np.uint64(no_key))


def dra_mdev_devices(n=1 << 16, seed=43):
    """n published vGPUs with every optional attribute present and the longest fields the host produces: a 64-byte
    product name, a 40-byte type key, a 12-byte parent address, a 10-byte PCIe root, 4-digit ids, one NUMA node, 9-digit
    groups"""
    from .binding import DRAMDEV_DTYPE
    rng = np.random.default_rng(seed)
    d = np.zeros(n, DRAMDEV_DTYPE)
    alnum = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_", np.uint8)
    d["product"] = alnum[rng.integers(0, len(alnum), (n, 64))]
    d["product_len"] = 64
    d["mdev_type"] = b"NVIDIA_H100XM-1-10C_with_a_long_type.key"
    i = np.arange(n)
    d["uuid"] = [b"%08x-%04x-4%03x-8%03x-%012x" % (k, k & 0xffff, k & 0xfff, (k >> 12) & 0xfff, (k * 2654435761) & (1 << 48) - 1)
                 for k in range(n)]
    par = i >> 4  # sixteen vGPUs per parent
    d["parent"] = [b"%04x:%02x:%02x.%d" % (k >> 13, (k >> 5) & 0xff, (k >> 3) & 0x1f, k & 7) for k in par.tolist()]
    d["pcie_root"] = [b"pci%04x:%02x" % (k >> 13, (k >> 5) & 0xff) for k in par.tolist()]
    d["vendor"], d["device"] = b"10de", b"2330"
    d["numa_mask"] = np.left_shift(np.uint64(1), (par % 8).astype(np.uint64))
    d["iommu_group"] = 100000000 + i
    return d


def dra_vf_vgpu_devices(n=1 << 16, seed=47):
    """n published vGPUs on SR-IOV VFs with every optional attribute present and the longest fields the host produces:
    a 64-byte product name, a 40-byte type key, 12-byte VF and PF addresses, a 10-byte PCIe root, 4-digit ids, a 4-digit
    type ID, one NUMA node, 9-digit groups"""
    from .binding import DRAVFVGPU_DTYPE
    rng = np.random.default_rng(seed)
    d = np.zeros(n, DRAVFVGPU_DTYPE)
    alnum = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_", np.uint8)
    d["product"] = alnum[rng.integers(0, len(alnum), (n, 64))]
    d["product_len"] = 64
    d["type_key"] = b"NVIDIA_H100XM-1-10C_with_a_long_type.key"
    d["type_id"] = 1058 + np.arange(n) % 4
    i = np.arange(n)
    par = i >> 4  # sixteen VFs per PF
    d["parent"] = [b"%04x:%02x:%02x.0" % (k >> 13, (k >> 5) & 0xff, k & 0x1f) for k in par.tolist()]
    d["bdf"] = [b"%04x:%02x:%02x.%d" % (k >> 17, (k >> 9) & 0xff, (k >> 4) & 0x1f, 1 + (k & 7) % 7) for k in i.tolist()]
    d["pcie_root"] = [b"pci%04x:%02x" % (k >> 13, (k >> 5) & 0xff) for k in par.tolist()]
    d["vendor"], d["device"] = b"10de", b"2330"
    d["numa_mask"] = np.left_shift(np.uint64(1), (par % 8).astype(np.uint64))
    d["iommu_group"] = 100000000 + i
    return d


AER_FATAL_NAMES = ["Undefined", "DLP", "SDES", "TLP", "FCP", "CmpltTO", "CmpltAbrt", "UnxCmplt", "RxOF", "MalfTLP",
                   "ECRC", "UnsupReq", "ACSViol", "UncorrIntErr", "BlockedTLP", "AtomicOpBlocked", "TLPBlockedErr",
                   "PoisonTLPBlocked"]


def aer_file(total_name, counts):
    """an aer_dev_fatal / aer_dev_nonfatal text as the kernel writes it: one "<name> <count>" line per error kind, then
    "<total_name> <sum>" (total_name TOTAL_ERR_FATAL or TOTAL_ERR_NONFATAL)"""
    lines = ["%s %d\n" % (nm, c) for nm, c in zip(AER_FATAL_NAMES, counts)]
    return ("".join(lines) + "%s %d\n" % (total_name, sum(counts))).encode()


def aer_records(n=1 << 20, seed=51, vgpus_per_parent=0):
    """kxpu_aer_health inputs for n records: dict(text, file_off, file_len, group_off, group_members).  Each physical
    function has its own pair of sysfs-format files, most with zero counts, about one in 64 with fatal or non-fatal
    errors; with vgpus_per_parent = k, runs of k records share their parent's two files, as vGPUs do.  The files are
    packed at odd offsets (each one follows a 1..7-byte gap), and the records are grouped one to four per group."""
    rng = np.random.default_rng(seed)
    share = max(1, vgpus_per_parent)
    n_fn = (n + share - 1) // share
    zero_f, zero_n = aer_file("TOTAL_ERR_FATAL", [0] * 18), aer_file("TOTAL_ERR_NONFATAL", [0] * 18)
    parts, off, pos = [], np.zeros(2 * n_fn, np.uint64), 0
    flen = np.zeros(2 * n_fn, np.uint32)
    bad = rng.integers(0, 64, n_fn) == 0
    for f in range(n_fn):
        for k, (name, zero) in enumerate((("TOTAL_ERR_FATAL", zero_f), ("TOTAL_ERR_NONFATAL", zero_n))):
            txt = zero
            if bad[f]:
                counts = [0] * 18
                counts[int(rng.integers(0, 18))] = int(rng.integers(1, 1000))
                txt = aer_file(name, counts)
            gap = int(rng.integers(1, 8))
            parts.append(b"\n" * gap)
            pos += gap
            off[2 * f + k], flen[2 * f + k] = pos, len(txt)
            parts.append(txt)
            pos += len(txt)
    fn_of = np.arange(n) // share
    file_off = np.empty(2 * n, np.uint64)
    file_len = np.empty(2 * n, np.uint32)
    file_off[0::2], file_off[1::2] = off[2 * fn_of], off[2 * fn_of + 1]
    file_len[0::2], file_len[1::2] = flen[2 * fn_of], flen[2 * fn_of + 1]
    sizes = rng.integers(1, 5, n)
    group_off = np.concatenate([[0], np.cumsum(sizes)])
    group_off = group_off[group_off <= n]
    if group_off[-1] != n:
        group_off = np.append(group_off, n)
    return dict(text=b"".join(parts), file_off=file_off, file_len=file_len, group_off=group_off.astype(np.uint32),
                group_members=rng.permutation(n).astype(np.uint32))


def sriov_walk(n=1 << 20, seed=41):
    """n records (DEVREC_DTYPE, bdfs in walk order, one group each) with their kxpu_sriovrec side records: function 0 of
    every device is a PF and functions 1..7 are its VFs (1 record in 8 a PF carrying 7 VFs).  PFs alternate between
    vfio-pci with sriov_numvfs "7\\n" and a host driver; VFs are on vfio-pci and name their PF; 1 in 64 physfn reads
    failed.  Returns (recs, srs)."""
    from .binding import SR_PHYSFN_ERR, SRIOVREC_DTYPE
    rng = np.random.default_rng(seed)
    i = np.arange(n, dtype=np.int64)
    is_pf = (i & 7) == 0
    vfio_pf = ((i >> 3) & 1) == 0
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    recs["bdf"] = enumerate_bdfs(n).view("S16").reshape(n)
    recs["driver"] = np.where(is_pf & ~vfio_pf, b"nvidia", b"vfio-pci")
    recs["vendor_txt"] = _id_text(np.full(n, 0x10DE))
    recs["device_txt"] = _id_text(np.full(n, 0x2330))
    recs["vendor_len"] = recs["device_len"] = 7
    recs["iommu_group"] = i + 1
    srs = np.zeros(n, dtype=SRIOVREC_DTYPE)
    srs["physfn"] = np.where(is_pf, b"", recs["bdf"][i & ~7])
    srs["numvfs_txt"][is_pf & vfio_pf, :2] = np.frombuffer(b"7\n", np.uint8)
    srs["numvfs_len"] = np.where(is_pf & vfio_pf, 2, 0)
    srs["flags"] = np.where(rng.integers(0, 64, n) == 0, SR_PHYSFN_ERR, 0)
    return recs, srs



def mdev_pf_walk(n_recs=1 << 20, n_pfs=1 << 15, n_mdevs=1 << 20, seed=91):
    """kxpu_mdev_pf's input at scale: a PCI walk of n_recs records (DEVREC_DTYPE, canonical bdfs in walk order) in which
    record k * (n_recs // n_pfs) is the PF of card k < n_pfs and the records after it are its VFs, and n_mdevs mdevs
    (MDEVREC_DTYPE, parent only) with their side records (SRIOVREC_DTYPE, physfn only).  An mdev sits on a random VF and
    names that VF's PF, except: 1 in 16 sits on a PF (no physfn), and 1 in 16 has a link that cannot resolve -- a
    non-canonical address, a failed read, a PF outside the walk, or a link to its own parent, in turn.  Returns (recs, mrecs,
    msrs, want), want being the pf_of the header's rules give."""
    from .binding import MDEVREC_DTYPE, NO_PF, SR_PHYSFN_ERR, SRIOVREC_DTYPE
    rng = np.random.default_rng(seed)
    per = n_recs // n_pfs
    recs = np.zeros(n_recs, dtype=DEVREC_DTYPE)
    bdf = enumerate_bdfs(n_recs).view("S16").reshape(n_recs)
    recs["bdf"] = bdf
    recs["driver"] = b"nvidia"
    recs["vendor_txt"] = _id_text(np.full(n_recs, 0x10DE))
    recs["device_txt"] = _id_text(np.full(n_recs, 0x2330))
    recs["vendor_len"] = recs["device_len"] = 7
    recs["iommu_group"] = np.arange(n_recs) + 1
    card = rng.integers(0, n_pfs, n_mdevs)
    pf = card * per
    vf = pf + rng.integers(1, per, n_mdevs)
    kind = rng.integers(0, 64, n_mdevs)  # 0..3: an unresolvable link; 4..7: an mdev on a PF; else on a VF
    on_pf = (kind >= 4) & (kind < 8)
    mrecs = np.zeros(n_mdevs, dtype=MDEVREC_DTYPE)
    mrecs["uuid"] = uuids(n_mdevs, seed).view("S36").reshape(n_mdevs)
    mrecs["parent"] = np.where(on_pf, bdf[pf], bdf[vf])
    msrs = np.zeros(n_mdevs, dtype=SRIOVREC_DTYPE)
    msrs["physfn"] = np.where(on_pf, b"", bdf[pf])
    msrs["physfn"] = np.where(kind == 0, np.char.replace(bdf[pf], b":", b"-"), msrs["physfn"])
    msrs["flags"] = np.where(kind == 1, SR_PHYSFN_ERR, 0)
    msrs["physfn"] = np.where(kind == 2, b"ffff:ff:1f.7", msrs["physfn"])
    msrs["physfn"] = np.where(kind == 3, mrecs["parent"], msrs["physfn"])
    want = np.where(kind >= 8, pf, NO_PF).astype(np.uint32)
    return recs, mrecs, msrs, want

# An H100 80GB vGPU type table: (type ID, name).  The IDs are synthetic; the names follow NVIDIA's time-sliced and
# MIG-backed C-series profiles.
H100_VGPU_TYPES = [(1000 + k, n) for k, n in enumerate(
    ["NVIDIA H100-1-10C", "NVIDIA H100-1-20C", "NVIDIA H100-2-20C", "NVIDIA H100-3-40C", "NVIDIA H100-4-40C",
     "NVIDIA H100-7-80C", "NVIDIA H100-4C", "NVIDIA H100-5C", "NVIDIA H100-8C", "NVIDIA H100-10C", "NVIDIA H100-16C",
     "NVIDIA H100-20C", "NVIDIA H100-40C", "NVIDIA H100-80C"])]


def vf_vgpu_walk(n=1 << 20, seed=61):
    """n records (DEVREC_DTYPE, bdfs in walk order, one group each) of GPUs on the vGPU manager's driver "nvidia": record
    32k is a PF, records 32k+1 .. 32k+31 its VFs.  Of the VFs, 1 in 4 is free (type 0) and lists the H100 type table in
    creatable_vgpu_types; the others carry a type: mostly one of the table's, 1 in 64 an ID no table names, 1 in 128 a
    text that does not parse.  Returns (recs, vts, tables): the side records (the PFs are not read) and one table per free
    VF in walk order."""
    from .binding import VFVGPUREC_DTYPE, VT_READ
    rng = np.random.default_rng(seed)
    i = np.arange(n, dtype=np.int64)
    is_pf = (i & 31) == 0
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    recs["bdf"] = enumerate_bdfs(n).view("S16").reshape(n)
    recs["driver"] = b"nvidia"
    recs["vendor_txt"] = _id_text(np.full(n, 0x10DE))
    recs["device_txt"] = _id_text(np.where(is_pf, 0x2330, 0x2331))
    recs["vendor_len"] = recs["device_len"] = 7
    recs["iommu_group"] = i + 1
    ids = np.array([t for t, _ in H100_VGPU_TYPES])
    kind = rng.integers(0, 512, n)
    cur = np.where(kind < 128, 0, ids[rng.integers(0, len(ids), n)])
    cur = np.where((kind >= 128) & (kind < 136), 4242, cur)  # unnamed
    texts = [b"%d\n" % c for c in cur]
    bad = (kind >= 136) & (kind < 140)
    vts = np.zeros(n, dtype=VFVGPUREC_DTYPE)
    flat = np.zeros((n, 16), np.uint8)
    lens = np.zeros(n, np.uint8)
    for k in np.nonzero(~is_pf)[0]:
        t = b"x\n" if bad[k] else texts[k]
        flat[k, :len(t)] = np.frombuffer(t, np.uint8)
        lens[k] = len(t)
    vts["cur_txt"], vts["cur_len"] = flat, lens
    vts["flags"] = np.where(is_pf, 0, VT_READ)
    table = b"ID    : vGPU Name\n" + b"".join(b"%d : %s\n" % (t, nm.encode()) for t, nm in H100_VGPU_TYPES)
    tables = [table] * int(((cur == 0) & ~is_pf & ~bad).sum())
    return recs, vts, tables


def vf_vgpu_cdi_devices(n=1 << 20, seed=63):
    """n served VFs (VFVGPUCDI_DTYPE) for the typed CDI layouts: cfg5_devices' bdfs, groups and indices, cdev numbers of
    every width, and a type of the H100 table with its type key (keys of 12 to 19 bytes, IDs of four digits)."""
    from .binding import VFVGPUCDI_DTYPE
    rng = np.random.default_rng(seed)
    devs = np.zeros(n, dtype=VFVGPUCDI_DTYPE)
    devs["dev"] = cfg5_devices(n)
    devs["dev"]["reserved"] = (np.arange(n, dtype=np.uint64) * 2654435761) % (1 << 32)  # the cdev number
    pick = rng.integers(0, len(H100_VGPU_TYPES), n)
    keys = np.array([nm.replace(" ", "_").encode() for _, nm in H100_VGPU_TYPES])
    devs["type_id"] = np.array([t for t, _ in H100_VGPU_TYPES], np.uint32)[pick]
    devs["key"] = keys[pick]
    devs["key_len"] = np.array([len(k) for k in keys], np.uint8)[pick]
    return devs


def reset_walk(n=1 << 20, seed=71):
    """n records (DEVREC_DTYPE, bdfs in walk order, one group each) with their kxpu_pcipath and kxpu_resetrec side
    records, on pcie_walk's board (8 functions per down port; 2 % of the buses behind a VMD domain, 1 % with chains of
    exactly 8, 1 % of 9 (unknown)).  reset_method: 70 % "flr bus\\n", 15 % "bus\\n", 2 % "pm\\n", 1 % a kernel without
    reset_method but with reset, 12 % neither file (no method: withheld, since a down port's eight functions lie in eight
    groups).  Returns (recs, paths, rrs)."""
    from .binding import PCIPATH_DTYPE, RESETREC_DTYPE, RS_ABSENT, RS_LEGACY
    rng = np.random.default_rng(seed)
    recs = np.zeros(n, dtype=DEVREC_DTYPE)
    bdfs = enumerate_bdfs(n)
    recs["bdf"] = bdfs.view("S16").reshape(n)
    recs["driver"] = b"vfio-pci"
    recs["vendor_txt"] = _id_text(np.full(n, 0x10DE))
    recs["device_txt"] = _id_text(np.full(n, 0x2330))
    recs["vendor_len"] = recs["device_len"] = 7
    recs["iommu_group"] = np.arange(1, n + 1, dtype=np.uint32)
    i = np.arange(n, dtype=np.int64)
    dom, bus, dev = i >> 16, (i >> 8) & 255, (i >> 3) & 31
    bus_kind = rng.choice(4, size=int((n + 255) >> 8), p=[0.96, 0.02, 0.01, 0.01])
    prefix = {}
    texts = []
    for k in range(n):
        pre = prefix.get(k >> 3)
        if pre is None:
            pre = prefix[k >> 3] = _pcie_prefix(int(dom[k]), int(bus[k]), int(dev[k]), int(bus_kind[k >> 8])).encode()
        texts.append(pre + bytes(bdfs[k][:12]))
    paths = np.zeros(n, dtype=PCIPATH_DTYPE)
    paths["path"] = np.array(texts, dtype="S120")
    paths["len"] = np.array([len(t) for t in texts], np.uint8)
    rrs = np.zeros(n, dtype=RESETREC_DTYPE)
    kind = rng.choice(5, size=n, p=[0.70, 0.15, 0.02, 0.01, 0.12])
    for k, text in enumerate((b"flr bus\n", b"bus\n", b"pm\n")):
        rows = kind == k
        rrs["txt"][rows, :len(text)] = np.frombuffer(text, np.uint8)
        rrs["len"][rows] = len(text)
    rrs["flags"][kind == 3] = RS_ABSENT | RS_LEGACY
    rrs["flags"][kind == 4] = RS_ABSENT
    return recs, paths, rrs


def metrics_devices(n=1 << 20, seed=81):
    """n devices of kxpu_metrics_devices (METRICDEV_DTYPE), their strings and reasons (METRICREASON_DTYPE): eight
    resources, one bdf per device, 1 in 8 devices with one reason, 1 in 64 with three, details of about 80 bytes of
    which 1 in 256 carries a non-ASCII or escaped byte, every device with both AER values.  Returns (devs, strings,
    reasons)."""
    from .binding import METRICDEV_DTYPE, METRICREASON_DTYPE
    rng = np.random.default_rng(seed)
    resources = [b"nvidia.com/GH100_H100_SXM5_80GB", b"nvidia.com/GH100_H100_NVL", b"amd.com/MI300X",
                 b"nvidia.com/NVIDIA_H100-4C", b"nvidia.com/NVIDIA_H100-10C", b"nvidia.com/NVIDIA_H100-20C",
                 b"nvidia.com/GA100_A100_PCIE_80GB", b"intel.com/Gaudi3"]
    parts = [b"".join(resources)]
    roff = np.cumsum([0] + [len(r) for r in resources])[:-1]
    base = len(parts[0])
    bdfs = enumerate_bdfs(n)
    parts.append(bdfs[:, :12].tobytes())
    devs = np.zeros(n, METRICDEV_DTYPE)
    which = rng.integers(0, len(resources), n)
    devs["resource_off"] = roff[which]
    devs["resource_len"] = np.array([len(r) for r in resources], np.uint32)[which]
    devs["address_off"] = base + 12 * np.arange(n, dtype=np.uint64)
    devs["address_len"] = 12
    devs["group"] = rng.permutation(n).astype(np.uint32) + 1
    devs["aer_fatal"] = rng.integers(0, 3, n)
    devs["aer_nonfatal"] = rng.integers(0, 1000, n)
    count = np.zeros(n, np.uint32)
    count[rng.random(n) < 1 / 8] = 1
    count[rng.random(n) < 1 / 64] = 3
    devs["reason_count"] = count
    devs["reason_off"] = np.concatenate([[0], np.cumsum(count)[:-1]])
    devs["healthy"] = count == 0
    m = int(count.sum())
    reasons = np.zeros(m, METRICREASON_DTYPE)
    first = np.repeat(rng.integers(1, 5, n).astype(np.uint32), count)  # a kind, then kind + 1, kind + 2 for three
    step = np.arange(m) - np.repeat(devs["reason_off"].astype(np.int64), count)
    reasons["kind"] = np.minimum(first, 4) + step
    texts = (b"0000:%02x:00.1 on its bus is bound to snd_hda_intel and cannot be reset between tenants%s" % (k, t)
             for k, t in enumerate([b"", b" \xe2\x80\x94 \"x\"", b"\\n", b"\xff"] * 64))
    pool = list(texts)
    pick = np.where(rng.random(m) < 1 / 256, rng.integers(0, len(pool), m), (rng.integers(0, len(pool) // 4, m) * 4))
    off = base + 12 * n
    pool_off = np.cumsum([0] + [len(t) for t in pool])[:-1] + off
    parts.append(b"".join(pool))
    reasons["detail_off"] = pool_off[pick]
    reasons["detail_len"] = np.array([len(t) for t in pool], np.uint32)[pick]
    return devs, b"".join(parts), reasons
