"""Synthetic inputs for BASELINE.json configs[0..4] (SURVEY.md 8(d)).  Pure numpy, seeded;
shared by tests/ and bench.py.  Nothing here is on the product path."""
import gzip
import os

import numpy as np

from .binding import CDIDEV_DTYPE, DEVREC_DTYPE, REC_DRIVER_ERR

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
