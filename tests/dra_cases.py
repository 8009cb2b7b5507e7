"""Records for the DRA ResourceSlice tests (kxpu_dra_slices, ABI v9): a record builder, the cfg1 device and a seeded
generator that mixes every optional attribute inside one slice."""
import numpy as np

from oracle.dra_oracle import DRADEV_DTYPE

CFG1 = dict(driver="vfio.nvidia.com", pool="node-a", node="node-a", gen=1)


def rec(group=214, bdf=b"0000:c1:00.0", vendor=b"10de", device=b"2330", product=b"GH100_H100_SXM5_80GB",
        root=b"pci0000:c0", numa=1 << 1, product_len=None):
    r = np.zeros(1, DRADEV_DTYPE)
    r["product"][0, :len(product)] = np.frombuffer(product, np.uint8)
    r["product_len"] = len(product) if product_len is None else product_len
    r["bdf"], r["pcie_root"], r["vendor"], r["device"] = bdf, root, vendor, device
    r["numa_mask"], r["iommu_group"] = numa, group
    return r


def cfg1():
    return rec()


_PCHARS = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_.-", np.uint8)
_HEX = np.frombuffer(b"0123456789abcdef", np.uint8)


def random_devs(n, seed, all_attrs=False):
    """n in-domain records: product lengths 0..64, NUMA masks 0 / one bit / two bits, roots present or not, ids of
    1..6 hex digits, groups over the whole range (all_attrs: every optional attribute present, longest fields)"""
    rng = np.random.default_rng(seed)
    d = np.zeros(n, DRADEV_DTYPE)
    if n == 0:
        return d
    pl = np.full(n, 64) if all_attrs else rng.choice([0, 1, 20, 63, 64], n)
    prod = _PCHARS[rng.integers(0, len(_PCHARS), (n, 64))]
    prod[np.arange(64)[None, :] >= pl[:, None]] = 0
    d["product"], d["product_len"] = prod, pl
    d["iommu_group"] = rng.choice([0, 1, 9, 10, 214, 99999, 4294967294], n) if not all_attrs else 4294967294 - np.arange(n) % 7
    bits = rng.integers(0, 64, n).astype(np.uint64)
    one = np.left_shift(np.uint64(1), bits)
    kind = np.zeros(n, np.int64) if all_attrs else rng.integers(0, 3, n)
    d["numa_mask"] = np.where(kind == 0, one, np.where(kind == 1, np.uint64(0), one | np.uint64(1) << ((bits + 1) % 64)))
    for f, w in (("bdf", 16), ("pcie_root", 16), ("vendor", 8), ("device", 8)):
        a = np.zeros((n, w), np.uint8)
        if f == "bdf":
            ln = np.full(n, 16) if all_attrs else rng.integers(1, 17, n)
            a[:] = np.frombuffer(b"0123456789abcdef:."[:18], np.uint8)[rng.integers(0, 18, (n, w))]
        elif f == "pcie_root":
            ln = np.full(n, 16) if all_attrs else rng.choice([0, 4, 10, 16], n)
            a[:] = np.frombuffer(b"0123456789abcdef:", np.uint8)[rng.integers(0, 17, (n, w))]
            a[:, :3] = np.frombuffer(b"pci", np.uint8)
        else:
            ln = np.full(n, 6) if all_attrs else rng.integers(1, 7, n)
            a[:] = _HEX[rng.integers(0, 16, (n, w))]
        a[np.arange(w)[None, :] >= ln[:, None]] = 0
        d[f] = a.view("S%d" % w).reshape(n)
    return d


# one field per out-of-domain case: (name of the rule, field, value)
BAD = [
    ("product", "product", b"GH100 H100"),
    ("product", "product", b"A\"B"),
    ("bdf", "bdf", b""),
    ("bdf", "bdf", b"0000:C1:00.0"),
    ("bdf", "bdf", b"0000:c1:00.0\\"),
    ("pcie_root", "pcie_root", b"pci"),
    ("pcie_root", "pcie_root", b"pcz0000:c0"),
    ("pcie_root", "pcie_root", b"pci0000:C0"),
    ("pcie_root", "pcie_root", b"pci0000.c0"),
    ("vendor", "vendor", b""),
    ("vendor", "vendor", b"10DE"),
    ("vendor", "vendor", b"1234567"),
    ("device", "device", b"233g"),
    ("device", "device", b"12345678"),
    ("iommu_group", "iommu_group", 0xFFFFFFFF),
    ("product_len", "product_len", 65),
]


def bad_rec(field, value):
    r = rec()
    if field == "product":
        r["product"][0] = 0
        r["product"][0, :len(value)] = np.frombuffer(value, np.uint8)
        r["product_len"] = len(value)
    else:
        r[field] = value
    return r
