"""Records for the vGPU DRA ResourceSlice tests (kxpu_dra_slices_mdev, ABI v10): a record builder, the cfg1 vGPU, a
seeded generator that mixes every optional attribute inside one slice, and the out-of-domain cases."""
import numpy as np

from oracle.dra_mdev_oracle import DRAMDEV_DTYPE

CFG1 = dict(driver="vgpu.nvidia.com", pool="node-a", node="node-a", gen=1)
UUID = b"4b20d080-1b54-4048-85b3-a6a62d165c01"


def rec(group=300, mdev_type=b"NVIDIA_H100XM-1-10C", uuid=UUID, parent=b"0000:c1:00.0", root=b"pci0000:c0",
        vendor=b"10de", device=b"2330", product=b"GH100_H100_SXM5_80GB", numa=1 << 1, product_len=None):
    r = np.zeros(1, DRAMDEV_DTYPE)
    r["product"][0, :len(product)] = np.frombuffer(product, np.uint8)
    r["product_len"] = len(product) if product_len is None else product_len
    r["mdev_type"], r["uuid"], r["parent"], r["pcie_root"] = mdev_type, uuid, parent, root
    r["vendor"], r["device"], r["numa_mask"], r["iommu_group"] = vendor, device, numa, group
    return r


def cfg1():
    return rec()


_PCHARS = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_.-", np.uint8)
_HEX = np.frombuffer(b"0123456789abcdef", np.uint8)


def _text(rng, n, width, alphabet, lens):
    a = alphabet[rng.integers(0, len(alphabet), (n, width))]
    a[np.arange(width)[None, :] >= lens[:, None]] = 0
    return a


def random_devs(n, seed, all_attrs=False):
    """n in-domain records: product lengths 0..64, type keys of 1..40 bytes, NUMA masks 0 / one bit / two bits, roots
    and device ids present or not, groups over the whole range (all_attrs: every optional attribute present, longest
    fields)"""
    rng = np.random.default_rng(seed)
    d = np.zeros(n, DRAMDEV_DTYPE)
    if n == 0:
        return d
    pick = (lambda full, choices: np.full(n, full)) if all_attrs else (lambda full, choices: rng.choice(choices, n))
    pl = pick(64, [0, 1, 20, 63, 64])
    d["product"], d["product_len"] = _text(rng, n, 64, _PCHARS, pl), pl
    d["mdev_type"] = _text(rng, n, 40, _PCHARS, pick(40, [1, 5, 19, 39, 40])).view("S40").reshape(n)
    u = _HEX[rng.integers(0, 16, (n, 36))]
    u[:, [8, 13, 18, 23]] = ord("-")
    d["uuid"] = u.view("S36").reshape(n)
    d["parent"] = _text(rng, n, 16, np.frombuffer(b"0123456789abcdef:.", np.uint8), pick(16, [1, 7, 12, 16])).view("S16").reshape(n)
    root = _text(rng, n, 16, np.frombuffer(b"0123456789abcdef:", np.uint8), pick(16, [0, 4, 10, 16]))
    root[:, :3] = np.where(root[:, 3:4] != 0, np.frombuffer(b"pci", np.uint8)[None, :], 0)
    d["pcie_root"] = root.view("S16").reshape(n)
    d["vendor"] = _text(rng, n, 8, _HEX, pick(6, [1, 4, 6])).view("S8").reshape(n)
    d["device"] = _text(rng, n, 8, _HEX, pick(6, [0, 1, 4, 6])).view("S8").reshape(n)
    d["iommu_group"] = 4294967294 - np.arange(n) % 7 if all_attrs else rng.choice([0, 1, 9, 10, 214, 99999, 4294967294], n)
    bits = rng.integers(0, 64, n).astype(np.uint64)
    one = np.left_shift(np.uint64(1), bits)
    kind = np.zeros(n, np.int64) if all_attrs else rng.integers(0, 3, n)
    d["numa_mask"] = np.where(kind == 0, one, np.where(kind == 1, np.uint64(0), one | np.uint64(1) << ((bits + 1) % 64)))
    return d


# one field per out-of-domain case: (name of the rule, field, value)
BAD = [
    ("product", "product", b"GH100 H100"),
    ("product", "product", b"A\"B"),
    ("mdev_type", "mdev_type", b""),
    ("mdev_type", "mdev_type", b"GRID T4-1Q"),
    ("mdev_type", "mdev_type", b"nvidia/222"),
    ("uuid", "uuid", b""),
    ("uuid", "uuid", b"4B20D080-1B54-4048-85B3-A6A62D165C01"),
    ("uuid", "uuid", b"4b20d080-1b54-4048-85b3-a6a62d165c0"),
    ("uuid", "uuid", b"4b20d0801-b54-4048-85b3-a6a62d165c01"),
    ("parent", "parent", b""),
    ("parent", "parent", b"0000:C1:00.0"),
    ("pcie_root", "pcie_root", b"pci"),
    ("pcie_root", "pcie_root", b"pcz0000:c0"),
    ("pcie_root", "pcie_root", b"pci0000.c0"),
    ("vendor", "vendor", b""),
    ("vendor", "vendor", b"10DE"),
    ("vendor", "vendor", b"1234567"),
    ("device", "device", b"233g"),
    ("device", "device", b"1234567"),
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
