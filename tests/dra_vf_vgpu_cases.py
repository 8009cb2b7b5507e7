"""Records for the VF-vGPU DRA ResourceSlice tests (kxpu_dra_slices_vf_vgpu): a record builder, the cfg1 vGPU (one VF of
an H100 SXM PF), a seeded generator that mixes every optional attribute inside one slice, the out-of-domain cases and
the taint tables the host publishes."""
import numpy as np

from kxpu_b200.binding import DRAVFVGPU_DTYPE

CFG1 = dict(driver="vgpu-vf.nvidia.com", pool="node-a", node="node-a", gen=1)
# the host's tables: <driver>/unhealthy alone, or with the two AER entries
TAINTS1 = [("vgpu-vf.nvidia.com/unhealthy", "vfio-device-missing", "NoSchedule")]
TAINTS3 = TAINTS1 + [("vgpu-vf.nvidia.com/pcie-aer", "fatal", "NoSchedule"),
                     ("vgpu-vf.nvidia.com/pcie-aer", "nonfatal", "NoSchedule")]


def rec(group=301, type_key=b"NVIDIA_H100XM-1-10C", type_id=1058, bdf=b"0000:c1:00.4", parent=b"0000:c1:00.0",
        root=b"pci0000:c0", vendor=b"10de", device=b"2330", product=b"GH100_H100_SXM5_80GB", numa=1 << 1, product_len=None):
    r = np.zeros(1, DRAVFVGPU_DTYPE)
    r["product"][0, :len(product)] = np.frombuffer(product, np.uint8)
    r["product_len"] = len(product) if product_len is None else product_len
    r["type_key"], r["type_id"], r["bdf"], r["parent"], r["pcie_root"] = type_key, type_id, bdf, parent, root
    r["vendor"], r["device"], r["numa_mask"], r["iommu_group"] = vendor, device, numa, group
    return r


def cfg1():
    return rec()


_PCHARS = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_.-", np.uint8)
_HEX = np.frombuffer(b"0123456789abcdef", np.uint8)
_ADDR = np.frombuffer(b"0123456789abcdef:.", np.uint8)


def _text(rng, n, width, alphabet, lens):
    a = alphabet[rng.integers(0, len(alphabet), (n, width))]
    a[np.arange(width)[None, :] >= lens[:, None]] = 0
    return a


def random_devs(n, seed, all_attrs=False):
    """n in-domain records: product lengths 0..64, type keys of 1..40 bytes, type IDs over the whole range, NUMA masks
    0 / one bit / two bits, roots and device ids present or not, groups over the whole range (all_attrs: every optional
    attribute present, longest fields)"""
    rng = np.random.default_rng(seed)
    d = np.zeros(n, DRAVFVGPU_DTYPE)
    if n == 0:
        return d
    pick = (lambda full, choices: np.full(n, full)) if all_attrs else (lambda full, choices: rng.choice(choices, n))
    pl = pick(64, [0, 1, 20, 63, 64])
    d["product"], d["product_len"] = _text(rng, n, 64, _PCHARS, pl), pl
    d["type_key"] = _text(rng, n, 40, _PCHARS, pick(40, [1, 5, 19, 39, 40])).view("S40").reshape(n)
    d["bdf"] = _text(rng, n, 16, _ADDR, pick(16, [1, 7, 12, 16])).view("S16").reshape(n)
    d["parent"] = _text(rng, n, 16, _ADDR, pick(16, [1, 7, 12, 16])).view("S16").reshape(n)
    root = _text(rng, n, 16, np.frombuffer(b"0123456789abcdef:", np.uint8), pick(16, [0, 4, 10, 16]))
    root[:, :3] = np.where(root[:, 3:4] != 0, np.frombuffer(b"pci", np.uint8)[None, :], 0)
    d["pcie_root"] = root.view("S16").reshape(n)
    d["vendor"] = _text(rng, n, 8, _HEX, pick(6, [1, 4, 6])).view("S8").reshape(n)
    d["device"] = _text(rng, n, 8, _HEX, pick(6, [0, 1, 4, 6])).view("S8").reshape(n)
    d["iommu_group"] = 4294967294 - np.arange(n) % 7 if all_attrs else rng.choice([0, 1, 9, 10, 214, 99999, 4294967294], n)
    d["type_id"] = 4294967295 - np.arange(n) % 5 if all_attrs else rng.choice([1, 9, 10, 557, 99999, 4294967295], n)
    bits = rng.integers(0, 64, n).astype(np.uint64)
    one = np.left_shift(np.uint64(1), bits)
    kind = np.zeros(n, np.int64) if all_attrs else rng.integers(0, 3, n)
    d["numa_mask"] = np.where(kind == 0, one, np.where(kind == 1, np.uint64(0), one | np.uint64(1) << ((bits + 1) % 64)))
    return d


# one field per out-of-domain case: (name of the rule, field, value)
BAD = [
    ("product", "product", b"GH100 H100"),
    ("product", "product", b"A\"B"),
    ("type_key", "type_key", b""),
    ("type_key", "type_key", b"NVIDIA H100-4C"),
    ("type_key", "type_key", b"nvidia/557"),
    ("bdf", "bdf", b""),
    ("bdf", "bdf", b"0000:C1:00.4"),
    ("bdf", "bdf", b"0000_c1:00.4"),
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
    ("type_id", "type_id", 0),
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
