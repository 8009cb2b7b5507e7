"""Records for the tests of passthrough SR-IOV VFs in DRA (kxpu_dra_slices_pf, an addition to ABI v14): the slice record
built on kxpu_dra_slices' record, the cfg1 pair (a VF of an Intel Data Center GPU Flex 170 and an H100 that is no VF), a
seeded generator that mixes every optional attribute, and the out-of-domain cases."""
import numpy as np

import dra_cases as DC
import dra_mdev_cases as MC
from kxpu_b200.binding import DRADEVPF_DTYPE  # noqa: F401

CFG1 = dict(driver="vfio.example.com", pool="node-a", node="node-a", gen=1)
TAINTS1 = [("vfio.example.com/unhealthy", "vfio-device-missing", "NoSchedule")]
TAINTS3 = TAINTS1 + [("vfio.example.com/pcie-aer", "fatal", "NoSchedule"),
                     ("vfio.example.com/pcie-aer", "nonfatal", "NoSchedule")]


def rec(physfn=b"", physfn_device=b"", **kw):
    r = np.zeros(1, DRADEVPF_DTYPE)
    r["dev"] = DC.rec(**kw)
    r["physfn"], r["physfn_device"] = physfn, physfn_device
    return r


def cfg1():
    """VF 0000:4d:00.1 of the Flex 170 PF 0000:4d:00.0, and the H100 0000:c1:00.0, which is no VF"""
    return np.concatenate([
        rec(group=45, bdf=b"0000:4d:00.1", vendor=b"8086", device=b"56c0", product=b"Data_Center_GPU_Flex_170",
            root=b"pci0000:4a", numa=1 << 0, physfn=b"0000:4d:00.0", physfn_device=b"56c0"),
        rec()])


def random_devs(n, seed, all_attrs=False, no_physfn=False, vf_every=None):
    """n in-domain records: kxpu_dra_slices' generator, then physfn present (16, 12 or 1 bytes) or not and physfn_device
    0..6 bytes where physfn is present (all_attrs: both at their longest; no_physfn: both empty; vf_every = k: a
    canonical 12-byte physfn and a 4-digit id on every k-th record only, as a pool of mostly whole GPUs has them)"""
    rng = np.random.default_rng(seed + 7)
    d = np.zeros(n, DRADEVPF_DTYPE)
    if n == 0:
        return d
    d["dev"] = DC.random_devs(n, seed, all_attrs)
    if no_physfn:
        return d
    if vf_every:
        vf = np.arange(n) % vf_every == 0
        d["physfn"] = np.where(vf, b"0000:4d:00.0", b"")
        d["physfn_device"] = np.where(vf, b"56c0", b"")
        return d
    addr = np.frombuffer(b"0123456789abcdef:.", np.uint8)
    xl = np.full(n, 16) if all_attrs else rng.choice([0, 1, 12, 16], n)
    yl = np.full(n, 6) if all_attrs else np.where(xl > 0, rng.choice([0, 1, 4, 6], n), 0)
    d["physfn"] = MC._text(rng, n, 16, addr, xl).view("S16").reshape(n)
    d["physfn_device"] = MC._text(rng, n, 8, DC._HEX, yl).view("S8").reshape(n)
    return d


# one field per out-of-domain case of the two new fields: (name of the rule, field, value)
BAD = [
    ("physfn", "physfn", b"0000:4d:00.0/"),
    ("physfn", "physfn", b"0000:4D:00.0"),
    ("physfn", "physfn", b"0000 4d:00.0"),
    ("physfn_device", "physfn_device", b"56C0"),
    ("physfn_device", "physfn_device", b"1234567"),
]


def bad_rec(field, value, physfn=b"0000:4d:00.0"):
    r = rec(physfn=physfn)
    r[field] = value
    return r
