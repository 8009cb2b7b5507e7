"""Records for the tests of mdev vGPUs on SR-IOV VFs (kxpu_mdev_pf and kxpu_dra_slices_mdev_pf, additions to ABI v14):
builders for the join's PCI records, mdev records and side records, the slice record built on the mdev layout's, the
cfg1 pair (an mdev on a VF of a 0000:41:00.0 H100 and an mdev on a PF), a seeded generator that mixes every optional
attribute, and the out-of-domain cases."""
import numpy as np

import dra_mdev_cases as MC
from kxpu_b200.binding import (DEVREC_DTYPE, DRAMDEVPF_DTYPE, MDEVREC_DTYPE, NO_PF, SR_PHYSFN_ERR,  # noqa: F401
                               SRIOVREC_DTYPE)

CFG1 = dict(driver="vgpu.nvidia.com", pool="node-a", node="node-a", gen=1)
TAINTS1 = [("vgpu.nvidia.com/unhealthy", "vfio-device-missing", "NoSchedule")]
TAINTS3 = TAINTS1 + [("vgpu.nvidia.com/pcie-aer", "fatal", "NoSchedule"),
                     ("vgpu.nvidia.com/pcie-aer", "nonfatal", "NoSchedule")]
U = [b"4b20d080-1b54-4048-85b3-a6a62d16%04x" % k for k in range(64)]


def walk(bdfs):
    """PCI records with these addresses (bytes), one group each"""
    r = np.zeros(len(bdfs), DEVREC_DTYPE)
    r["bdf"] = bdfs
    r["iommu_group"] = np.arange(len(bdfs)) + 1
    return r


def mdevs(pairs):
    """(mdev records, side records) from (parent, physfn, flags) triples"""
    m = np.zeros(len(pairs), MDEVREC_DTYPE)
    s = np.zeros(len(pairs), SRIOVREC_DTYPE)
    for i, (parent, physfn, flags) in enumerate(pairs):
        m[i]["uuid"], m[i]["parent"] = U[i % len(U)], parent
        s[i]["physfn"], s[i]["flags"] = physfn, flags
    return m, s


def rec(physfn=b"", physfn_device=b"", **kw):
    r = np.zeros(1, DRAMDEVPF_DTYPE)
    r["dev"] = MC.rec(**kw)
    r["physfn"], r["physfn_device"] = physfn, physfn_device
    return r


def cfg1():
    """an mdev on VF 0000:41:00.4 of the H100 0000:41:00.0 (the VF's device id not read, the PF's model as productName),
    and an mdev on the PF 0000:c1:00.0 of another H100"""
    return np.concatenate([
        rec(group=300, uuid=U[1], parent=b"0000:41:00.4", root=b"pci0000:40", device=b"", numa=1 << 0,
            physfn=b"0000:41:00.0", physfn_device=b"2330"),
        rec(group=301, uuid=U[2], parent=b"0000:c1:00.0", root=b"pci0000:c0", device=b"2330", numa=1 << 1)])


def random_devs(n, seed, all_attrs=False, no_physfn=False):
    """n in-domain records: the mdev layout's generator, then physfn present (16, 12 or 1 bytes) or not and physfn_device
    0..6 bytes where physfn is present (all_attrs: both at their longest; no_physfn: both empty)"""
    rng = np.random.default_rng(seed + 7)
    d = np.zeros(n, DRAMDEVPF_DTYPE)
    if n == 0:
        return d
    d["dev"] = MC.random_devs(n, seed, all_attrs)
    if no_physfn:
        return d
    addr = np.frombuffer(b"0123456789abcdef:.", np.uint8)
    xl = np.full(n, 16) if all_attrs else rng.choice([0, 1, 12, 16], n)
    yl = np.full(n, 6) if all_attrs else np.where(xl > 0, rng.choice([0, 1, 4, 6], n), 0)
    d["physfn"] = MC._text(rng, n, 16, addr, xl).view("S16").reshape(n)
    d["physfn_device"] = MC._text(rng, n, 8, MC._HEX, yl).view("S8").reshape(n)
    return d


# one field per out-of-domain case of the two new fields: (name of the rule, field, value)
BAD = [
    ("physfn", "physfn", b"0000:41:00.0/"),
    ("physfn", "physfn", b"0000:41:0G.0"),
    ("physfn_device", "physfn_device", b"233g"),
    ("physfn_device", "physfn_device", b"1234567"),
]


def bad_rec(field, value, physfn=b"0000:41:00.0"):
    r = rec(physfn=physfn)
    r[field] = value
    return r
