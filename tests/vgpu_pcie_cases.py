"""Inputs for the tests of PCIe root ports and switches of vGPUs in DRA (kxpu_pcie_ports_mdev,
kxpu_dra_slices_mdev_pcie and kxpu_dra_slices_vf_vgpu_pcie, additions to ABI v14): the rule's hand cases as mdev walks
with their expected keys, a seeded mdev walk with the parents' own PCI records, the two slice records built on the
mdev-PF and VF-vGPU records, the cfg1 pools and one attribute domain per position among each layout's keys."""
import numpy as np

import dra_vf_vgpu_cases as VF
import mdev_pf_cases as MP
import pcie_mdev_cases as MC
from dra_pcie_cases import DOMAIN, NO, fkey  # noqa: F401
from kxpu_b200.binding import DEVREC_DTYPE, DRAMDEVPCIE_DTYPE, DRAVFVGPUPCIE_DTYPE, PCIPATH_DTYPE

# (name, rows of (uuid number, parent, parent's own path), groups or None, expected (root port, switch) per group)
HAND = [
    ("below_switch", [(1, "0000:03:00.0", "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0")], None,
     [("0000:00:01.0", "0000:01:00.0")]),
    ("below_root_port", [(2, "0000:01:00.0", "pci0000:00/0000:00:01.0/0000:01:00.0")], None, [("0000:00:01.0", None)]),
    ("below_host_bridge", [(3, "0000:00:05.0", "pci0000:00/0000:00:05.0")], None, [(None, None)]),
    ("vf_parent", [(4, "0000:03:00.4", "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.4")], None,
     [("0000:00:01.0", "0000:01:00.0")]),
    ("vmd_domain", [(5, "10000:e1:00.0", "pci0000:00/0000:00:0e.0/pci10000:e0/10000:e0:1d.0/10000:e1:00.0")], None,
     [("10000:e0:1d.0", None)]),
    # a host bridge and five functions: the longest chain the 120-byte cap leaves beside the UUID
    ("at_depth_cap", [(7, "0000:04:00.0", "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0/0000:04:00.0")],
     None, [("0000:00:01.0", "0000:03:00.0")]),
    ("two_gpus_one_switch", [(8, "0000:03:00.0", "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:00.0/0000:03:00.0"),
                             (9, "0000:04:00.0", "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:01.0/0000:04:00.0")],
     [[0, 1]], [("0000:00:01.0", "0000:01:00.0")]),
    ("unknown_path", [(10, "0000:03:00.0", None)], None, [(None, None)]),
]


def hand_walk(rows, groups):
    return MC.walk([MC.mdev(MC.uuid(k), parent, chain) if chain else (MC.rec(MC.uuid(k), parent), MC.path(""))
                    for k, parent, chain in rows], groups)


def expected(pairs):
    k = lambda a: NO if a is None else fkey(a)  # noqa: E731
    return [k(a) for a, _ in pairs], [k(b) for _, b in pairs]


def random_walk(n, seed, unknown=0.05, per_group=1):
    """n mdevs on parents drawn from a small forest (two host bridges, root ports, switches 0..2 deep, VF parents beside
    their PFs, a VMD domain), per_group consecutive mdevs to a group (the last group may be shorter), so a group's
    members may sit below different parents; returns (mdev walk, the parents' PCI walk with the same groups: recs,
    paths, off, members)"""
    rng = np.random.default_rng(seed)
    rows, prow = [], []
    for i in range(n):
        hb = int(rng.integers(2)) * 0x80
        comps = ["pci0000:%02x" % hb]
        dom = "0000"
        if rng.random() < 0.1:
            comps += ["0000:%02x:0e.0" % hb, "pci1%04x:e0" % int(rng.integers(0x10000))]
            dom = comps[-1][3:8]
        if rng.random() < 0.95:
            comps.append("%s:%02x:%02x.0" % (dom, hb if dom == "0000" else 0xe0, 1 + int(rng.integers(3))))
        for d in range(int(rng.integers(0, 5))):
            comps.append("%s:%02x:%02x.0" % (dom, 1 + int(rng.integers(200)), int(rng.integers(32))))
        parent = "%s:%02x:%02x.%d" % (dom, int(rng.integers(256)), int(rng.integers(32)),
                                      int(rng.integers(8)) if rng.random() < 0.3 else 0)
        while len(comps) > 1 and len("/".join(comps + [parent])) + 37 > 120:  # the mdev's link within the cap
            comps.pop()
        chain = "/".join(comps + [parent])
        u = MC.uuid(i)
        r, p = MC.mdev(u, parent, chain)
        if rng.random() < unknown:
            p = MC.path(chain + "/" + MC.uuid(i + 1))  # a leaf that is not the record's UUID
        rows.append((r, p))
        prow.append((parent, chain))
    groups = [list(range(g, min(n, g + per_group))) for g in range(0, n, per_group)]
    mwalk = MC.walk(rows, groups)
    precs = np.zeros(n, DEVREC_DTYPE)
    ppaths = np.zeros(n, PCIPATH_DTYPE)
    for i, (parent, chain) in enumerate(prow):
        precs[i]["bdf"] = parent.encode()
        b = chain.encode()
        if len(b) <= 120:
            ppaths[i]["path"], ppaths[i]["len"] = b, len(b)
    return mwalk, (precs, ppaths, mwalk[2], mwalk[3])


def mdev_rec(root_port=NO, pcie_switch=NO, **kw):
    r = np.zeros(1, DRAMDEVPCIE_DTYPE)
    r["pf"] = MP.rec(**kw)
    r["root_port"], r["pcie_switch"] = root_port, pcie_switch
    return r


def vf_rec(root_port=NO, pcie_switch=NO, **kw):
    r = np.zeros(1, DRAVFVGPUPCIE_DTYPE)
    r["dev"] = VF.rec(**kw)
    r["root_port"], r["pcie_switch"] = root_port, pcie_switch
    return r


def mdev_cfg1():
    """mdev_pf's cfg1 with the ports the rule gives: the mdev on VF 0000:41:00.4 of an H100 directly below root port
    0000:40:01.0 (no switch), and the mdev on H100 0000:c3:00.0 below root port 0000:c0:01.0 and the switch whose
    upstream port is 0000:c1:00.0 (its downstream port 0000:c2:00.0)"""
    d = np.zeros(2, DRAMDEVPCIE_DTYPE)
    d["pf"] = MP.cfg1()
    d["pf"]["dev"]["parent"][1] = b"0000:c3:00.0"
    d["root_port"] = [fkey("0000:40:01.0"), fkey("0000:c0:01.0")]
    d["pcie_switch"] = [NO, fkey("0000:c1:00.0")]
    return d


def vf_cfg1():
    """a vGPU on VF 0000:c3:00.4 of the H100 0000:c3:00.0 below root port 0000:c0:01.0 and the switch 0000:c1:00.0, and
    one on VF 0000:41:00.4 whose path was unknown (no ports)"""
    return np.concatenate([vf_rec(bdf=b"0000:c3:00.4", parent=b"0000:c3:00.0", root_port=fkey("0000:c0:01.0"),
                                  pcie_switch=fkey("0000:c1:00.0")),
                           vf_rec(group=302, bdf=b"0000:41:00.4", parent=b"0000:41:00.0", root=b"pci0000:40", numa=1 << 0)])


def random_mdev_devs(n, seed, all_attrs=False, no_keys=False, no_physfn=False, long_addr=False):
    d = np.zeros(n, DRAMDEVPCIE_DTYPE)
    d["root_port"], d["pcie_switch"] = NO, NO
    if n == 0:
        return d
    d["pf"] = MP.random_devs(n, seed, all_attrs=all_attrs, no_physfn=no_physfn)
    if not no_keys:
        _keys(d, n, seed, all_attrs, long_addr)
    return d


def random_vf_devs(n, seed, all_attrs=False, no_keys=False, long_addr=False):
    d = np.zeros(n, DRAVFVGPUPCIE_DTYPE)
    d["root_port"], d["pcie_switch"] = NO, NO
    if n == 0:
        return d
    d["dev"] = VF.random_devs(n, seed, all_attrs=all_attrs)
    if not no_keys:
        _keys(d, n, seed, all_attrs, long_addr)
    return d


def _keys(d, n, seed, all_attrs, long_addr):
    """a root port on most records and a switch on some of those (long_addr: 8-digit VMD domains, 16-byte addresses)"""
    rng = np.random.default_rng(seed + 13)
    dom = rng.integers(0x10000000, 0x100000000, n, dtype=np.uint64) if long_addr else \
        np.where(rng.random(n) < 0.1, rng.integers(0x10000, 0x100000, n), rng.integers(0, 0x10000, n)).astype(np.uint64)
    low = rng.integers(0, 1 << 16, n, dtype=np.uint64)
    has_rp = np.ones(n, bool) if all_attrs else rng.random(n) < 0.8
    has_sw = has_rp & (np.ones(n, bool) if all_attrs else rng.random(n) < 0.6)
    d["root_port"] = np.where(has_rp, dom << np.uint64(16) | low, np.uint64(NO))
    d["pcie_switch"] = np.where(has_sw, dom << np.uint64(16) | (low ^ np.uint64(0x100)), np.uint64(NO))


# the layouts' sorted keys
MDEV_KEYS = ["iommuGroup", "mdevType", "numaNode", "parentAddress", "parentDeviceID", "parentVendorID", "physfnAddress",
             "physfnDeviceID", "productName", "resource.kubernetes.io/pcieRoot", "uuid"]
VF_KEYS = ["iommuGroup", "numaNode", "parentAddress", "parentDeviceID", "parentVendorID", "pciAddress", "productName",
           "resource.kubernetes.io/pcieRoot", "vgpuType", "vgpuTypeID"]
# one attribute domain per position among each layout's keys, None where no lowercase domain can sort
MDEV_POSITIONS = ["example.com", "j.io", "n.io", "o.io", None, None, "pb.io", None, "pr.io", "q.io", "s.io", "x.io"]
VF_POSITIONS = ["example.com", "j.io", "o.io", None, None, "pb.io", "pd.io", "q.io", "s.io", None, "x.io"]


def position(keys, domain):
    """the count of keys that sort before "<domain>/pcieRootPort\""""
    return sum(k < domain + "/pcieRootPort" for k in keys)
