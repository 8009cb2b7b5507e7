"""Inputs for the tests of PCIe root ports and switches in DRA (kxpu_pcie_ports and kxpu_dra_slices_pcie, additions to
ABI v14): the rule's hand cases as walks with their expected keys, a seeded walk generator, the slice record built on
kxpu_dra_slices_pf's record, the cfg1 pool, one attribute domain per position among the nine keys, and the
out-of-domain cases."""
import numpy as np

import dra_pf_cases as PF
import pcie_example as EX
from kxpu_b200.binding import DEVREC_DTYPE, DRADEVPCIE_DTYPE, PCIE_NO_KEY, PCIPATH_DTYPE

NO = PCIE_NO_KEY
DOMAIN = "pcie.example.com"


def fkey(addr):
    """function key of "dddd:bb:dd.f" (the domain may have 5..8 digits)"""
    dom, bus, df = addr.split(":")
    dev, fn = df.split(".")
    return int(dom, 16) << 16 | int(bus, 16) << 8 | int(dev, 16) << 3 | int(fn)


def walk(groups):
    """groups: lists of (bdf, path or None) -> (recs, paths, group_off, group_members), one record per member"""
    members = [m for g in groups for m in g]
    recs = np.zeros(len(members), DEVREC_DTYPE)
    paths = np.zeros(len(members), PCIPATH_DTYPE)
    for i, (bdf, path) in enumerate(members):
        recs[i]["bdf"] = bdf.encode()
        if path is not None:
            paths[i]["path"] = path.encode()
            paths[i]["len"] = len(path)
    off = np.cumsum([0] + [len(g) for g in groups]).astype(np.uint32)
    return recs, paths, off, np.arange(len(members), dtype=np.uint32)


def _p(*comps):
    return "/".join(comps)


# (name, groups, [(root port, switch) per group]) -- addresses, or None for KXPU_PCIE_NO_KEY
HAND = [
    ("pcie_example", [[m] for m in EX.gpu_paths()],
     [("0000:00:01.0", "0000:01:00.0")] * 2 + [("0000:00:02.0", "0000:05:00.0")] * 2 +
     [("0000:80:01.0", "0000:81:00.0")] * 2 + [("0000:80:02.0", "0000:85:00.0")] * 2),
    ("below_root_port", [[("0000:06:00.0", _p("pci0000:00", "0000:00:03.0", "0000:06:00.0"))]],
     [("0000:00:03.0", None)]),
    ("two_level_switch", [[("0000:05:00.0", _p("pci0000:00", "0000:00:01.0", "0000:01:00.0", "0000:02:00.0",
                                              "0000:03:00.0", "0000:04:08.0", "0000:05:00.0"))]],
     [("0000:00:01.0", "0000:03:00.0")]),
    ("vmd", [[("10000:e3:00.0", _p("pci0000:00", "0000:00:0e.0", "pci10000:e0", "10000:e0:1d.0", "10000:e1:00.0",
                                   "10000:e2:00.0", "10000:e3:00.0"))],
             [("10000:e0:1e.0", _p("pci0000:00", "0000:00:0e.0", "pci10000:e0", "10000:e0:1e.0"))]],
     [("10000:e0:1d.0", "10000:e1:00.0"), (None, None)]),
    ("two_down_ports", [[("0000:03:00.0", _p("pci0000:00", "0000:00:01.0", "0000:01:00.0", "0000:02:00.0", "0000:03:00.0")),
                         ("0000:04:00.0", _p("pci0000:00", "0000:00:01.0", "0000:01:00.0", "0000:02:01.0", "0000:04:00.0"))]],
     [("0000:00:01.0", "0000:01:00.0")]),
    ("two_root_ports", [[("0000:03:00.0", _p("pci0000:00", "0000:00:01.0", "0000:03:00.0")),
                         ("0000:04:00.0", _p("pci0000:00", "0000:00:02.0", "0000:04:00.0"))]],
     [(None, None)]),
    ("vf_beside_pf", [[("0000:3b:00.0", _p("pci0000:3a", "0000:3a:00.0", "0000:3b:00.0"))],
                      [("0000:9b:00.1", _p("pci0000:98", "0000:98:01.0", "0000:99:00.0", "0000:9a:04.0", "0000:9b:00.1"))],
                      [("0000:9b:00.0", _p("pci0000:98", "0000:98:01.0", "0000:99:00.0", "0000:9a:04.0", "0000:9b:00.0"))]],
     [("0000:3a:00.0", None), ("0000:98:01.0", "0000:99:00.0"), ("0000:98:01.0", "0000:99:00.0")]),
    ("pcie_to_pci_bridge", [[("0000:08:01.0", _p("pci0000:00", "0000:00:1c.0", "0000:07:00.0", "0000:08:01.0"))]],
     [("0000:00:1c.0", "0000:07:00.0")]),
    ("eight_deep", [[("0000:07:00.0", _p("pci0000:00", *["0000:%02x:%02x.0" % (b, 1 if b == 0 else 0) for b in range(7)],
                                          "0000:07:00.0"))],
                    [("0000:08:00.0", _p("pci0000:00", *["0000:%02x:%02x.0" % (b, 1 if b == 0 else 0) for b in range(8)],
                                          "0000:08:00.0"))]],  # nine deep: unknown
     [("0000:00:01.0", "0000:05:00.0"), (None, None)]),
    ("unknown", [[("0000:03:00.0", None)], [("0000:03:00.0", "pci0000:00/0000:00:01.0/0000:03:00.1")],
                 [("0000:03:00.0", None), ("0000:04:00.0", _p("pci0000:00", "0000:00:01.0", "0000:01:00.0", "0000:04:00.0"))],
                 []],
     [(None, None), (None, None), ("0000:00:01.0", "0000:01:00.0"), (None, None)]),
]


def expected(pairs):
    """the wanted keys of a hand case"""
    k = lambda a: NO if a is None else fkey(a)  # noqa: E731
    return [k(a) for a, _ in pairs], [k(b) for _, b in pairs]


def random_walk(n_groups, seed, unknown=0.1, max_members=3):
    """a seeded walk: groups of 0..max_members members whose paths come from a small random PCIe forest (two domains,
    one of them a VMD domain, switch trees 0..3 deep), some of them unknown or malformed"""
    rng = np.random.default_rng(seed)
    groups = []
    for g in range(n_groups):
        members = []
        base = ["pci0000:%02x" % (rng.integers(4) * 0x40)]
        if rng.random() < 0.2:  # behind a VMD endpoint
            base += ["0000:%s:0e.0" % base[0][-2:], "pci1%04x:e0" % rng.integers(0x10000)]
        dom = "0000" if len(base) == 1 else base[-1][3:8]
        chain = base + ["%s:%s:%02x.0" % (dom, base[-1][-2:], 1 + rng.integers(3))]
        for d in range(int(rng.integers(0, 7))):
            chain.append("%s:%02x:%02x.%d" % (dom, 1 + rng.integers(200), rng.integers(32), rng.integers(8)))
        for m in range(int(rng.integers(0, max_members + 1))):
            c = list(chain)
            if m and rng.random() < 0.5:  # the next member diverges somewhere
                c = c[:int(rng.integers(1, len(c) + 1))]
                c.append("%s:%02x:%02x.0" % (dom, 1 + rng.integers(200), rng.integers(32)))
            bdf = "%s:%02x:%02x.%d" % (dom, rng.integers(256), rng.integers(32), rng.integers(8))
            path = _p(*c[:8], bdf)
            r = rng.random()
            if r < unknown / 2:
                path = None
            elif r < unknown:
                path = path.replace(":", ";", 1) if rng.random() < 0.5 else path + "/"
            members.append((bdf, path))
        groups.append(members)
    return walk(groups)


def rec(root_port=NO, pcie_switch=NO, **kw):
    r = np.zeros(1, DRADEVPCIE_DTYPE)
    r["pf"] = PF.rec(**kw)
    r["root_port"], r["pcie_switch"] = root_port, pcie_switch
    return r


def cfg1():
    """an H100 under a switch, a NIC VF below the same switch, a GPU directly below its root port, and a function whose
    ports are unknown"""
    return np.concatenate([
        rec(group=214, root_port=fkey("0000:c0:01.0"), pcie_switch=fkey("0000:c1:00.0"), bdf=b"0000:c3:00.0",
            root=b"pci0000:c0", numa=1 << 1),
        rec(group=45, bdf=b"0000:c4:00.2", vendor=b"15b3", device=b"101e", product=b"ConnectX-7_VF",
            root=b"pci0000:c0", numa=1 << 1, physfn=b"0000:c4:00.0", physfn_device=b"1021",
            root_port=fkey("0000:c0:01.0"), pcie_switch=fkey("0000:c1:00.0")),
        rec(group=7, bdf=b"10000:e1:00.0", root=b"pci10000:e0", root_port=fkey("10000:e0:1d.0")),
        rec(group=9, bdf=b"0000:41:00.0", root=b"pci0000:40")])


def random_devs(n, seed, all_attrs=False, no_keys=False, no_physfn=False, long_addr=False):
    """n in-domain records: kxpu_dra_slices_pf's generator, then a root port on most and a switch on some of those
    (no_keys: none; long_addr: 8-digit VMD domains, 16-byte addresses)"""
    rng = np.random.default_rng(seed + 11)
    d = np.zeros(n, DRADEVPCIE_DTYPE)
    d["root_port"], d["pcie_switch"] = NO, NO
    if n == 0:
        return d
    d["pf"] = PF.random_devs(n, seed, all_attrs=all_attrs, no_physfn=no_physfn)
    if no_keys:
        return d
    dom = rng.integers(0x10000000, 0x100000000, n, dtype=np.uint64) if long_addr else \
        np.where(rng.random(n) < 0.1, rng.integers(0x10000, 0x100000, n), rng.integers(0, 0x10000, n)).astype(np.uint64)
    low = rng.integers(0, 1 << 16, n, dtype=np.uint64)
    has_rp = np.ones(n, bool) if all_attrs else rng.random(n) < 0.8
    has_sw = has_rp & (np.ones(n, bool) if all_attrs else rng.random(n) < 0.6)
    d["root_port"] = np.where(has_rp, dom << np.uint64(16) | low, np.uint64(NO))
    d["pcie_switch"] = np.where(has_sw, dom << np.uint64(16) | (low ^ np.uint64(0x100)), np.uint64(NO))
    return d


# one attribute domain per position among the nine keys (the position is the count of keys before "<domain>/..."), and
# None where no lowercase domain can sort: between physfnAddress and physfnDeviceID
POSITIONS = ["a.io", "e.io", "j.io", "o.io", "pcia.io", None, "physfnd.io", "q.io", "s.io", "w.io"]

# domains kxpu_dra_slices_pcie refuses
BAD_DOMAINS = [None, "", "Pcie.example.com", "pcie_example.com", "-pcie.example.com", "pcie..example.com",
               "a" * 64, ("a" * 31 + ".") * 2 + "b", "kubernetes.io", "k8s.io", "pcie.kubernetes.io", "x.k8s.io",
               "pcie.example.com/x"]
# and ones it takes (near the reserved names, at the length limit)
GOOD_DOMAINS = ["xkubernetes.io", "k8s.io.example.com", "a" * 63, ("a" * 30 + ".") * 2 + "a", "1"]

# out-of-domain port keys: (name of the rule, root_port, pcie_switch)
BAD_KEYS = [
    ("port_key", 1 << 63 | 0x80 << 8, NO),                 # a host-bridge key
    ("port_key", fkey("0000:00:01.0"), 1 << 48 | 0x100),  # bit 48
    ("port_key", (1 << 62) | 8, NO),                       # bit 62
    ("port_orphan", NO, fkey("0000:01:00.0")),             # a switch without a root port
]
