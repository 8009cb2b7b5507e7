"""The worked example of include/kxpu.h's kxpu_preferred_allocation_pcie (and of the issue that introduced it): two
sockets, each a host bridge with two root ports, a switch under each root port and two GPUs under each switch's down
ports.  Groups 10-13 sit on NUMA node 0 under pci0000:00, groups 20-23 on node 1 under pci0000:80; device positions
are 0..7 in that order.  Shared by the CPU, GPU and host tests."""
import numpy as np

from oracle import xpu_oracle as XO
from kxpu_b200.binding import PCIPATH_DTYPE

GROUPS = [10, 11, 12, 13, 20, 21, 22, 23]


def gpu_paths():
    """bdf -> the sysfs link target below devices/ of each GPU, in position order."""
    out = []
    for b in (0x00, 0x80):  # root port -> switch -> down port -> GPU
        rows = [("%02x:01.0" % b, "%02x:00.0" % (b + 1), "%02x:00.0" % (b + 2), "%02x:00.0" % (b + 3)),
                ("%02x:01.0" % b, "%02x:00.0" % (b + 1), "%02x:01.0" % (b + 2), "%02x:00.0" % (b + 4)),
                ("%02x:02.0" % b, "%02x:00.0" % (b + 5), "%02x:00.0" % (b + 6), "%02x:00.0" % (b + 7)),
                ("%02x:02.0" % b, "%02x:00.0" % (b + 5), "%02x:01.0" % (b + 6), "%02x:00.0" % (b + 8))]
        for rp, sw, dp, gpu in rows:
            bdf = "0000:" + gpu
            out.append((bdf, "pci0000:%02x/0000:%s/0000:%s/0000:%s/%s" % (b, rp, sw, dp, bdf)))
    return out


def records():
    """(recs, paths, group_off, group_members): one accepted function per group, walk order = position order."""
    gp = gpu_paths()
    recs = np.zeros(len(gp), XO.DEVREC_DTYPE)
    paths = np.zeros(len(gp), PCIPATH_DTYPE)
    for i, (bdf, path) in enumerate(gp):
        recs[i]["bdf"] = bdf.encode()
        recs[i]["iommu_group"] = GROUPS[i]
        paths[i]["path"] = path.encode()
        paths[i]["len"] = len(path)
    return recs, paths, np.arange(len(gp) + 1, dtype=np.uint32), np.arange(len(gp), dtype=np.uint32)


DEV_NUMA = np.array([1, 1, 1, 1, 2, 2, 2, 2], np.uint64)

# (available groups, must-include groups, size, answer groups) -- the table of the example
ALL = GROUPS


def _but(g):
    return [x for x in GROUPS if x != g]


TABLE = [
    (ALL, [], 2, [10, 11]),
    (_but(10), [], 2, [12, 13]),
    (_but(10), [], 1, [11]),
    (_but(12), [], 1, [13]),
    (ALL, [12], 3, [12, 13, 10]),
    (ALL, [], 5, [10, 11, 12, 13, 20]),
]


def requests():
    pos = {g: i for i, g in enumerate(GROUPS)}
    return [([pos[g] for g in av], [pos[g] for g in mu], size) for av, mu, size, _ in TABLE]


def answers():
    pos = {g: i for i, g in enumerate(GROUPS)}
    return [[pos[g] for g in ans] for _, _, _, ans in TABLE]
