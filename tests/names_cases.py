"""Inputs for the resource-name tests (kxpu_classify_named): hand walks, name tables and hypothesis strategies, shared by
the CPU and the GPU tests."""
import numpy as np
from hypothesis import strategies as st

import vf_vgpu_cases as VV
from oracle import xpu_oracle as XO

RULES = VV.RULES  # 0: 10de/vfio-pci, 1: 1002/vfio-pci, 2: 10de/nvidia (vGPU types with VGPU_BIT)
VGPU_BIT = VV.VGPU_BIT
DEVICES = [b"0x2330\n", b"0x2331\n", b"0x2321\n", b"0x22a3\n", b"0x74a1\n", b"0x5\n", b"0x2330"]


def walk(*devs):
    """records from (group, device, driver, vendor[, flags]) tuples, addresses in order"""
    recs = []
    for i, d in enumerate(devs):
        g, dev, drv, ven = d[:4]
        recs.append(VV.dev(b"0000:%02x:%02x.0" % (i // 32, i % 32), g, driver=drv, vendor=ven, device=dev,
                           flags=d[4] if len(d) > 4 else 0))
    return np.array(recs, XO.DEVREC_DTYPE)


NV, AMD, MGR = (b"vfio-pci", b"0x10de\n"), (b"vfio-pci", b"0x1002\n"), (b"nvidia", b"0x10de\n")
# (name, records, keys rows or None, vgpu bits, table)
HAND = [
    ("listed ids", walk((1, b"0x2330\n", *NV), (2, b"0x2331\n", *NV), (3, b"0x2321\n", *NV)), None, 0,
     [(0, b"2330", 0), (0, b"2331", 1)]),
    ("star", walk((1, b"0x2330\n", *NV), (2, b"0x2331\n", *NV), (3, b"0x2321\n", *NV)), None, 0, [(0, b"*", 0)]),
    ("two ids one name", walk((1, b"0x2331\n", *NV), (2, b"0x2330\n", *NV), (3, b"0x2331\n", *NV), (4, b"0x2321\n", *NV)),
     None, 0, [(0, b"2330", 0), (0, b"2331", 0)]),
    ("unlisted beside named", walk((1, b"0x2330\n", *NV), (2, b"0x22a3\n", *NV), (3, b"0x2330\n", *NV), (4, b"0x5\n", *NV)),
     None, 0, [(0, b"22a3", 1), (0, b"*", 0)]),
    ("unlisted only", walk((1, b"0x2330\n", *NV), (2, b"0x22a3\n", *NV)), None, 0, [(0, b"22a3", 0)]),
    ("named and unnamed rules", walk((1, b"0x2330\n", *NV), (2, b"0x74a1\n", *AMD), (3, b"0x2331\n", *NV),
                                     (4, b"0x74a1\n", *AMD)), None, 0, [(0, b"*", 0)]),
    ("slot of a non-first member", walk((1, b"0x2330\n", *NV), (1, b"0x2331\n", *NV), (2, b"0x2331\n", *NV)), None, 0,
     [(0, b"2331", 0)]),
    ("failed device read", walk((1, b"0x2330\n", *NV, VV.VC.DEVICE_ERR), (1, b"0x2330\n", *NV), (2, b"0x2331\n", *NV)), None,
     0, [(0, b"*", 0)]),
]


def vgpu_case():
    """a named class next to a vfVgpu class in one walk"""
    recs = walk((1, b"0x2330\n", *NV), (2, b"0x2331\n", *MGR), (3, b"0x2331\n", *MGR), (4, b"0x2331\n", *NV),
                (5, b"0x2331\n", *MGR))
    keys = np.array([VV.key(k) for k in (b"", b"NVIDIA_H100-4C", b"NVIDIA_H100-8C", b"", b"NVIDIA_H100-4C")],
                    VV.VGPUKEY_DTYPE)
    return recs, keys, VGPU_BIT, [(0, b"*", 0), (1, b"74a1", 1)]


# (table, n_rules, vgpu bits) the call refuses
INVALID = [
    ([(3, b"2330", 0)], 3, 0),                      # rule >= n_rules
    ([(2, b"2330", 0)], 3, VGPU_BIT),               # a vGPU rule
    ([(0, b"233", 0)], 3, 0),                       # three digits
    ([(0, b"2330\0\0\0x", 0)], 3, 0),               # a byte after the NUL
    ([(0, b"23A0", 0)], 3, 0),                      # upper case
    ([(0, b"**", 0)], 3, 0),
    ([(0, b"", 0)], 3, 0),
    ([(0, b"2330", 0), (0, b"2330", 1)], 3, 0),     # one (rule, id) twice
    ([(0, b"*", 0), (0, b"*", 0)], 3, 0),
    ([(0, b"2330", 1)], 3, 0),                      # slot >= n_names
    ([(0, b"%04x" % k, 0) for k in range(65)], 3, 0),  # over KXPU_MAX_NAMES
]


@st.composite
def named_inputs(draw):
    """(recs, keys, table) over the three rules: ids from a small pool, some groups shared, a random table"""
    recs, keys = draw(VV.classify_inputs())
    recs = np.array(recs, copy=True)
    for i in range(len(recs)):
        d = draw(st.sampled_from(DEVICES))
        recs[i]["device_txt"] = np.frombuffer(d.ljust(8, b"\0"), np.uint8)
        recs[i]["device_len"] = len(d)
    ids = draw(st.lists(st.tuples(st.sampled_from([0, 1]), st.sampled_from([b"2330", b"2331", b"2321", b"22a3", b"74a1",
                                                                              b"*"])), unique=True, max_size=8))
    table = [(r, d, draw(st.integers(0, max(len(ids) - 1, 0)))) for r, d in ids]
    return recs, keys, table
