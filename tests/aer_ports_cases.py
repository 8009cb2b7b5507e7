"""Inputs for the tests of kxpu_aer_ports and kxpu_aer_ports_mdev (additions to ABI v14): the rule's hand cases as PCI
and mdev walks with the ports each record must get, and the expected outputs built from them by first occurrence."""
import numpy as np

import pcie_mdev_cases as MC
from dra_pcie_cases import fkey
from kxpu_b200.binding import DEVREC_DTYPE, PCIPATH_DTYPE


def _p(*comps):
    return "/".join(comps)


def pci_walk(rows):
    """rows of (bdf, path text or None, or an int: that length with a valid-looking text) -> (recs, paths)"""
    recs = np.zeros(len(rows), DEVREC_DTYPE)
    paths = np.zeros(len(rows), PCIPATH_DTYPE)
    for i, (bdf, path) in enumerate(rows):
        recs[i]["bdf"] = bdf.encode()
        if isinstance(path, int):  # a length field above the text (over 120: unknown)
            paths[i]["path"] = (b"pci0000:00/0000:00:01.0/" + bdf.encode()).ljust(120, b"0")
            paths[i]["len"] = path
        elif path is not None:
            paths[i]["path"] = path.encode()
            paths[i]["len"] = len(path)
    return recs, paths


_SW = ("pci0000:00", "0000:00:01.0", "0000:01:00.0")  # a root port and a switch upstream port
_DEEP = ["0000:%02x:%02x.0" % (b, 1 if b == 0 else 0) for b in range(8)]

# (name, rows, the port addresses of each record, nearest first)
PCI = [
    ("below_switch", [("0000:03:00.0", _p(*_SW, "0000:02:00.0", "0000:03:00.0"))],
     [["0000:02:00.0", "0000:01:00.0", "0000:00:01.0"]]),
    ("shared_switch", [("0000:03:00.0", _p(*_SW, "0000:02:00.0", "0000:03:00.0")),
                       ("0000:04:00.0", _p(*_SW, "0000:02:01.0", "0000:04:00.0")),
                       ("0000:03:00.1", _p(*_SW, "0000:02:00.0", "0000:03:00.1"))],
     [["0000:02:00.0", "0000:01:00.0", "0000:00:01.0"], ["0000:02:01.0", "0000:01:00.0", "0000:00:01.0"],
      ["0000:02:00.0", "0000:01:00.0", "0000:00:01.0"]]),
    ("vmd", [("10000:e3:00.0", _p("pci0000:00", "0000:00:0e.0", "pci10000:e0", "10000:e0:1d.0", "10000:e1:00.0",
                                  "10000:e2:00.0", "10000:e3:00.0")),
             ("10000:e0:1e.0", _p("pci0000:00", "0000:00:0e.0", "pci10000:e0", "10000:e0:1e.0"))],
     [["10000:e2:00.0", "10000:e1:00.0", "10000:e0:1d.0", "0000:00:0e.0"], ["0000:00:0e.0"]]),
    ("host_bridge_only", [("0000:00:05.0", _p("pci0000:00", "0000:00:05.0"))], [[]]),
    ("unknown", [("0000:03:00.0", None), ("0000:03:00.0", _p("pci0000:00", "0000:00:01.0", "0000:03:00.1")),
                 ("0000:03:00.0", _p("0000:00:01.0", "0000:03:00.0")), ("0000:03:00.0", 121),
                 ("0000:03:00.0", _p(*_SW, "0000:03:00.0") + "/")],
     [[], [], [], [], []]),
    ("eight_deep", [("0000:07:00.0", _p("pci0000:00", *_DEEP[:7], "0000:07:00.0")),
                    ("0000:08:00.0", _p("pci0000:00", *_DEEP, "0000:08:00.0"))],  # nine keys of chain: unknown
     [list(reversed(_DEEP[:7])), []]),
    ("first_occurrence", [("0000:42:00.0", _p("pci0000:40", "0000:40:01.0", "0000:41:00.0", "0000:42:00.0")),
                          ("0000:03:00.0", _p(*_SW, "0000:02:00.0", "0000:03:00.0")),
                          ("0000:41:00.0", _p("pci0000:40", "0000:40:01.0", "0000:41:00.0")),
                          ("0000:02:00.0", _p(*_SW, "0000:02:00.0"))],
     [["0000:41:00.0", "0000:40:01.0"], ["0000:02:00.0", "0000:01:00.0", "0000:00:01.0"], ["0000:40:01.0"],
      ["0000:01:00.0", "0000:00:01.0"]]),
]

_GPU = _p(*_SW, "0000:02:00.0")
# (name, rows of (uuid number, parent, the parent's own path or None), the port addresses of each mdev)
MDEV = [
    ("on_pf", [(1, "0000:03:00.0", _GPU + "/0000:03:00.0"), (2, "0000:03:00.0", _GPU + "/0000:03:00.0")],
     [["0000:02:00.0", "0000:01:00.0", "0000:00:01.0"]] * 2),
    ("on_vf", [(3, "0000:03:00.4", _GPU + "/0000:03:00.4")], [["0000:02:00.0", "0000:01:00.0", "0000:00:01.0"]]),
    ("below_host_bridge", [(4, "0000:00:05.0", "pci0000:00/0000:00:05.0")], [[]]),
    ("vmd", [(5, "10000:e1:00.0", "pci0000:00/0000:00:0e.0/pci10000:e0/10000:e0:1d.0/10000:e1:00.0")],
     [["10000:e0:1d.0", "0000:00:0e.0"]]),
    ("unknown", [(6, "0000:03:00.0", None), (7, "0000:03:00.0", "pci0000:00/0000:00:01.0/0000:03:00.1")], [[], []]),
]


def mdev_walk(rows):
    recs, paths, _, _ = MC.walk([MC.mdev(MC.uuid(k), parent, chain) if chain else (MC.rec(MC.uuid(k), parent), MC.path(""))
                                 for k, parent, chain in rows])
    return recs, paths


def expected(port_lists):
    """(port_off, port_of, port_key) lists of a hand case, numbered by first occurrence"""
    number, off, of = {}, [0], []
    for ports in port_lists:
        for a in ports:
            of.append(number.setdefault(fkey(a), len(number)))
        off.append(len(of))
    return off, of, list(number)
