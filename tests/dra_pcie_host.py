"""Fake-sysfs helpers for Plugin::draPcieDomain (PCIe root ports and switches in DRA): pcie_example's eight GPUs, a
NIC PF on its vendor driver below the first switch of each socket with VFs on vfio-pci in a second class, the
setting, and the slices of both pools."""
import ctypes as C
import json

import pcie_example as EX
import pcie_host
import sriov_host as SH

CLASSES = ("10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-nvidia;"
           "15b3,vfio-pci,mellanox.com,mellanox.com/nic,cdi-vfio-nic")
DRIVERS = ["gpu.example.com", "nic.example.com"]
DOMAIN = "pcie.example.com"
RP, SW = DOMAIN + "/pcieRootPort", DOMAIN + "/pcieSwitch"
NV = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
NIC = dict(vendor=b"0x15b3\n", device=b"0x101e\n")
PF_A, PF_B = "0000:0a:00.0", "0000:8a:00.0"
VFS_A, VFS_B = ["0000:0a:00.1", "0000:0a:00.2"], ["0000:8a:00.1"]
_SW_A = "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:02.0/"  # a third down port of socket 0's first switch
_SW_B = "pci0000:80/0000:80:01.0/0000:81:00.0/0000:82:02.0/"


def devices():
    gpus = [dict(bdf=bdf, path=path, group=g, **NV) for (bdf, path), g in zip(EX.gpu_paths(), EX.GROUPS)]
    nics = [dict(bdf=PF_A, path=_SW_A + PF_A, group=70, driver="mlx5_core", **NIC),
            dict(bdf=VFS_A[0], path=_SW_A + VFS_A[0], group=71, driver="vfio-pci", **NIC),
            dict(bdf=VFS_A[1], path=_SW_A + VFS_A[1], group=72, driver="vfio-pci", **NIC),
            dict(bdf=PF_B, path=_SW_B + PF_B, group=80, driver="mlx5_core", **NIC),
            dict(bdf=VFS_B[0], path=_SW_B + VFS_B[0], group=81, driver="vfio-pci", **NIC)]
    return gpus + nics


def make_tree(root):
    base = pcie_host.make_nested_tree(root, devices(), relative=True)
    SH.link_vfs(base, PF_A, VFS_A, b"2\n")
    SH.link_vfs(base, PF_B, VFS_B, b"1\n")
    return base


def set_domain(hp, domain):
    hp.L.kxh_set_dra_pcie_domain.argtypes = [C.c_void_p, C.c_char_p]
    hp.L.kxh_set_dra_pcie_domain(hp.h, None if domain is None else domain.encode())


def devices_of(blob):
    """device name -> device of a pool's slices"""
    return {d["name"]: d for line in blob.splitlines() for d in json.loads(line)["spec"]["devices"]}
