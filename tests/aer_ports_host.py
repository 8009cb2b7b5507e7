"""Fake-sysfs helpers for Plugin::aerPortHealth (the AER errors of the PCIe ports above a device): pcie_example's eight
GPUs with their root ports, switch upstream and downstream ports as entries of their own under the base path (bound to
pcieport, as on real sysfs), vGPUs on GPUs below the same ports, and the setting."""
import ctypes as C
import os

import aer_host as AH
import fake_mdev
import pcie_example as EX
import pcie_host
from fake_sysfs import host_lib

CLASS = "10de,vfio-pci,nvidia.com,nvidia.com/gpu,cdi-vfio-nvidia"
DRIVER = "gpu.example.com"
VGPU = [("10de", "nvidia-vgpu", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")]
NV = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
PORT = dict(vendor=b"0x1000\n", device=b"0xc030\n", driver="pcieport")
GPUS = EX.gpu_paths()  # (bdf, path), groups EX.GROUPS
# vGPU parents on socket 0's second root port: a GPU below its own switch, and a VF of it beside the PF
VGPU_PARENTS = {"0000:13:00.0": "pci0000:00/0000:00:03.0/0000:11:00.0/0000:12:00.0/0000:13:00.0",
                "0000:13:00.4": "pci0000:00/0000:00:03.0/0000:11:00.0/0000:12:00.0/0000:13:00.4"}
SIBLING = ("0000:02:02.0", "pci0000:00/0000:00:01.0/0000:01:00.0/0000:02:02.0")  # a down port with no GPU below
MDEVS = [dict(uuid="%08x-0000-4000-8000-%012x" % (k, k), parent=p, group=500 + k, driver="nvidia-vgpu",
              type_id="nvidia-471", name=b"GRID A100-10C\n") for k, p in enumerate(VGPU_PARENTS)]


def ports_of(path):
    """(bdf, path) of each function above the device at path, root first"""
    comps = path.split("/")
    return [(c, "/".join(comps[:k + 1])) for k, c in enumerate(comps[:-1]) if not c.startswith("pci")]


def make_tree(root, with_mdevs=False):
    """the PCI tree (GPUs and every port above them, each port with zero AER counts, each GPU too) and, with_mdevs, the
    vGPU parents' ports and the mdev tree; returns (pci base, mdev base or None)"""
    ports = {}
    for _, path in GPUS + (list(VGPU_PARENTS.items()) if with_mdevs else []):
        ports.update(ports_of(path))
    devs = [dict(bdf=b, path=p, group=g, **NV) for (b, p), g in zip(GPUS, EX.GROUPS)]
    ports[SIBLING[0]] = SIBLING[1]
    devs += [dict(bdf=b, path=p, **PORT) for b, p in sorted(ports.items())]
    base = pcie_host.make_nested_tree(root, devs, relative=True)
    for d in devs:
        AH.write(os.path.join(base, d["bdf"]))
    mbase = None
    if with_mdevs:
        mbase = fake_mdev.make_tree(root, [dict(m, parent=VGPU_PARENTS[m["parent"]]) for m in MDEVS],
                                    parents={p: b"0x10de\n" for p in VGPU_PARENTS.values()})
        for m in MDEVS:
            link = os.path.join(mbase, m["uuid"])
            os.remove(link)
            os.symlink(os.path.join("../../../devices", VGPU_PARENTS[m["parent"]], m["uuid"]), link)
        for p, path in VGPU_PARENTS.items():  # the parents' own files (their entries are not in the PCI walk's classes)
            AH.write(os.path.join(root, "devices", path))
            os.symlink(os.path.join("../../../devices", path), os.path.join(base, p))
    return base, mbase


def enable(hp, on=True):
    L = host_lib()
    L.kxh_set_aer_port_health.argtypes = [C.c_void_p, C.c_int]
    L.kxh_set_aer_port_health(hp.h, int(on))
