"""GPU end to end of the host plugin with a vGPU class served through VFIO cdevs (XpuClass::mdevCdev, with a DRA driver)
beside a vGPU class and a passthrough class served through group nodes, on a fake sysfs: the specs, an mdev without a
cdev (Unhealthy with its reason, refused by Allocate and PrepareDraDevices, left out of the spec and the DRA pool), a
moved cdev across Allocate and rediscover, a restart with resumeIndices and the setting switched both ways, and the
setting off reading nothing under vfio-dev/."""
import os

import numpy as np
import pytest

import cdev_host as H
import dra_host as DH
import dra_mdev_host as MH
import fake_mdev
import fake_sysfs
import mdev_cdev_cases as K
import viab_host
from oracle import mdev_oracle as MO

pytestmark = pytest.mark.gpu

PARENTS = [dict(bdf="0000:3b:00.0", vendor=b"0x10de\n", device=b"0x1eb8\n", driver="nvidia", group=40),
           dict(bdf="0000:00:02.0", vendor=b"0x8086\n", device=b"0x3e92\n", driver="i915", group=1),
           dict(bdf="0000:81:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=80)]
U = ["0b2ad9a2-6e2c-4a55-9d41-%012x" % k for k in range(8)]
MDEVS = [dict(uuid=U[1], parent="0000:3b:00.0", group=300),
         dict(uuid=U[2], parent="0000:3b:00.0", group=301),
         dict(uuid=U[3], parent="0000:3b:00.0", group=302),  # no vfio-dev/: no cdev
         dict(uuid=U[4], parent="0000:00:02.0", group=310, type_id="i915-GVTg_V5_4", name=b"GVTg_V5_4\n")]
CDEVS = {U[1]: 7, U[2]: 8, U[4]: 9}  # U[4]'s class does not set mdevCdev: never read
NVV = ("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")
INTEL = ("8086", "vfio_mdev", "intel.com", "intel.com/gvt", "cdi-mdev-intel")
VDRV = "vgpu.nvidia.com"
WHY = U[3] + " has no VFIO cdev"


def _plugin(kx, tree, cdev, resume=False):
    base, mbase, pciids, cdi = tree
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    fake_mdev.set_vgpu(hp, mbase, [NVV + ("mdev-cdev",) if cdev else NVV, INTEL])
    MH.set_vgpu_dra(hp, [VDRV, ""])
    if resume:
        import ctypes as C
        hp.L.kxh_set_resume.argtypes = [C.c_void_p, C.c_int]
        hp.L.kxh_set_resume(hp.h, 1)
    return hp


def _vgpu_plugin(state, cls):
    return next(i for i, p in enumerate(state["plugins"]) if p["vgpu"] and p["class"] == cls)


def _records(state, nodes):
    """the MDEVCDEV records of the NVIDIA class's mdevs named in `nodes` (uuid -> N), in ascending index"""
    rows = []
    for group, devs in state["mdevMap"]:
        for uuid, parent, index, cls in devs:
            if cls == 0 and uuid in nodes:
                rows.append(((uuid.encode(), int(group), parent.encode(), index), nodes[uuid]))
    rows.sort(key=lambda r: r[0][3])
    a = np.zeros(len(rows), K.MDEVCDEV_DTYPE)
    for i, (d, n) in enumerate(rows):
        a[i]["dev"], a[i]["vfio_cdev"] = d, n
    return a


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = fake_sysfs.make_tree(root, PARENTS)
    mbase = fake_mdev.make_tree(root, MDEVS)
    for u, n in CDEVS.items():
        H.set_vfio_dev(mbase, u, ["vfio%d" % n])
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = str(tmp_path / "cdi") + "/"
    os.makedirs(cdi)
    return base, mbase, str(tmp_path / "pci.ids"), cdi


def test_mdev_cdev_class_end_to_end(kx, tree):
    base, mbase, pciids, cdi = tree
    nv_file, intel_file, pt_file = cdi + "cdi-mdev-nvidia.yaml", cdi + "cdi-mdev-intel.yaml", cdi + "cdi-vfio-xxxx.yaml"

    # the setting off: nothing under vfio-dev/ is read, the vGPU spec is the group layout's
    off = _plugin(kx, tree, False)
    a = off.init()
    assert H.cdev_reads(off) == 0
    files_off = {f: open(f, "rb").read() for f in (nv_file, intel_file, pt_file)}
    assert files_off[nv_file] == MO.cdi_emit_mdev(K.FMT_YAML, b"nvidia.com/vgpu",
                                                  np.ascontiguousarray(_records(a, {U[1]: 0, U[2]: 0, U[3]: 0})["dev"]))
    vp = _vgpu_plugin(a, 0)
    assert H.plugin_nodes(off, vp) == {"path": "/dev/vfio/", "nodes": {}, "blockers": {}}
    off.close()

    hp = _plugin(kx, tree, True)
    b = hp.init()
    assert H.cdev_reads(hp) == 3  # the NVIDIA class's three mdevs
    assert b["mdevSnapshot"] == a["mdevSnapshot"] and b["mdevMap"] == a["mdevMap"] and b["plugins"] == a["plugins"]
    # the cdev class's spec names each mdev's node and leaves out U[3]; the other specs are byte-identical
    assert open(nv_file, "rb").read() == K.oracle_doc(K.FMT_YAML, b"nvidia.com/vgpu", _records(b, {U[1]: 7, U[2]: 8}))
    assert open(intel_file, "rb").read() == files_off[intel_file]
    assert open(pt_file, "rb").read() == files_off[pt_file]
    # U[3]'s group: Unhealthy with its reason, refused by Allocate and PrepareDraDevices, not in the pool
    assert vp == _vgpu_plugin(b, 0)
    assert viab_host.devs(hp, vp) == {"300": ("Healthy", None), "301": ("Healthy", None), "302": ("Healthy", WHY)}
    nodes = H.plugin_nodes(hp, vp)
    assert nodes["path"] == "/dev/vfio/devices/" and nodes["nodes"] == {"300": ["vfio7"], "301": ["vfio8"], "302": []}
    ip = _vgpu_plugin(b, 1)
    assert H.plugin_nodes(hp, ip) == {"path": "/dev/vfio/", "nodes": {}, "blockers": {}}
    with pytest.raises(RuntimeError, match="IOMMU group 302 is not viable: " + WHY):
        hp.allocate(["302"])
    assert hp.allocate(["300"])["cdi_devices"] == ["nvidia.com/vgpu=0"]
    blob = MH.slices(hp, 0)[0]
    assert b'"name":"vfio300"' in blob and b'"name":"vfio301"' in blob and b'"name":"vfio302"' not in blob
    with pytest.raises(RuntimeError, match="not viable: " + WHY):
        DH.prepare(hp, VDRV, "node-a", ["vfio302"])
    assert DH.prepare(hp, VDRV, "node-a", ["vfio301"]) == [["nvidia.com/vgpu=1"]]

    # a moved cdev: the live path refuses; rediscover keeps the index, rewrites the spec and lists the plugin
    H.set_vfio_dev(mbase, U[2], ["vfio12"])
    with pytest.raises(RuntimeError, match="the VFIO cdev of %s changed since discovery" % U[2]):
        hp.allocate(["301"])
    r = viab_host.rediscover(hp)
    assert r["mdevSnapshot"] == b["mdevSnapshot"]
    assert vp in r["report"]["changed"] and ip not in r["report"]["changed"]
    assert nv_file in r["report"]["written"] and intel_file not in r["report"]["written"]
    assert open(nv_file, "rb").read() == K.oracle_doc(K.FMT_YAML, b"nvidia.com/vgpu", _records(r, {U[1]: 7, U[2]: 12}))
    assert H.plugin_nodes(hp, vp)["nodes"]["301"] == ["vfio12"]
    assert hp.allocate(["301"])["cdi_devices"] == ["nvidia.com/vgpu=1"]
    snap = [s[4] for s in r["mdevSnapshot"]]
    hp.close()
    assert snap == [0, 1, 2, 3]

    # restart with resumeIndices and the setting off: the cdev spec is read with the group layout's parser; U[3], which
    # it left out, gets an index above every one named
    back = _plugin(kx, tree, False, resume=True)
    c = back.init()
    assert [s[4] for s in c["mdevSnapshot"]] == [0, 1, 4, 3]
    doc = open(nv_file, "rb").read()
    assert b"/dev/vfio/302\n" in doc and b"/dev/vfio/devices/" not in doc
    back.close()
    # and on again: the group-layout spec is read with the cdev layout's parser second
    on = _plugin(kx, tree, True, resume=True)
    d = on.init()
    assert [s[4] for s in d["mdevSnapshot"]] == [0, 1, 4, 3]
    assert b"/dev/vfio/devices/vfio12\n" in open(nv_file, "rb").read()
    on.close()
