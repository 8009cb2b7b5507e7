"""GPU end to end of Plugin::draVgpuPcie on a fake tree: an mdev pool on two H100s below different switches (the first
one's vGPUs on its VFs), a VF-vGPU class whose GPU sits below the first switch, and a NIC VF class below the same switch,
each class with its own DRA driver.  With the setting the vGPU, VF-vGPU and NIC-VF pools publish equal pcieSwitch
values exactly where they share a switch, and the other attributes are those without it; the physfn attributes follow
vgpuSriovAware; with the setting off every pool's bytes, generation and read counter are those of a plugin without it;
a rediscovery that moves an mdev's parent GPU under another switch, or an mdev to another parent, moves
draVgpuGeneration() and not draGeneration(); one that moves the VF-vGPU's GPU moves draGeneration() and not
draVgpuGeneration()."""
import ctypes as C
import os

import pytest

import dra_host as DH
import dra_mdev_host as MH
import dra_pcie_host as PCH
import dra_vf_vgpu_host as DVH
import fake_mdev
import fake_sysfs
import mdev_pf_host as MPH
import pcie_mdev_host as PMH
import sriov_host as SH
import vf_vgpu_host as VVH

pytestmark = pytest.mark.gpu

CLASSES = "15b3,vfio-pci,mellanox.com,mellanox.com/nic,cdi-vfio-nic;" + VVH.VGPU  # class 1 serves vGPUs on VFs
VGPU = [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/mdev-vgpu", "cdi-mdev-nvidia")]  # a kind of its own
NIC_DRV, VF_DRV, MDEV_DRV = "nic.example.com", "vgpu-vf.example.com", "vgpu.example.com"
DOMAIN = PCH.DOMAIN
RP, SW = PCH.RP, PCH.SW
SW0 = "pci0000:00/0000:00:01.0/0000:01:00.0"        # root port 0000:00:01.0, switch 0000:01:00.0
SW1 = "pci0000:80/0000:80:01.0/0000:81:00.0"        # root port 0000:80:01.0, switch 0000:81:00.0
SW2 = "pci0000:80/0000:80:02.0/0000:85:00.0"        # socket 1's second switch
SW3 = "pci0000:00/0000:00:02.0/0000:11:00.0"        # socket 0's second switch
PF_A, VF_A = "0000:03:00.0", ["0000:03:00.4", "0000:03:00.5"]
PF_B = "0000:83:00.0"
PF_C, VF_C = "0000:05:00.0", ["0000:05:00.1", "0000:05:00.2"]
NIC = "0000:0a:00.1"
MDEV_PARENT = dict(vendor=b"0x10de\n", driver="nvidia-vgpu-host", numa=b"0\n")
PARENTS = [
    dict(bdf=PF_A, group=30, path=SW0 + "/0000:02:00.0/" + PF_A, device=b"0x2330\n", **MDEV_PARENT),
    dict(bdf=VF_A[0], group=34, path=SW0 + "/0000:02:00.0/" + VF_A[0], device=b"0x2331\n", **MDEV_PARENT),
    dict(bdf=VF_A[1], group=35, path=SW0 + "/0000:02:00.0/" + VF_A[1], device=b"0x2331\n", **MDEV_PARENT),
    dict(bdf=PF_B, group=38, path=SW1 + "/0000:82:00.0/" + PF_B, device=b"0x2330\n", **dict(MDEV_PARENT, numa=b"1\n")),
    dict(bdf=PF_C, group=50, path=SW0 + "/0000:02:01.0/" + PF_C, vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia",
         numa=b"0\n"),
    dict(bdf=VF_C[0], group=51, path=SW0 + "/0000:02:01.0/" + VF_C[0], vendor=b"0x10de\n", device=b"0x2331\n",
         driver="nvidia", numa=b"0\n"),
    dict(bdf=VF_C[1], group=52, path=SW0 + "/0000:02:01.0/" + VF_C[1], vendor=b"0x10de\n", device=b"0x2331\n",
         driver="nvidia", numa=b"0\n"),
    dict(bdf=NIC, group=71, path=SW0 + "/0000:02:02.0/" + NIC, vendor=b"0x15b3\n", device=b"0x101e\n", driver="vfio-pci",
         numa=b"0\n"),
]
U = ["5c0ffee0-6e2c-4a55-9d41-%012x" % k for k in range(4)]
MDEVS = [dict(uuid=U[0], parent=VF_A[0], group=300), dict(uuid=U[1], parent=VF_A[1], group=301),
         dict(uuid=U[2], parent=PF_B, group=302), dict(uuid=U[3], parent=PF_B, group=303)]
FIRST = ("0000:00:01.0", "0000:01:00.0")
SECOND = ("0000:80:01.0", "0000:81:00.0")


@pytest.fixture
def tree(tmp_path, pci_text):
    root = str(tmp_path)
    base, mbase = MH.make_tree(root, PARENTS, MDEVS)
    SH.link_vfs(base, PF_A, VF_A, b"2\n")
    SH.link_vfs(base, PF_C, VF_C, b"2\n")
    VVH.set_files(base, VF_C[0], b"557\n", VVH.HEADER)
    VVH.set_files(base, VF_C[1], b"0\n", VVH.HEADER + b"557   : NVIDIA H100-4C\n")
    (tmp_path / "pci.ids").write_bytes(pci_text)
    (tmp_path / "cdi").mkdir()
    return root, base, mbase, str(tmp_path / "pci.ids"), str(tmp_path / "cdi") + "/"


def _plugin(kx, tree, domain=None, on=False, sriov=True):
    root, base, mbase, pciids, cdi = tree
    for f in os.listdir(cdi):
        os.remove(os.path.join(cdi, f))
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    assert hp.L.kxh_set_classes(hp.h, CLASSES.encode()) == 0
    VVH.set_vf_vgpu(hp, 1)
    DH.configure(hp, dra=[NIC_DRV, ""])
    DVH.set_driver(hp, 1, VF_DRV)
    fake_mdev.set_vgpu(hp, mbase, VGPU)
    MH.set_vgpu_dra(hp, [MDEV_DRV], "node-a")
    MPH.enable(hp, sriov)
    if domain is not None:
        PCH.set_domain(hp, domain)
    hp.L.kxh_set_dra_vgpu_pcie.argtypes = [C.c_void_p, C.c_int]
    hp.L.kxh_set_dra_vgpu_pcie(hp.h, int(on))
    return hp


def _outputs(hp):
    return dict(mdev=MH.slices(hp, 0), vf=DVH.slices(hp, 1), nic=DH.slices(hp, 0), gen=DH.generation(hp),
                vgen=MH.generation(hp))


def _run(kx, tree, **kw):
    hp = _plugin(kx, tree, **kw)
    counter = DH.Counter(hp)
    try:
        hp.init("YAML")
        out = _outputs(hp)
        out["reads"] = (counter.reads(), MPH.reads(hp), VVH.reads(hp))
        return out
    finally:
        hp.close()


def _same(a, b):
    assert a[0] == b[0] and list(a[1]) == list(b[1])


def _ports(blob, name):
    a = PCH.devices_of(blob)[name]["attributes"]
    return (a[RP]["string"] if RP in a else None, a[SW]["string"] if SW in a else None)


def _without_ports(blob):
    return {n: {k: v for k, v in d["attributes"].items() if k not in (RP, SW)} for n, d in PCH.devices_of(blob).items()}


def test_off_changes_nothing(kx, tree):
    unset, off = _run(kx, tree), _run(kx, tree, domain=DOMAIN)
    for k in ("mdev", "vf"):
        _same(unset[k], off[k])
    assert (unset["gen"], unset["vgen"], unset["reads"]) == (off["gen"], off["vgen"], off["reads"])
    assert not any(RP in d["attributes"] for d in PCH.devices_of(off["mdev"][0]).values())
    assert not any(RP in d["attributes"] for d in PCH.devices_of(off["vf"][0]).values())


def test_pools_share_switches(kx, tree):
    off, on = _run(kx, tree, domain=DOMAIN), _run(kx, tree, domain=DOMAIN, on=True)
    assert (on["gen"], on["vgen"], on["reads"]) == (off["gen"], off["vgen"], off["reads"])  # no new read
    _same(on["nic"], off["nic"])
    mdev, vf, nic = on["mdev"][0], on["vf"][0], on["nic"][0]
    assert set(PCH.devices_of(mdev)) == {"vfio300", "vfio301", "vfio302", "vfio303"}
    assert set(PCH.devices_of(vf)) == {"vfio51"} and set(PCH.devices_of(nic)) == {"vfio71"}
    want = {"vfio300": FIRST, "vfio301": FIRST, "vfio302": SECOND, "vfio303": SECOND}
    assert {n: _ports(mdev, n) for n in want} == want
    assert _ports(vf, "vfio51") == FIRST and _ports(nic, "vfio71") == FIRST
    # the vGPUs on the first GPU's VFs, the VF-vGPU and the NIC VF share one switch; the second GPU's do not
    sw = {n: _ports(b, n)[1] for b, names in ((mdev, want), (vf, ["vfio51"]), (nic, ["vfio71"])) for n in names}
    assert {n for n, s in sw.items() if s == sw["vfio71"]} == {"vfio300", "vfio301", "vfio51", "vfio71"}
    assert _without_ports(mdev) == _without_ports(off["mdev"][0])
    assert _without_ports(vf) == _without_ports(off["vf"][0])
    a = PCH.devices_of(mdev)["vfio300"]["attributes"]
    assert a["physfnAddress"] == {"string": PF_A} and a["productName"] == PCH.devices_of(off["mdev"][0])["vfio300"][
        "attributes"]["productName"]


def test_physfn_only_with_sriov(kx, tree):
    on = _run(kx, tree, domain=DOMAIN, on=True, sriov=False)
    plain = _run(kx, tree, sriov=False)
    assert not any("physfnAddress" in d["attributes"] for d in PCH.devices_of(on["mdev"][0]).values())
    assert _without_ports(on["mdev"][0]) == _without_ports(plain["mdev"][0])
    assert _ports(on["mdev"][0], "vfio300") == FIRST


def _move_dir(root, old, new, bdfs=(), uuids=()):
    """devices/<old> moves to devices/<new> with everything below it: the PCI links of bdfs, the mdev links of uuids and
    each mdev's mdev_type link follow it"""
    src, dst = os.path.join(root, "devices", old), os.path.join(root, "devices", new)
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    os.rename(src, dst)
    for bdf in bdfs:
        link = os.path.join(root, "bus", "pci", "devices", bdf)
        rel = os.readlink(link).replace("devices/" + old, "devices/" + new)
        os.remove(link)
        os.symlink(rel, link)
    for u in uuids:
        link = os.path.join(root, "bus", "mdev", "devices", u)
        rel = os.readlink(link).replace("devices/" + old, "devices/" + new)
        os.remove(link)
        os.symlink(rel, link)
        mt = os.path.join(root, os.path.normpath(os.path.join("bus", "mdev", "devices", rel)), "mdev_type")
        t = os.readlink(mt).replace(src, dst)
        os.remove(mt)
        os.symlink(t, mt)


def test_rediscover_mdev(kx, tree):
    root = tree[0]
    hp = _plugin(kx, tree, domain=DOMAIN, on=True)
    try:
        hp.init("YAML")
        gen, vgen, blob = DH.generation(hp), MH.generation(hp), MH.slices(hp, 0)[0]
        DH.rediscover(hp)  # nothing changed: same bytes, same generations
        assert (DH.generation(hp), MH.generation(hp), MH.slices(hp, 0)[0]) == (gen, vgen, blob)
        # the second GPU moves below socket 1's second switch, its mdevs with it: only their ports change
        _move_dir(root, SW1 + "/0000:82:00.0", SW2 + "/0000:86:00.0", [PF_B], [U[2], U[3]])
        DH.rediscover(hp)
        assert (DH.generation(hp), MH.generation(hp)) == (gen, vgen + 1)
        after = MH.slices(hp, 0)[0]
        assert _ports(after, "vfio302") == ("0000:80:02.0", "0000:85:00.0")
        assert _without_ports(after) == _without_ports(blob)
        # an mdev moves to the first GPU (another parent): its ports follow
        PMH.move(root, U[3], SW2 + "/0000:86:00.0/" + PF_B, SW0 + "/0000:02:00.0/" + PF_A)
        DH.rediscover(hp)
        assert (DH.generation(hp), MH.generation(hp)) == (gen, vgen + 2)
        assert _ports(MH.slices(hp, 0)[0], "vfio303") == FIRST
    finally:
        hp.close()
    # without the setting the GPU's move changes nothing the vGPU pool publishes: no generation moves
    _move_dir(root, SW2 + "/0000:86:00.0", SW1 + "/0000:82:00.0", [PF_B], [U[2]])
    hp = _plugin(kx, tree, domain=DOMAIN)
    try:
        hp.init("YAML")
        gen, vgen = DH.generation(hp), MH.generation(hp)
        _move_dir(root, SW1 + "/0000:82:00.0", SW2 + "/0000:86:00.0", [PF_B], [U[2]])
        DH.rediscover(hp)
        assert (DH.generation(hp), MH.generation(hp)) == (gen, vgen)
    finally:
        hp.close()


def test_rediscover_vf_vgpu(kx, tree):
    root = tree[0]
    hp = _plugin(kx, tree, domain=DOMAIN, on=True)
    try:
        hp.init("YAML")
        gen, vgen, blob = DH.generation(hp), MH.generation(hp), DVH.slices(hp, 1)[0]
        assert _ports(blob, "vfio51") == FIRST
        # the VF-vGPU's GPU and its VFs move below socket 0's second switch: the PCI walk's ports comparison covers
        # its group, so draGeneration() moves and draVgpuGeneration() does not
        _move_dir(root, SW0 + "/0000:02:01.0", SW3 + "/0000:12:01.0", [PF_C] + VF_C)
        DH.rediscover(hp)
        assert (DH.generation(hp), MH.generation(hp)) == (gen + 1, vgen)
        after = DVH.slices(hp, 1)[0]
        assert _ports(after, "vfio51") == ("0000:00:02.0", "0000:11:00.0")
        assert _without_ports(after) == _without_ports(blob)
        DH.rediscover(hp)
        assert (DH.generation(hp), MH.generation(hp)) == (gen + 1, vgen)
    finally:
        hp.close()
