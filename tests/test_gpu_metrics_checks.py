"""GPU host flows of Plugin::MetricsText for the checks the reset tree does not have: a VFIO cdev blocker, SR-IOV as the
blocker and as a second reason behind a viability or cdev blocker, a VF whose vGPU type drifted, a vGPU (mdev) plugin
with its parent's AER counts, and a tree with no reason at all.  rediscover reports the same changedPlugins, and every
output is the same, whether or not MetricsText was called in between."""
import os

import pytest

import aer_host as AH
import cdev_host as CH
import dra_host as DH
import fake_mdev
import fake_sysfs
import metrics_host as M
import sriov_host as SH
import vf_vgpu_host as VG
import viab_host
from test_gpu_dra_mdev_host import MDEVS, PARENTS, VGPU
from test_gpu_dra_taint_host import mdev_tree  # noqa: F401
from test_gpu_vf_vgpu_health_host import VFS, _health_plugin, _start, refresh, tree  # noqa: F401

pytestmark = pytest.mark.gpu

GPU = dict(vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci")
VF = dict(vendor=b"0x10de\n", device=b"0x2331\n", driver="vfio-pci")
DEVS = [dict(bdf="0000:01:00.0", group=40, **GPU),                                                   # PF, 1 VF on
        dict(bdf="0000:01:00.1", group=40, vendor=b"0x10de\n", device=b"0x22a3\n", driver="snd_hda_intel"),
        dict(bdf="0000:01:10.0", group=45, **VF),
        dict(bdf="0000:02:00.0", group=41, **GPU),                                                   # served
        dict(bdf="0000:03:00.0", group=42, **GPU),                                                   # PF, no cdev
        dict(bdf="0000:03:10.0", group=46, **VF)]
CDEVS = {"0000:01:00.0": 3, "0000:01:00.1": 4, "0000:01:10.0": 7, "0000:02:00.0": 5, "0000:03:10.0": 8}
SNDS = b"0000:01:00.1 is bound to snd_hda_intel"
PF40, PF42 = b"0000:01:00.0 has 1 VFs enabled", b"0000:03:00.0 has 1 VFs enabled"
REASONS = {"40": [(1, SNDS), (3, PF40)],                                   # viability, then SR-IOV behind it
           "45": [(3, b"0000:01:10.0 needs the VF token of 0000:01:00.0 (bound to vfio-pci)")],
           "42": [(2, b"0000:03:00.0 has no VFIO cdev"), (3, PF42)],       # a cdev blocker, then SR-IOV behind it
           "46": [(3, b"0000:03:10.0 needs the VF token of 0000:03:00.0 (bound to vfio-pci)")]}


@pytest.fixture
def sriov_tree(tmp_path, pci_text):
    root = str(tmp_path)
    base = fake_sysfs.make_tree(root, DEVS)
    for bdf, n in CDEVS.items():
        CH.set_vfio_dev(base, bdf, ["vfio%d" % n])
    SH.link_vfs(base, "0000:01:00.0", ["0000:01:10.0"], b"1\n")
    SH.link_vfs(base, "0000:03:00.0", ["0000:03:10.0"], b"1\n")
    (tmp_path / "pci.ids").write_bytes(pci_text)
    return root, base, str(tmp_path / "pci.ids")


def _sriov_plugin(kx, t, cdi):
    root, base, pciids = t
    os.makedirs(cdi, exist_ok=True)
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    assert hp.L.kxh_set_classes(hp.h, CH.spec([CH.NV_CDEV])) == 0
    viab_host.set_viability(hp, True)
    SH.set_sriov(hp, True)
    return hp


def _report(r):
    """a rediscover report without the spec files' paths, which name each plugin's own CDI directory"""
    return {k: v for k, v in r["report"].items() if "file" not in k.lower() and "written" not in k.lower()}


def test_cdev_and_sriov_reasons(kx, sriov_tree, tmp_path):
    root, base, _ = sriov_tree
    cdi_a, cdi_b = str(tmp_path / "cdi_a") + "/", str(tmp_path / "cdi_b") + "/"
    a, b = _sriov_plugin(kx, sriov_tree, cdi_a), _sriov_plugin(kx, sriov_tree, cdi_b)  # b is never scraped
    try:
        st = a.init("YAML")
        assert b.init("YAML")["plugins"] == st["plugins"]
        assert "41" in [g for p in st["plugins"] for g, _ in p["devs"]]
        M.scrape(a, cdi_a, M.document(st, REASONS))
        # the audio function rebound to vfio-pci (it has a cdev): group 40 is viable, and SR-IOV becomes its blocker
        SH.rebind(root, base, "0000:01:00.1", "vfio-pci")
        ra, rb = viab_host.rediscover(a), viab_host.rediscover(b)
        assert _report(ra) == _report(rb) and ra["report"]["changed"]
        reasons = dict(REASONS, **{"40": [(3, PF40)]})
        M.scrape(a, cdi_a, M.document(ra, reasons))
        # the PF's VFs off: group 40 is served; its VF still needs the token of a PF on vfio-pci
        open(os.path.join(os.path.realpath(os.path.join(base, "0000:01:00.0")), "sriov_numvfs"), "wb").write(b"0\n")
        ra, rb = viab_host.rediscover(a), viab_host.rediscover(b)
        assert _report(ra) == _report(rb) and ra["report"]["changed"]
        reasons = {g: r for g, r in reasons.items() if g != "40"}
        M.scrape(a, cdi_a, M.document(ra, reasons))
        assert M.outputs(a, cdi_a)[1] == M.outputs(b, cdi_b)[1]  # ListAndWatch of every plugin, scraped or not
        assert M.counters(a) == M.counters(b)
        assert {f: open(cdi_a + f, "rb").read() for f in os.listdir(cdi_a)} == \
               {f: open(cdi_b + f, "rb").read() for f in os.listdir(cdi_b)}
    finally:
        a.close()
        b.close()


def test_no_reason_then_vgpu_type_drift(kx, tree):  # noqa: F811
    base, cdi = tree[1], tree[3]
    hp = _health_plugin(kx, tree)
    try:
        st = _start(hp)
        doc = M.document(st)
        assert b"unhealthy_reason" not in doc and b"aer_errors" not in doc  # only the families that have samples
        M.scrape(hp, cdi, doc)
        VG.set_files(base, VFS[0], b"0\n")
        refresh(hp)
        drifted = {"31": [(6, b"0000:03:00.1 now carries vGPU type 0 (was 557)")]}
        M.scrape(hp, cdi, M.document(st, drifted))
        VG.set_files(base, VFS[0], b"557\n")
        refresh(hp)
        M.scrape(hp, cdi, doc)
    finally:
        hp.close()


def test_vgpu_plugin(kx, mdev_tree, tmp_path):  # noqa: F811
    root, base, mbase, pciids, cdi = mdev_tree
    parents = [p["bdf"] for p in PARENTS if os.path.isdir(os.path.join(base, p["bdf"]))]
    for p in parents:
        AH.write(os.path.join(base, p), fatal=1 if p == "0000:c1:00.0" else 0, nonfatal=4 if p == "0000:41:00.0" else 0)
    hp = fake_sysfs.HostPlugin(kx, base, pciids, cdi)
    try:
        DH.configure(hp, node="node-a")
        fake_mdev.set_vgpu(hp, mbase, VGPU)
        AH.enable(hp, True, 0, 10)
        st = hp.init("YAML")
        assert any(p["vgpu"] for p in st["plugins"])
        served = {g for p in st["plugins"] if p["vgpu"] for g, _ in p["devs"]}
        parent = {str(m["group"]): m["parent"] for m in MDEVS}
        aer = {g: ((1 if parent[g] == "0000:c1:00.0" else 0), (4 if parent[g] == "0000:41:00.0" else 0))
               for g in served if parent[g] in parents}
        reasons = {g: [(5, b"0000:c1:00.0 reported 1 fatal uncorrectable PCIe errors (limit 0)")]
                   for g in served if parent[g] == "0000:c1:00.0"}
        assert reasons and aer
        members = dict((g, [m[0] for m in ms]) for g, ms in st["iommuMap"])
        passthrough = {g for p in st["plugins"] if not p["vgpu"] for g, _ in p["devs"]}
        aer.update({g: (0, 0) for g in passthrough if all(b in parents for b in members[g])})  # passthrough files: 0
        M.scrape(hp, cdi, M.document(st, reasons, aer))
        # the counters reset: the reason goes, the counts stay as samples
        AH.write(os.path.join(base, "0000:c1:00.0"))
        AH.refresh(hp)
        aer = {g: (0, v[1]) for g, v in aer.items()}
        M.scrape(hp, cdi, M.document(st, {}, aer))
    finally:
        hp.close()

