"""GPU end to end of Plugin::resumeIndices on fake PCI and mdev trees: two Plugin objects share one cdiConfigPath, the
second one standing for the restarted process.  A restart keeps the CDI index of every function and vGPU that is still
there, hands every other one an index above everything handed out before, rewrites no file when nothing changed, and
falls back to fresh numbering when a previous spec cannot be trusted.  With resumeIndices off nothing changes."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import fake_mdev
import fake_sysfs
from oracle import mdev_oracle as mo
from oracle import oracle as O

pytestmark = pytest.mark.gpu

VGPU = [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")]
A, B, Cf, D = "0000:01:00.0", "0000:02:00.0", "0000:03:00.0", "0000:04:00.0"
PARENT = dict(bdf="0000:3b:00.0", vendor=b"0x10de\n", device=b"0x1eb8\n", driver="nvidia", group=40)
U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(16)]
SPEC, MSPEC, STATE = "cdi-vfio-xxxx.yaml", "cdi-mdev-nvidia.yaml", ".kata-xpu-cdi-index"


def gpu(bdf, group):
    return dict(bdf=bdf, vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=group)


def add_pci(root, d):
    real = os.path.join(root, "devices", d["bdf"])
    os.makedirs(real)
    open(os.path.join(real, "vendor"), "wb").write(d["vendor"])
    open(os.path.join(real, "device"), "wb").write(d["device"])
    for link, target in (("driver", os.path.join(root, "drivers", d["driver"])),
                         ("iommu_group", os.path.join(root, "iommu_groups", str(d["group"])))):
        os.makedirs(target, exist_ok=True)
        os.symlink(target, os.path.join(real, link))
    os.symlink(real, os.path.join(root, "bus", "pci", "devices", d["bdf"]))


def relink(root, bdf, link, target):
    p = os.path.join(root, "devices", bdf, link)
    os.makedirs(target, exist_ok=True)
    os.unlink(p)
    os.symlink(target, p)


def add_mdev(root, uuid, group):
    pdir = os.path.join(root, "devices", PARENT["bdf"])
    target = os.path.join(pdir, uuid)
    os.makedirs(target)
    tdir = os.path.join(pdir, "mdev_supported_types", "nvidia-222")
    os.makedirs(tdir, exist_ok=True)
    open(os.path.join(tdir, "name"), "wb").write(b"GRID T4-1Q\n")
    os.symlink(tdir, os.path.join(target, "mdev_type"))
    os.symlink(os.path.join(root, "drivers", "vfio_mdev"), os.path.join(target, "driver"))
    grp = os.path.join(root, "iommu_groups", str(group))
    os.makedirs(grp, exist_ok=True)
    os.symlink(grp, os.path.join(target, "iommu_group"))
    os.symlink(target, os.path.join(root, "bus", "mdev", "devices", uuid))


def del_mdev(root, uuid):
    os.unlink(os.path.join(root, "bus", "mdev", "devices", uuid))


class Host(fake_sysfs.HostPlugin):
    def __init__(self, kx, root, pciids, cdi, resume=True, vgpu=False):
        super().__init__(kx, os.path.join(root, "bus", "pci", "devices"), pciids, cdi + "/")
        if vgpu:
            fake_mdev.set_vgpu(self, os.path.join(root, "bus", "mdev", "devices"), VGPU)
        L = self.L
        L.kxh_set_resume.argtypes = [C.c_void_p, C.c_int]
        L.kxh_initiate.restype = C.c_int
        L.kxh_initiate.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        L.kxh_state.restype = C.c_int
        L.kxh_state.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        L.kxh_rediscover.restype = C.c_int
        L.kxh_rediscover.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_size_t]
        L.kxh_set_resume(self.h, int(resume))

    def start(self):
        buf = C.create_string_buffer(1 << 22)
        if self.L.kxh_initiate(self.h, buf, len(buf)) < 0:
            raise RuntimeError(buf.value.decode())
        assert self.L.kxh_state(self.h, buf, len(buf)) >= 0
        return json.loads(buf.value.decode())

    def rediscover(self):
        buf = C.create_string_buffer(1 << 22)
        if self.L.kxh_rediscover(self.h, b"YAML", buf, len(buf)) < 0:
            raise RuntimeError(buf.value.decode())
        return json.loads(buf.value.decode())


@pytest.fixture
def env(tmp_path, kx, pci_text):
    root = str(tmp_path / "sys")
    fake_sysfs.make_tree(root, [PARENT, gpu(A, 10), gpu(B, 11), gpu(Cf, 12)])
    fake_mdev.make_tree(root, [])
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = str(tmp_path / "cdi")
    os.makedirs(cdi)
    hosts = []

    def new(resume=True, vgpu=False):
        h = Host(kx, root, str(tmp_path / "pci.ids"), cdi, resume, vgpu)
        hosts.append(h)
        return h

    yield dict(root=root, cdi=cdi, new=new)
    for h in hosts:
        h.close()


def pci_index(st):
    return {s[0]: s[4] for s in st["pciSnapshot"]}


def mdev_index(st):
    return {s[0]: s[4] for s in st["mdevSnapshot"]}


def file_id(path):
    s = os.stat(path)
    return s.st_ino, open(path, "rb").read()


def spec_doc(devs):
    """The oracle's PCI spec of [(bdf, group, index)] in the given order."""
    a = np.zeros(len(devs), O.CDIDEV_DTYPE)
    for k, (bdf, g, i) in enumerate(devs):
        a[k]["bdf"], a[k]["iommu_group"], a[k]["index"] = bdf.encode(), g, i
    return O.cdi_emit(0, a)


def retire_a(env):
    """A, B, C start as 0, 1, 2; A is unbound and a rediscovery leaves B = 1, C = 2."""
    h = env["new"]()
    st = h.start()
    assert pci_index(st) == {A: 0, B: 1, Cf: 2}
    relink(env["root"], A, "driver", os.path.join(env["root"], "drivers", "nvidia"))
    st = h.rediscover()
    assert pci_index(st) == {B: 1, Cf: 2} and st["pciNext"] == 3
    assert h.allocate(["11"])["cdi_devices"] == ["nvidia.com/gpu=1"]
    assert open(os.path.join(env["cdi"], STATE), "rb").read() == b"pci 3\nmdev 0\n"
    return h


def test_restart_keeps_indices(env):
    retire_a(env)
    before = {f: file_id(os.path.join(env["cdi"], f)) for f in (SPEC, STATE)}
    st = env["new"]().start()
    assert pci_index(st) == {B: 1, Cf: 2} and st["pciNext"] == 3
    r = st["resume"]
    assert r["pci"]["fallback"] == "" and r["pci"]["n_kept"] == 2 and r["pci"]["n_new"] == 0
    assert r["pci"]["files"] == [os.path.join(env["cdi"], SPEC)] and r["stateRead"] and r["statePci"] == 3
    assert r["written"] == []
    assert {f: file_id(os.path.join(env["cdi"], f)) for f in (SPEC, STATE)} == before  # same inode, same bytes
    h2 = env["new"]()
    h2.start()
    assert h2.allocate(["11"])["cdi_devices"] == ["nvidia.com/gpu=1"]
    assert h2.allocate(["12"])["cdi_devices"] == ["nvidia.com/gpu=2"]
    # without resume the restarted plugin numbers by walk order: the container holding gpu=1 would get C
    st = env["new"](resume=False).start()
    assert pci_index(st) == {B: 0, Cf: 1}


def test_added_and_moved_get_fresh_indices(env):
    retire_a(env)
    add_pci(env["root"], gpu(D, 13))  # added while the plugin was down
    relink(env["root"], Cf, "iommu_group", os.path.join(env["root"], "iommu_groups", "22"))  # C's group changed
    st = env["new"]().start()
    idx = pci_index(st)
    assert idx[B] == 1
    assert sorted((idx[Cf], idx[D])) == [3, 4] and st["pciNext"] == 5
    assert st["resume"]["pci"]["n_changed"] == 1 and st["resume"]["pci"]["n_new"] == 1
    assert open(os.path.join(env["cdi"], STATE), "rb").read() == b"pci 5\nmdev 0\n"
    assert open(os.path.join(env["cdi"], SPEC), "rb").read() == spec_doc(sorted(
        [(B, 11, 1), (Cf, 22, idx[Cf]), (D, 13, idx[D])], key=lambda t: t[2]))


def test_retired_top_index_is_not_reused(env):
    h = env["new"]()
    h.start()
    relink(env["root"], Cf, "driver", os.path.join(env["root"], "drivers", "nvidia"))  # C (index 2) leaves
    assert pci_index(h.rediscover()) == {A: 0, B: 1}
    relink(env["root"], Cf, "driver", os.path.join(env["root"], "drivers", "vfio-pci"))  # back while the plugin is down
    st = env["new"]().start()
    assert pci_index(st) == {A: 0, B: 1, Cf: 3}  # the specs alone would say 2 is free; the state file says it is not


def test_vgpu_churn_keeps_survivors(env):
    root = env["root"]
    for k in (1, 2, 3):
        add_mdev(root, U[k], 300 + k)
    h = env["new"](vgpu=True)
    assert mdev_index(h.start()) == {U[1]: 0, U[2]: 1, U[3]: 2}
    del_mdev(root, U[1])
    add_mdev(root, U[4], 304)
    assert mdev_index(h.rediscover()) == {U[2]: 1, U[3]: 2, U[4]: 3}
    del_mdev(root, U[2])  # while the plugin is down
    add_mdev(root, U[5], 305)
    st = env["new"](vgpu=True).start()
    assert mdev_index(st) == {U[3]: 2, U[4]: 3, U[5]: 4} and st["mdevNext"] == 5
    assert st["resume"]["mdev"]["n_kept"] == 2 and st["resume"]["mdev"]["fallback"] == ""
    assert pci_index(st) == {A: 0, B: 1, Cf: 2}
    h2 = env["new"](vgpu=True)
    h2.start()
    assert h2.allocate(["303"])["cdi_devices"] == ["nvidia.com/vgpu=2"]
    md = sorted([(U[3], 303, 2), (U[4], 304, 3), (U[5], 305, 4)], key=lambda t: t[2])
    b = np.zeros(len(md), mo.MDEVCDI_DTYPE)
    for k, (u, g, i) in enumerate(md):
        b[k] = (u.encode(), g, PARENT["bdf"].encode(), i)
    assert open(os.path.join(env["cdi"], MSPEC), "rb").read() == mo.cdi_emit_mdev(0, b"nvidia.com/vgpu", b)


def test_corrupt_spec_falls_back(env):
    retire_a(env)
    path = os.path.join(env["cdi"], SPEC)
    doc = bytearray(open(path, "rb").read())
    doc[-20] ^= 0x01
    open(path, "wb").write(bytes(doc))
    st = env["new"]().start()
    assert SPEC in st["resume"]["pci"]["fallback"]
    assert pci_index(st) == {B: 3, Cf: 4}  # fresh, above the state file's 3
    open(path, "wb").write(bytes(doc))
    os.remove(os.path.join(env["cdi"], STATE))
    st = env["new"]().start()
    assert SPEC in st["resume"]["pci"]["fallback"] and not st["resume"]["stateRead"]
    assert pci_index(st) == {B: 0, Cf: 1}  # corrupt and no state file: walk order


def test_repeated_index_falls_back(env):
    retire_a(env)
    open(os.path.join(env["cdi"], SPEC), "wb").write(spec_doc([(B, 11, 1), (Cf, 12, 1)]))
    st = env["new"]().start()
    assert "named twice" in st["resume"]["pci"]["fallback"]
    assert pci_index(st) == {B: 3, Cf: 4}


def test_spec_in_another_order_is_accepted(env):
    retire_a(env)
    path = os.path.join(env["cdi"], SPEC)
    open(path, "wb").write(spec_doc([(Cf, 12, 2), (B, 11, 1)]))  # Go's map order
    st = env["new"]().start()
    assert pci_index(st) == {B: 1, Cf: 2} and st["resume"]["pci"]["fallback"] == ""
    assert open(path, "rb").read() == spec_doc([(B, 11, 1), (Cf, 12, 2)])  # rewritten in ascending index
    assert path in st["resume"]["written"]


def test_off_changes_nothing(env):
    h = env["new"](resume=False, vgpu=True)
    add_mdev(env["root"], U[1], 301)
    st = h.start()
    assert pci_index(st) == {A: 0, B: 1, Cf: 2} and mdev_index(st) == {U[1]: 0}
    assert open(os.path.join(env["cdi"], SPEC), "rb").read() == spec_doc([(A, 10, 0), (B, 11, 1), (Cf, 12, 2)])
    relink(env["root"], A, "driver", os.path.join(env["root"], "drivers", "nvidia"))
    h.rediscover()
    assert not os.path.exists(os.path.join(env["cdi"], STATE))
    st = env["new"](resume=False, vgpu=True).start()
    assert pci_index(st) == {B: 0, Cf: 1} and st["resume"]["pci"]["files"] == []
    assert not os.path.exists(os.path.join(env["cdi"], STATE))
    assert sorted(os.listdir(env["cdi"])) == sorted([SPEC, MSPEC])
