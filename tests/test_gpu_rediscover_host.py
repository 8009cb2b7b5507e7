"""GPU end to end of Plugin::rediscover on fake PCI and mdev trees, through a sequence of changes.  After every step the
rediscovered state must equal a fresh start-up on the same tree (structure), pyref_reconcile over the previous snapshot
(indices), the oracle's CDI documents (rewritten only when they changed), the oracle's ListAndWatch bytes with health
carried over, and Allocate's answers; a HealthWatcher started before the changes keeps working and the snapshot
validation of Allocate is in use again after each rediscovery."""
import ctypes as C
import json
import os
import threading

import numpy as np
import pytest

import fake_mdev
import fake_sysfs
import pyref_reconcile as P
from oracle import mdev_oracle as mo
from oracle import oracle as O

pytestmark = pytest.mark.gpu

VGPU = [("10de", "vfio_mdev", "nvidia.com", "nvidia.com/vgpu", "cdi-mdev-nvidia")]
PCI = [dict(bdf="0000:3b:00.0", vendor=b"0x10de\n", device=b"0x1eb8\n", driver="nvidia", group=40),  # the vGPU parent
       dict(bdf="0000:c1:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=214),
       dict(bdf="0000:c5:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=215),
       dict(bdf="0000:3d:00.0", vendor=b"0x10de\n", device=b"0x20b5\n", driver="vfio-pci", group=75)]
U = ["%08x-0000-4000-8000-%012x" % (k, k) for k in range(16)]
MDEVS = [dict(uuid=U[1], parent="0000:3b:00.0", group=300), dict(uuid=U[2], parent="0000:3b:00.0", group=301)]


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


def add_mdev(root, m):
    pdir = os.path.join(root, "devices", m["parent"])
    target = os.path.join(pdir, m["uuid"])
    os.makedirs(target)
    os.symlink(os.path.join(pdir, "mdev_supported_types", "nvidia-222"), os.path.join(target, "mdev_type"))
    os.symlink(os.path.join(root, "drivers", "vfio_mdev"), os.path.join(target, "driver"))
    grp = os.path.join(root, "iommu_groups", str(m["group"]))
    os.makedirs(grp, exist_ok=True)
    os.symlink(grp, os.path.join(target, "iommu_group"))
    os.symlink(target, os.path.join(root, "bus", "mdev", "devices", m["uuid"]))


class Host(fake_sysfs.HostPlugin):
    def __init__(self, kx, root, pciids, cdi):
        super().__init__(kx, os.path.join(root, "bus", "pci", "devices"), pciids, cdi + "/")
        fake_mdev.set_vgpu(self, os.path.join(root, "bus", "mdev", "devices"), VGPU)
        L = self.L
        L.kxh_rediscover.restype = C.c_int
        L.kxh_rediscover.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_size_t]
        L.kxh_discovery_stale.restype = C.c_int
        L.kxh_discovery_stale.argtypes = [C.c_void_p]
        L.kxh_snapshot_enable.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.kxh_mdev_generation_seam.argtypes = [C.c_void_p, C.c_void_p]
        L.kxh_validation_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.kxh_set_device_path.argtypes = [C.c_void_p, C.c_int, C.c_char_p]
        L.kxh_health_resync.restype = C.c_int
        L.kxh_health_resync.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]

    def rediscover(self):
        buf = C.create_string_buffer(1 << 22)
        rc = self.L.kxh_rediscover(self.h, b"YAML", buf, len(buf))
        if rc < 0:
            raise RuntimeError(buf.value.decode())
        return json.loads(buf.value.decode())

    def counts(self):
        live, snap = C.c_uint64(), C.c_uint64()
        self.L.kxh_validation_counts(self.h, C.byref(live), C.byref(snap))
        return live.value, snap.value


def fresh(kx, root, pciids, tmp):
    cdi = os.path.join(tmp, "fresh-cdi")
    os.makedirs(cdi, exist_ok=True)
    h = Host(kx, root, pciids, cdi)
    st = h.init("YAML")
    h.close()
    return st


def snap_rows(s):
    return [(k.encode(), g, c, t, i) for k, g, c, t, i in s]


def structure(st):
    plugins = {(p["resource"], p["class"], p["vgpu"]): [d[0] for d in p["devs"]] for p in st["plugins"] if p["devs"]}
    return (
        [[g, [d[0] for d in devs]] for g, devs in st["iommuMap"]], st["deviceMap"],
        [[g, [d[0] for d in devs]] for g, devs in st["mdevMap"]], st["typeMap"], plugins)


def check_state(st, want, prev_pci, prev_pci_next, prev_mdev, prev_mdev_next):
    assert structure(st) == structure(want)
    for snap, prev, nxt, key in ((st["pciSnapshot"], prev_pci, prev_pci_next, "pciSnapshot"),
                                 (st["mdevSnapshot"], prev_mdev, prev_mdev_next, "mdevSnapshot")):
        exp = P.reconcile(snap_rows(prev), snap_rows(want[key]), nxt)
        assert [s[4] for s in snap] == exp["index"]
        assert [s[:4] for s in snap] == [s[:4] for s in want[key]]
    idx = {s[0]: s[4] for s in st["pciSnapshot"]}
    for g, devs in st["iommuMap"]:
        assert [d[1] for d in devs] == [idx[d[0]] for d in devs]
    midx = {s[0]: s[4] for s in st["mdevSnapshot"]}
    for g, devs in st["mdevMap"]:
        assert [d[2] for d in devs] == [midx[d[0]] for d in devs]


def expected_docs(st):
    devs = sorted(((d[0], int(g), d[1]) for g, ds in st["iommuMap"] for d in ds), key=lambda t: t[2])
    a = np.zeros(len(devs), O.CDIDEV_DTYPE)
    for k, (bdf, g, i) in enumerate(devs):
        a[k]["bdf"], a[k]["iommu_group"], a[k]["index"] = bdf.encode(), g, i
    md = sorted(((m[0], int(g), m[1], m[2]) for g, ms in st["mdevMap"] for m in ms), key=lambda t: t[3])
    b = np.zeros(len(md), mo.MDEVCDI_DTYPE)
    for k, (u, g, par, i) in enumerate(md):
        b[k] = (u.encode(), g, par.encode(), i)
    return {"cdi-vfio-xxxx.yaml": O.cdi_emit(0, a), "cdi-mdev-nvidia.yaml": mo.cdi_emit_mdev(0, VGPU[0][3].encode(), b)}


def test_rediscover_sequence(tmp_path, kx, pci_text):
    root, tmp = str(tmp_path), str(tmp_path)
    fake_sysfs.make_tree(root, PCI)
    fake_mdev.make_tree(root, MDEVS)
    pciids = str(tmp_path / "pci.ids")
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = str(tmp_path / "cdi")
    os.makedirs(cdi)
    h = Host(kx, root, pciids, cdi)
    gen, mgen = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    h.L.kxh_snapshot_enable(h.h, gen.ctypes.data, None)
    h.L.kxh_mdev_generation_seam(h.h, mgen.ctypes.data)
    st = h.init("YAML")
    assert [s[4] for s in st["pciSnapshot"]] == list(range(len(st["pciSnapshot"])))
    assert h.L.kxh_discovery_stale(h.h) == 0
    # a health watcher on the first plugin (the 0x2330 GPUs), started before any change
    vfio = tmp_path / "vfio"
    vfio.mkdir()
    for g in ("214", "215", "216", "75", "76", "77", "300", "301", "302"):
        (vfio / g).write_text("")
    p0 = [p["resource"] for p in st["plugins"]].index("nvidia.com/GH100_H100_SXM5_80GB")
    assert h.L.kxh_set_device_path(h.h, p0, (str(vfio) + "/").encode()) == 0
    err = C.create_string_buffer(512)
    w = h.L.kxh_health_start(h.h, p0, 0, err, len(err))
    assert w, err.value
    os.remove(vfio / "215")
    assert h.L.kxh_health_poll(w, 1000) == 1
    health = {"215": "Unhealthy"}

    old_names = {}  # group -> the Allocate answer while it existed

    def step_bind():
        add_pci(root, dict(bdf="0000:c2:00.0", vendor=b"0x10de\n", device=b"0x2330\n", driver="vfio-pci", group=216))
        add_pci(root, dict(bdf="0000:81:00.0", vendor=b"0x10de\n", device=b"0x2684\n", driver="vfio-pci", group=76))

    def step_unbind():
        relink(root, "0000:c5:00.0", "driver", os.path.join(root, "drivers", "nvidia"))

    def step_add_function():
        add_pci(root, dict(bdf="0000:3d:00.1", vendor=b"0x10de\n", device=b"0x1aef\n", driver="vfio-pci", group=75))

    def step_move_group():
        relink(root, "0000:81:00.0", "iommu_group", os.path.join(root, "iommu_groups", "77"))

    def step_swap_model():
        open(os.path.join(root, "devices", "0000:c2:00.0", "device"), "wb").write(b"0x2331\n")

    def step_mdev():
        add_mdev(root, dict(uuid=U[3], parent="0000:3b:00.0", group=302))
        os.unlink(os.path.join(root, "bus", "mdev", "devices", U[1]))

    steps = [("bind", step_bind, ["216", "76"], []), ("unbind", step_unbind, [], ["215"]),
             ("add_function", step_add_function, [], []), ("move_group", step_move_group, ["77"], ["76"]),
             ("swap_model", step_swap_model, [], []), ("mdev", step_mdev, ["302"], ["300"]), ("nothing", lambda: None, [], [])]
    docs = {f: open(os.path.join(cdi, f), "rb").read() for f in ("cdi-vfio-xxxx.yaml", "cdi-mdev-nvidia.yaml")}
    for g in ("214", "215", "75", "300"):
        old_names[g] = h.allocate([g])["cdi_devices"]
    for name, change, new_groups, gone_groups in steps:
        prev = st
        change()
        gen[0] += 1
        mgen[0] += name == "mdev"
        assert h.L.kxh_discovery_stale(h.h) == 1, name
        st = h.rediscover()
        assert h.L.kxh_discovery_stale(h.h) == 0, name
        want = fresh(kx, root, pciids, tmp)
        check_state(st, want, prev["pciSnapshot"], prev["pciNext"], prev["mdevSnapshot"], prev["mdevNext"])
        rep = st["report"]
        # CDI files: the oracle's documents of the reconciled devices, rewritten only when they changed
        exp = expected_docs(st)
        for f, doc in exp.items():
            assert open(os.path.join(cdi, f), "rb").read() == doc, (name, f)
            assert (os.path.join(cdi, f) in rep["written"]) == (doc != docs[f]), (name, f)
        docs = exp
        assert not [f for f in os.listdir(cdi) if f.endswith(".tmp")]
        if name == "nothing":
            assert rep["written"] == [] and rep["changed"] == [] and rep["added"] == []
            assert rep["pci"]["n_new"] == rep["pci"]["n_changed"] == rep["pci"]["n_retired"] == 0
        # ListAndWatch bytes with health carried over; added plugins were appended
        assert [p["resource"] for p in st["plugins"][:len(prev["plugins"])]] == [p["resource"] for p in prev["plugins"]]
        for k, p in enumerate(st["plugins"]):
            gids = np.array([int(d[0]) for d in p["devs"]], np.uint32)
            hl = np.array([health.get(d[0], "Healthy") == "Healthy" for d in p["devs"]], np.uint8)
            assert [d[1] for d in p["devs"]] == [health.get(d[0], "Healthy") for d in p["devs"]]
            assert h.list_and_watch(k) == O.lw_encode(gids, hl), (name, k)
        # Allocate: a retired group answers nothing, a new group its fresh name; served from the snapshot again
        before = h.counts()
        for g in gone_groups:
            assert h.allocate([g])["cdi_devices"] == [], (name, g)
        for g in new_groups:
            kind = "nvidia.com/vgpu" if g.startswith("30") else "nvidia.com/gpu"
            snap = st["mdevSnapshot"] if g.startswith("30") else st["pciSnapshot"]
            idx = sorted(s[4] for s in snap if str(s[1]) == g)
            got = h.allocate([g])["cdi_devices"]
            assert got == ["%s=%d" % (kind, i) for i in idx], (name, g)
            assert all(i >= prev["mdevNext" if g.startswith("30") else "pciNext"] for i in idx)
        for g, names in old_names.items():
            if any(str(s[1]) == g for s in st["pciSnapshot"] + st["mdevSnapshot"]) and g not in ("75",):
                assert h.allocate([g])["cdi_devices"] == names, (name, g)
        if h.allocate(["214"])["cdi_devices"]:
            assert h.counts()[1] > before[1], name  # snapshot validation in use again
    # the watcher started before the plugin-adding rediscoveries still flips health after a resync to the new list
    assert h.L.kxh_health_resync(w, err, len(err)) == 0, err.value
    os.remove(vfio / "214")
    assert h.L.kxh_health_poll(w, 1000) == 1
    devs = [p for p in h.rediscover()["plugins"] if p["resource"] == "nvidia.com/GH100_H100_SXM5_80GB"][0]["devs"]
    assert devs == [["214", "Unhealthy"]]
    h.L.kxh_health_stop(w)
    h.close()


def test_allocate_races_rediscover(tmp_path, kx, pci_text):
    """4 Allocate threads against 20 rediscoveries that alternately retire and re-add a GPU: every response is one of the
    answers the plugin gives with no rediscovery in flight."""
    root = str(tmp_path)
    fake_sysfs.make_tree(root, PCI)
    fake_mdev.make_tree(root, MDEVS)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    os.makedirs(str(tmp_path / "cdi"))
    h = Host(kx, root, str(tmp_path / "pci.ids"), str(tmp_path / "cdi"))
    h.init("YAML")
    stop, bad, seen = threading.Event(), [], []

    def worker():
        while not stop.is_set():
            try:
                r = tuple(h.allocate(["215", "214"])["cdi_devices"])
            except RuntimeError as e:  # pragma: no cover - reported below
                bad.append(str(e))
                return
            seen.append(r)

    answers = {tuple(h.allocate(["215", "214"])["cdi_devices"])}
    threads = [threading.Thread(target=worker) for _ in range(4)]
    for t in threads:
        t.start()
    try:
        for k in range(20):
            relink(root, "0000:c5:00.0", "driver", os.path.join(root, "drivers", "nvidia" if k % 2 == 0 else "vfio-pci"))
            h.rediscover()
            answers.add(tuple(h.allocate(["215", "214"])["cdi_devices"]))
    finally:
        stop.set()
        for t in threads:
            t.join()
    assert not bad, bad[:3]
    assert len(answers) == 12  # the start, 214 alone, and 215 with a fresh index each of the 10 times it came back
    assert seen and set(seen) <= answers, set(seen) - answers
    h.close()
