"""GPU end to end of restart resume (Plugin::resumeIndices) for a class that serves vGPUs on SR-IOV VFs
(XpuClass::vfVgpu), on test_gpu_vf_vgpu_host.py's fake tree: a PF on the vGPU manager's driver and eight VFs, three of
type 557, two of type 558 and three free ones that list both names.  With resume on, the class's spec carries each VF's
type ID and key; a restart on the full GPU learns the names back from it and keeps every index; a VF whose type changed
while the plugin was down gets a fresh index; a spec written with resume off is resumed under the tag-0 rule and
rewritten typed; a rediscover right after a resumed start-up changes nothing.  The same with vfioCdev.  With resume off,
the spec is kxpu_cdi_emit_kind's (or kxpu_cdi_emit_cdev's) document."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import cdev_host as CH
import dra_host as DH
import fake_sysfs
import sriov_host as SH
import vf_vgpu_host as H
from kxpu_b200 import binding as B

pytestmark = pytest.mark.gpu

VF = dict(vendor=b"0x10de\n", device=b"0x2331\n", driver="nvidia")
PF = "0000:03:00.0"
VFS = ["0000:03:00.%d" % k for k in range(1, 8)] + ["0000:03:01.0"]
GROUP = {PF: 30, **{bdf: 31 + k for k, bdf in enumerate(VFS)}}
TYPE = {VFS[0]: 557, VFS[1]: 557, VFS[2]: 557, VFS[3]: 558, VFS[4]: 558}  # VFS[5:] are free
LIST = H.HEADER + b"557   : NVIDIA H100-4C\n558   : NVIDIA H100-8C\n"
A, Bk = "NVIDIA_H100-4C", "NVIDIA_H100-8C"
KIND = "nvidia.com/vgpu"
SPEC = "cdi-vgpu-vf.yaml"


@pytest.fixture
def tree(tmp_path, pci_text):
    devs = [dict(bdf=PF, group=30, vendor=b"0x10de\n", device=b"0x2330\n", driver="nvidia")]
    devs += [dict(bdf=bdf, group=GROUP[bdf], **VF) for bdf in VFS]
    base = fake_sysfs.make_tree(str(tmp_path), devs)
    SH.link_vfs(base, PF, VFS, b"8\n")
    for k, bdf in enumerate([PF] + VFS):
        CH.set_vfio_dev(base, bdf, ["vfio%d" % (200 + k)])
    for bdf in VFS:
        t = TYPE.get(bdf, 0)
        H.set_files(base, bdf, b"%d\n" % t, H.HEADER if t else LIST)
    (tmp_path / "pci.ids").write_bytes(pci_text)
    cdi = tmp_path / "cdi"
    cdi.mkdir()
    return str(tmp_path), base, str(tmp_path / "pci.ids"), str(cdi) + "/"


class Plugin(fake_sysfs.HostPlugin):
    def __init__(self, kx, tree, cdev, resume=True):
        root, base, pciids, cdi = tree
        super().__init__(kx, base, pciids, cdi)
        classes = H.CLASSES + (",cdev" if cdev else "")
        assert self.L.kxh_set_classes(self.h, classes.encode()) == 0
        H.set_vf_vgpu(self, 1, True)
        self.L.kxh_set_resume.argtypes = [C.c_void_p, C.c_int]
        self.L.kxh_set_resume(self.h, int(resume))

    def start(self):
        """InitiateDevicePlugin (the start-up that resumes and writes the state file and the specs), then the state"""
        L = self.L
        L.kxh_initiate.restype = C.c_int
        L.kxh_initiate.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        L.kxh_state.restype = C.c_int
        L.kxh_state.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        buf = C.create_string_buffer(1 << 22)
        if L.kxh_initiate(self.h, buf, len(buf)) < 0:
            raise RuntimeError(buf.value.decode())
        assert L.kxh_state(self.h, buf, len(buf)) >= 0
        self.state = json.loads(buf.value.decode())
        return self.state

    def resume_report(self):
        return self.state["resume"]


def _start(kx, tree, cdev, resume=True):
    hp = Plugin(kx, tree, cdev, resume)
    try:
        return hp, hp.start()
    except BaseException:
        hp.close()
        raise


def _vgpu_plugins(state):
    """{type key: {group id: CDI index}} of the vGPU class's plugins"""
    index = {str(g): ms[0][1] for g, ms in state["iommuMap"]}
    return {p["name"]: {d[0]: index[d[0]] for d in p["devs"]} for p in state["plugins"]
            if p["resource"].startswith("nvidia.com/NVIDIA_H100")}


def _spec(tree):
    return open(os.path.join(tree[3], SPEC), "rb").read()


def _records(kx, tree, cdev):
    return kx.cdi_parse_vf_vgpu(B.FMT_YAML, _spec(tree), KIND, cdev=cdev)


def _types(recs):
    """{group: (type ID, key, index)} of parsed typed records"""
    return {int(r["dev"]["iommu_group"]): (int(r["type_id"]), bytes(r["key"])[:int(r["key_len"])].decode(),
                                           int(r["dev"]["index"])) for r in recs}


@pytest.mark.parametrize("cdev", [False, True])
def test_restart_on_full_gpu_and_type_change(kx, tree, cdev):
    root, base = tree[0], tree[1]
    hp, state = _start(kx, tree, cdev)
    try:
        first = _vgpu_plugins(state)
        assert sorted(first) == [A, Bk] and set(first[A]) == {"31", "32", "33"} and set(first[Bk]) == {"34", "35"}
        spec = _spec(tree)
        assert spec.count(b'      vgpu-type: "557"\n      vgpu-type-key: "NVIDIA_H100-4C"\n') == 3
        assert spec.count(b'      vgpu-type: "558"\n      vgpu-type-key: "NVIDIA_H100-8C"\n') == 2
        want = {31 + k: (TYPE[bdf], A if TYPE[bdf] == 557 else Bk, first[A if TYPE[bdf] == 557 else Bk][str(31 + k)])
                for k, bdf in enumerate(VFS[:5])}
        assert _types(_records(kx, tree, cdev)) == want
        if cdev:
            assert all(int(r["dev"]["reserved"]) == 200 + int(r["dev"]["iommu_group"]) - 30 for r in _records(kx, tree, cdev))
    finally:
        hp.close()
    # the GPU fills up while no plugin runs: the free VFs take type 557 and no list names a type any more
    for bdf in VFS[5:]:
        H.set_files(base, bdf, b"557\n")
    for bdf in VFS:
        H.set_files(base, bdf, creatable=H.HEADER)
    hp, state = _start(kx, tree, cdev)  # no vgpuTypeNames: the names come from the spec
    try:
        second = _vgpu_plugins(state)
        assert set(second[A]) == {"31", "32", "33", "36", "37", "38"} and set(second[Bk]) == {"34", "35"}
        for key in (A, Bk):
            for g, i in first[key].items():
                assert second[key][g] == i
        old_max = max(i for p in first.values() for i in p.values())
        assert min(second[A][g] for g in ("36", "37", "38")) > old_max
        assert H.learned(hp) == {557: A, 558: Bk}
        rep = hp.resume_report()["pci"]
        assert rep["fallback"] == "" and rep["typed"] == [1]
        assert (rep["n_kept"], rep["n_new"], rep["n_changed"]) == (5, 3, 0)
        assert len(_records(kx, tree, cdev)) == 8
        # a rediscover right after the resumed start-up: nothing changed, nothing written
        st = DH.rediscover(hp)
        assert (st["report"]["pci"]["n_changed"], st["report"]["pci"]["n_new"], st["report"]["pci"]["n_retired"]) == (0, 0, 0)
        assert st["report"]["written"] == []
        second_max = max(i for p in second.values() for i in p.values())
    finally:
        hp.close()
    # VF 31 moves from 557 to 558 while no plugin runs: a fresh index, and its old name leaves the spec
    H.set_files(base, VFS[0], b"558\n")
    hp, state = _start(kx, tree, cdev)
    try:
        third = _vgpu_plugins(state)
        assert set(third[A]) == {"32", "33", "36", "37", "38"} and set(third[Bk]) == {"31", "34", "35"}
        assert third[Bk]["31"] > second_max
        rep = hp.resume_report()["pci"]
        assert rep["fallback"] == "" and rep["n_changed"] == 1
        spec = _spec(tree)
        assert b"nvidia.com/vgpu=%d\n" % second[A]["31"] not in spec
        assert b"nvidia.com/vgpu=%d\n" % third[Bk]["31"] in spec
        assert _types(_records(kx, tree, cdev))[31] == (558, Bk, third[Bk]["31"])
        assert hp.allocate(["31"])["cdi_devices"] == ["nvidia.com/vgpu=%d" % third[Bk]["31"]]
    finally:
        hp.close()


def _plain_doc(kx, state, cdev):
    """kxpu_cdi_emit_kind's (cdev: kxpu_cdi_emit_cdev's) document of the served VFs, in ascending index"""
    index = {g: i for p in _vgpu_plugins(state).values() for g, i in p.items()}
    recs = np.zeros(len(index), B.CDIDEV_DTYPE)
    for k, (g, i) in enumerate(sorted(index.items(), key=lambda kv: kv[1])):
        recs[k]["bdf"], recs[k]["iommu_group"], recs[k]["index"] = VFS[int(g) - 31].encode(), int(g), i
        recs[k][B.CDEV_FIELD] = 200 + int(g) - 30
    return kx.cdi_emit_cdev(B.FMT_YAML, recs, KIND) if cdev else kx.cdi_emit(B.FMT_YAML, recs, KIND)


@pytest.mark.parametrize("cdev", [False, True])
def test_resume_from_a_plain_spec(kx, tree, cdev):
    hp, state = _start(kx, tree, cdev, resume=False)
    try:
        first = _vgpu_plugins(state)
        spec = _spec(tree)
        assert b"vgpu-type" not in spec
        assert spec == _plain_doc(kx, state, cdev)  # resume off: the untyped layout, byte for byte
    finally:
        hp.close()
    hp, state = _start(kx, tree, cdev)
    try:
        assert _vgpu_plugins(state) == first  # the tag-0 rule keeps every index
        rep = hp.resume_report()
        assert rep["pci"]["fallback"] == "" and rep["pci"]["typed"] == []
        assert (rep["pci"]["n_kept"], rep["pci"]["n_new"], rep["pci"]["n_changed"]) == (5, 0, 0)
        assert any(f.endswith(SPEC) for f in rep["written"])  # rewritten in the typed layout
        assert b'vgpu-type: "557"' in _spec(tree)
    finally:
        hp.close()
    hp, state = _start(kx, tree, cdev)
    try:
        assert _vgpu_plugins(state) == first
        rep = hp.resume_report()
        assert rep["pci"]["typed"] == [1] and rep["pci"]["n_kept"] == 5
        assert not any(f.endswith(SPEC) for f in rep["written"])
    finally:
        hp.close()
