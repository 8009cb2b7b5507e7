"""GPU end to end of Plugin::aerPortHealth on fake sysfs trees whose PCIe ports are entries with AER files of their own:
a downstream port's count flags the GPU below it only, a switch upstream port's every GPU below it, a sibling port's
nothing; the non-fatal limit; the reason text and order; the pcie-aer taint with a generation step; refreshAerHealth
reading each distinct port once; vGPUs on a PF and on its VF below the port; the start-up refusal without aerHealth; and,
with the setting off, the same bytes and counters whatever the ports' files say."""
import os

import pytest

import aer_host as AH
import aer_ports_host as H
import dra_host as DH
import fake_mdev
import fake_sysfs
from test_gpu_dra_taint_host import _lib as taint_lib
from test_metrics import host_metrics

pytestmark = pytest.mark.gpu
T0 = 1700000000
N_PORTS = 16  # per socket: two root ports, two switch upstream ports, four downstream ports above GPUs


def _reason(port, below, n, kind="fatal", limit=0):
    return "%s (PCIe port above %s) reported %d %s uncorrectable PCIe errors (limit %d)" % (port, below, n, kind, limit)


class Tree:
    def __init__(self, tmp_path, pci_text, with_mdevs=False):
        self.root = str(tmp_path / "sys")
        self.base, self.mbase = H.make_tree(self.root, with_mdevs)
        self.pciids = str(tmp_path / "pci.ids")
        open(self.pciids, "wb").write(pci_text)
        self.cdi = str(tmp_path / "cdi") + "/"
        os.makedirs(self.cdi)

    def write(self, bdf, **counts):
        AH.write(os.path.join(self.base, bdf), **counts)

    def plugin(self, kx, ports=True, aer=True, limits=(0, 0), dra=False, clock=None):
        hp = fake_sysfs.HostPlugin(kx, self.base, self.pciids, self.cdi)
        DH.configure(hp, classes=H.CLASS, dra=[H.DRIVER] if dra else None)
        if self.mbase:
            fake_mdev.set_vgpu(hp, self.mbase, H.VGPU)
        if dra:
            taint_lib().kxh_set_dra_taints(hp.h, 1)
            taint_lib().kxh_set_clock(hp.h, clock.ctypes.data)
        AH.enable(hp, aer, *limits)
        H.enable(hp, ports)
        return hp


@pytest.fixture
def tree(tmp_path, pci_text):
    return Tree(tmp_path, pci_text)


def _health(hp, state):
    """group -> (health, AER reason) over every plugin"""
    out = {}
    for k in range(len(state["plugins"])):
        why = AH.reasons(hp, k)
        for g, h in AH.health(hp, k).items():
            out[g] = (h, why.get(g, ""))
    return out


def _flagged(hp, state):
    return sorted(g for g, (h, _) in _health(hp, state).items() if h == "Unhealthy")


def test_downstream_port_flags_its_gpu_only(kx, tree):
    tree.write("0000:02:00.0", fatal=1)
    hp = tree.plugin(kx)
    try:
        state = hp.init("YAML")
        assert _flagged(hp, state) == ["10"]
        assert _health(hp, state)["10"] == ("Unhealthy", _reason("0000:02:00.0", "0000:03:00.0", 1))
    finally:
        hp.close()


def test_upstream_port_flags_every_gpu_below(kx, tree):
    tree.write("0000:81:00.0", fatal=2)
    hp = tree.plugin(kx)
    try:
        state = hp.init("YAML")
        assert _flagged(hp, state) == ["20", "21"]
        h = _health(hp, state)
        assert h["20"][1] == _reason("0000:81:00.0", "0000:83:00.0", 2)
        assert h["21"][1] == _reason("0000:81:00.0", "0000:84:00.0", 2)
    finally:
        hp.close()


def test_root_port_flags_its_subtree_and_a_sibling_nothing(kx, tree):
    tree.write(H.SIBLING[0], fatal=5)
    hp = tree.plugin(kx)
    try:
        state = hp.init("YAML")
        assert _flagged(hp, state) == []
        tree.write("0000:00:02.0", fatal=1)
        assert AH.refresh(hp)[0] != []
        assert _flagged(hp, state) == ["12", "13"]
    finally:
        hp.close()


def test_nonfatal_limit(kx, tree):
    tree.write("0000:80:01.0", nonfatal=3)
    tree.write("0000:86:01.0", nonfatal=2)
    hp = tree.plugin(kx, limits=(0, 2))
    try:
        state = hp.init("YAML")
        assert _flagged(hp, state) == ["20", "21"]
        assert _health(hp, state)["21"][1] == _reason("0000:80:01.0", "0000:84:00.0", 3, "non-fatal", 2)
    finally:
        hp.close()


def test_reason_order(kx, tree):
    tree.write("0000:03:00.0", nonfatal=1)  # the device's own non-fatal error: after every fatal one
    tree.write("0000:00:01.0", fatal=1)
    tree.write("0000:02:00.0", fatal=1)
    tree.write("0000:04:00.0", fatal=4)  # the device's own fatal error comes before its ports'
    tree.write("0000:02:01.0", fatal=1)
    hp = tree.plugin(kx)
    try:
        state = hp.init("YAML")
        h = _health(hp, state)
        assert h["10"][1] == _reason("0000:02:00.0", "0000:03:00.0", 1)  # nearest port first
        assert h["11"][1] == "0000:04:00.0 reported 4 fatal uncorrectable PCIe errors (limit 0)"
    finally:
        hp.close()


def test_taint_and_generation(kx, tree):
    import numpy as np
    clock = np.array([T0], np.int64)
    hp = tree.plugin(kx, dra=True, clock=clock)
    try:
        hp.init("YAML")
        gen = DH.generation(hp)
        assert b"pcie-aer" not in DH.slices(hp, 0)[0]
        tree.write("0000:06:01.0", fatal=1)
        clock[0] = T0 + 30
        assert AH.refresh(hp)[1] is True
        assert DH.generation(hp) == gen + 1
        blob = DH.slices(hp, 0)[0]
        assert blob.count(b'{"key":"%s/pcie-aer","value":"fatal","effect":"NoSchedule"' % H.DRIVER.encode()) == 1
    finally:
        hp.close()


def test_refresh_reads_each_port_once(kx, tree):
    hp = tree.plugin(kx)
    try:
        state = hp.init("YAML")
        r0 = AH.reads(hp)
        assert r0 == 2 * (8 + N_PORTS)
        assert AH.refresh(hp) == ([], False, False)
        assert AH.reads(hp) - r0 == 2 * (8 + N_PORTS)
        tree.write("0000:85:00.0", nonfatal=7)  # moved since the walk: picked up without one
        changed, _, _ = AH.refresh(hp)
        assert changed and _flagged(hp, state) == ["22", "23"]
        assert AH.reads(hp) - r0 == 4 * (8 + N_PORTS)
    finally:
        hp.close()


def test_vgpus_below_the_port(kx, tmp_path, pci_text):
    t = Tree(tmp_path, pci_text, with_mdevs=True)
    t.write("0000:11:00.0", fatal=1)
    hp = t.plugin(kx)
    try:
        state = hp.init("YAML")
        h = _health(hp, state)
        assert sorted(g for g, (x, _) in h.items() if x == "Unhealthy") == ["500", "501"]
        assert h["500"][1] == _reason("0000:11:00.0", "0000:13:00.0", 1)
        assert h["501"][1] == _reason("0000:11:00.0", "0000:13:00.4", 1)
    finally:
        hp.close()


def test_refused_without_aer_health(kx, tree):
    hp = tree.plugin(kx, aer=False)
    try:
        assert DH.initiate(hp) == "aerPortHealth is set but aerHealth is off"
    finally:
        hp.close()


def _outputs(hp, state, cdi, dra):
    specs = {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}
    return (specs, [hp.list_and_watch(k) for k in range(len(state["plugins"]))], DH.slices(hp, 0)[0] if dra else None,
            host_metrics(hp), AH.reads(hp))


@pytest.mark.parametrize("dra", [False, True])
def test_off_is_unchanged(kx, tmp_path, pci_text, dra):
    """the setting off on a tree whose ports report errors gives the bytes and counters of a tree whose ports do not;
    without a setting that reads entry links, none is read"""
    import numpy as np
    clock = np.array([T0], np.int64)
    got = []
    for k, errors in enumerate((False, True)):
        t = Tree(tmp_path / str(k), pci_text, with_mdevs=True)
        if errors:
            for port in ("0000:00:01.0", "0000:81:00.0", "0000:02:00.0", "0000:11:00.0"):
                t.write(port, fatal=3, nonfatal=3)
        hp = t.plugin(kx, ports=False, dra=dra, clock=clock)
        try:
            count = DH.Counter(hp)
            state = hp.init("YAML")
            AH.refresh(hp)
            got.append(_outputs(hp, state, t.cdi, dra) + (count.reads(),))
        finally:
            hp.close()
    assert got[0] == got[1]
    assert got[0][4] == 2 * 2 * (8 + 2)  # start-up and one refresh: the GPUs' and the vGPU parents' files only
    if not dra:
        assert got[0][5][1] == 0  # no entry link read
