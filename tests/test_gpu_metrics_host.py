"""GPU end to end of Plugin::MetricsText on the fake sysfs tree of the reset tests, with viability, reset checks, PCIe AER
health and a health watcher on: each check shows up as its reason sample (two on one device, in kind order), the AER
maxima as samples, a reason cleared by rediscover leaves no sample, and scrapes change no other output or counter."""
import ctypes as C
import json
import os

import pytest

import aer_host as AH
import dra_host as DH
import pyref_metrics as PM
import reset_host as H
import sriov_host
import viab_host
from test_gpu_dra_taint_host import Watched
from test_gpu_reset_host import DEVS, WHY, _plugin, tree  # noqa: F401
from test_metrics import host_metrics

pytestmark = pytest.mark.gpu

NOT_VIABLE = {"41": "0000:41:00.1 is bound to snd_hda_intel"}


def _counters(hp):
    live, snap = C.c_uint64(0), C.c_uint64(0)
    hp.L.kxh_validation_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    hp.L.kxh_validation_counts(hp.h, C.byref(live), C.byref(snap))
    return PM.counters(aer=AH.reads(hp), reset=H.reads(hp), live=live.value, snapshot=snap.value)


def _outputs(hp, tree):
    cdi = tree[3]
    specs = {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}
    hp.L.kxh_state.restype = C.c_int
    hp.L.kxh_state.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(1 << 20)
    assert hp.L.kxh_state(hp.h, buf, len(buf)) >= 0
    n = len(json.loads(buf.value.decode())["plugins"])
    blob, off = DH.slices(hp, 0)
    return (specs, [hp.list_and_watch(k) for k in range(n)], bytes(blob), [int(x) for x in off], DH.generation(hp),
            AH.reads(hp), H.reads(hp))


def _scrape(hp, tree, want):
    """MetricsText equals want, and leaves every other output and counter as it was"""
    before = _outputs(hp, tree)
    got = host_metrics(hp)
    assert got == want[0] + _counters(hp)
    assert host_metrics(hp) == got
    assert _outputs(hp, tree) == before


def test_metrics_flow(kx, tree, tmp_path):
    root, base = tree[0], tree[1]
    for d in DEVS:
        AH.write(os.path.join(base, d["bdf"]))
    AH.write(os.path.join(base, "0000:61:00.0"), fatal=2, nonfatal=1)
    AH.write(os.path.join(base, "0000:62:00.1"), nonfatal=9)
    hp = _plugin(kx, tree, True)
    DH.configure(hp, dra=["gpu.nvidia.com"], viability=True)
    AH.enable(hp, True, 0, 10)
    try:
        state = hp.init("YAML")
        assert [g for g, _ in state["plugins"][0]["devs"]] == ["5", "41", "42", "61", "62"]
        reasons = {g: [(4, WHY[g].encode())] for g in WHY}
        reasons["41"] = [(1, NOT_VIABLE["41"].encode()), (4, WHY["41"].encode())]  # both checks, in kind order
        reasons["61"] = [(5, b"0000:61:00.0 reported 2 fatal uncorrectable PCIe errors (limit 0)")]
        aer = {g: (0, 0) for g in ("5", "41", "42")}
        aer["61"], aer["62"] = (2, 1), (0, 9)  # the group's highest count of each severity over its members
        doc = PM.document(*_build(state, reasons, aer))
        _scrape(hp, tree, (doc,))
        # the watcher: device 62 of the first plugin loses its node
        w = Watched(hp, tmp_path, 0, [g for g, _ in state["plugins"][0]["devs"]])
        try:
            w.remove("62")
            _scrape(hp, tree, (PM.document(*_build(state, reasons, aer, missing={(0, "62")})),))
            w.create("62")
        finally:
            w.stop()
        # the audio function rebound to vfio-pci: group 41 is viable and can be reset, so its two samples go
        sriov_host.rebind(root, base, "0000:41:00.1", "vfio-pci")
        AH.write(os.path.join(base, "0000:41:00.1"))
        r = viab_host.rediscover(hp)
        del reasons["41"]
        _scrape(hp, tree, (PM.document(*_build(r, reasons, aer)),))
    finally:
        hp.close()


def _build(state, reasons, aer, missing=()):
    first = {g: m[0][0] for g, m in state["iommuMap"]}
    b = PM.Builder()
    for k, p in enumerate(state["plugins"]):
        for g, _ in p["devs"]:
            why = ([(0, b"")] if (k, g) in missing else []) + reasons.get(g, [])
            b.add(p["resource"].encode(), int(g), first[g].encode(), int(not why), why,
                  *aer.get(g, (PM.METRICS_NO_VALUE,) * 2))
    return b.arrays()
