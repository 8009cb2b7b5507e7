"""Helpers for the GPU host tests of Plugin::MetricsText: the host's counters as family 4, the expected device families of
a plugin state (kxh_init / kxh_state / kxh_rediscover JSON) built with tests/pyref_metrics.py, and the plugin's other
outputs, which a scrape must leave as they were."""
import ctypes as C
import difflib
import json
import os

import pyref_metrics as PM
from test_metrics import host_metrics


def _u64(hp, name):
    f = getattr(hp.L, name)
    f.restype, f.argtypes = C.c_uint64, [C.c_void_p]
    return f(hp.h)


def counters(hp):
    live, snap = C.c_uint64(0), C.c_uint64(0)
    hp.L.kxh_validation_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    hp.L.kxh_validation_counts(hp.h, C.byref(live), C.byref(snap))
    return PM.counters(aer=_u64(hp, "kxh_aer_reads"), cdev=_u64(hp, "kxh_cdev_reads"), sriov=_u64(hp, "kxh_sriov_reads"),
                       reset=_u64(hp, "kxh_reset_reads"), nvidia=_u64(hp, "kxh_vf_vgpu_reads"), live=live.value,
                       snapshot=snap.value)


def state(hp):
    hp.L.kxh_state.restype = C.c_int
    hp.L.kxh_state.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(1 << 22)
    assert hp.L.kxh_state(hp.h, buf, len(buf)) >= 0
    return json.loads(buf.value.decode())


def document(st, reasons=None, aer=None, missing=()):
    """families 1 to 3 of st's plugins.  reasons: group id -> [(kind, detail)]; aer: group id -> (fatal, nonfatal);
    missing: {(plugin index, group id)} the watcher flipped.  A group's address is its first member's bdf, or for a vGPU
    plugin its first mdev's UUID."""
    reasons, aer = reasons or {}, aer or {}
    first = {False: {g: m[0][0] for g, m in st["iommuMap"]}, True: {g: m[0][0] for g, m in st["mdevMap"]}}
    b = PM.Builder()
    for k, p in enumerate(st["plugins"]):
        for g, _ in p["devs"]:
            why = ([(0, b"")] if (k, g) in missing else []) + sorted(reasons.get(g, []))
            b.add(p["resource"].encode(), int(g), first[p["vgpu"]][g].encode(), int(not why), why,
                  *aer.get(g, (PM.METRICS_NO_VALUE,) * 2))
    return PM.document(*b.arrays())


def outputs(hp, cdi):
    """the CDI spec files, every plugin's ListAndWatch bytes and the counters"""
    specs = {f: open(os.path.join(cdi, f), "rb").read() for f in sorted(os.listdir(cdi))}
    return specs, [hp.list_and_watch(k) for k in range(len(state(hp)["plugins"]))], counters(hp)


def scrape(hp, cdi, want):
    """MetricsText is want plus the counters, twice, and leaves every other output as it was"""
    before = outputs(hp, cdi)
    got = host_metrics(hp)
    if got != want + counters(hp):  # this module's asserts are not rewritten by pytest: name the lines that differ
        raise AssertionError("\n".join(difflib.unified_diff((want + counters(hp)).decode().splitlines(),
                                                            got.decode().splitlines(), "want", "got", lineterm="")))
    if host_metrics(hp) != got or outputs(hp, cdi) != before:
        raise AssertionError("a scrape changed the next scrape or another output")
    return got
