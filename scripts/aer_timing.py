"""Kernel times of the PCIe AER health path (DESIGN.md K12).
  - kxpu_aer_health on 2^20 records in sysfs format (workloads.aer_records: one file pair per function, and vGPUs sharing
    their parent's files 16 to one), 40 calls: the two kernels' time under KXPU_T_CLASSIFY.
  - kxpu_dra_slices_taints / _mdev_taints against kxpu_dra_slices_taint / _mdev_taint on the same devices (every optional
    attribute present): 65 536 and 2^20 devices, 0 %, 1 % and 100 % of them tainted, tables of 1 and 3 entries (the
    3-entry table is the host's: vfio-device-missing, pcie-aer=fatal, pcie-aer=nonfatal, a device carrying the first
    and one of the other two), 40 calls of each, alternating; KXPU_T_EMIT.
Median [p10, p90].  Prints the card and its power limit, and one JSON object (also written to argv[1] when given), with
the SHA-256 of each taint call's output and slice offsets, so that two builds can be checked for identical bytes."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 40
SHARES = (0.0, 0.01, 1.0)
T3 = [(b"vfio.nvidia.com/unhealthy", b"vfio-device-missing", b"NoSchedule"),
      (b"vfio.nvidia.com/pcie-aer", b"fatal", b"NoSchedule"), (b"vfio.nvidia.com/pcie-aer", b"nonfatal", b"NoSchedule")]


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def digest(out, length, offs, n_slices):
    """SHA-256 of a call's output bytes and its slice offsets"""
    h = hashlib.sha256(memoryview(out[:length]))
    h.update(memoryview(offs[:n_slices + 1]))
    return h.hexdigest()


def since_of(n, share, k, seed=5):
    """[n, k] taint times: `share` of the devices tainted; with k = 3 a tainted device carries entry 0 and one of 1, 2"""
    rng = np.random.default_rng(seed)
    on = rng.random(n) < share if share < 1.0 else np.ones(n, bool)
    t = rng.integers(0, B.DRA_TAINT_SINCE_MAX + 1, (n, k), dtype=np.int64)
    s = np.where(on[:, None], t, -1)
    if k == 3:
        which = rng.integers(1, 3, n)
        s[np.arange(n), 3 - which] = -1
    return np.ascontiguousarray(s)


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "aer_health": {}, "taints": {}}
    for share in (0, 16):
        r = W.aer_records(1 << 20, vgpus_per_parent=share)
        for _ in range(3):
            kx.aer_health(r["text"], r["file_off"], r["file_len"], 0, 0, r["group_off"], r["group_members"])
        k = []
        for _ in range(REPS):
            kx.aer_health(r["text"], r["file_off"], r["file_len"], 0, 0, r["group_off"], r["group_members"])
            k.append(kx.timings()[B.T_CLASSIFY])
        name = "records_2^20_share%d" % share
        res["aer_health"][name] = dict(stats(k), text_bytes=len(r["text"]), groups=len(r["group_off"]) - 1)
        print("aer_health %s: %.4f ms [%.4f, %.4f], %d text bytes" % (name, np.median(k), np.percentile(k, 10),
                                                                      np.percentile(k, 90), len(r["text"])))
    for layout, devs_of, one, lst in (("pci", W.dra_devices, "kxpu_dra_slices_taint", "kxpu_dra_slices_taints"),
                                      ("mdev", W.dra_mdev_devices, "kxpu_dra_slices_mdev_taint", "kxpu_dra_slices_mdev_taints")):
        for n in (1 << 16, 1 << 20):
            devs = devs_of(n)
            ln, ns = C.c_size_t(0), C.c_size_t(0)
            offs = np.empty(n // 64 + 2, np.uint64)
            base = (kx.ctx, b"vfio.nvidia.com", b"node-a", b"node-a", 1, devs.ctypes.data, n)
            out = np.empty(n * 1600 + (1 << 20), np.uint8)
            for share in SHARES:
                for k in (1, 3):
                    since = since_of(n, share, k)
                    tab = (B.DraTaint * k)(*[B.DraTaint(*e) for e in T3[:k]])
                    s0 = np.ascontiguousarray(since[:, 0])

                    def call_one():
                        assert getattr(kx.L, one)(*base, T3[0][0], T3[0][1], T3[0][2], s0.ctypes.data, out.ctypes.data,
                                                  out.size, C.byref(ln), offs.ctypes.data, C.byref(ns)) == 0
                        return ln.value

                    def call_list():
                        assert getattr(kx.L, lst)(*base, C.cast(tab, C.c_void_p), k, since.ctypes.data, out.ctypes.data,
                                                  out.size, C.byref(ln), offs.ctypes.data, C.byref(ns)) == 0
                        return ln.value

                    for _ in range(3):
                        call_one(); call_list()
                    list_sha = digest(out, call_list(), offs, ns.value)
                    one_sha = digest(out, call_one(), offs, ns.value)
                    k_l, k_o = [], []
                    for _ in range(REPS):
                        list_len = call_list()
                        k_l.append(kx.timings()[B.T_EMIT])
                        one_len = call_one()
                        k_o.append(kx.timings()[B.T_EMIT])
                    name = "%s_%d_taint%g_entries%d" % (layout, n, 100 * share, k)
                    res["taints"][name] = {"taints_kernel": stats(k_l), "taint_kernel": stats(k_o),
                                           "taints_out_bytes": list_len, "taint_out_bytes": one_len,
                                           "taints_sha256": list_sha, "taint_sha256": one_sha,
                                           "ratio_median": round(float(np.median(k_l) / np.median(k_o)), 3)}
                    print("%-4s n=%-8d %5.1f %% tainted, %d entries: _taints %.4f ms [%.4f, %.4f] %d B | _taint %.4f ms "
                          "[%.4f, %.4f] %d B | x%.2f" % (layout, n, 100 * share, k, np.median(k_l), np.percentile(k_l, 10),
                                                         np.percentile(k_l, 90), list_len, np.median(k_o),
                                                         np.percentile(k_o, 10), np.percentile(k_o, 90), one_len,
                                                         np.median(k_l) / np.median(k_o)))
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
