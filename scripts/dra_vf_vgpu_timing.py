"""Device and call time of kxpu_dra_slices_vf_vgpu (DESIGN.md K11, the VF-vGPU layout) next to kxpu_dra_slices_taints
and kxpu_dra_slices_mdev_taints on the same count: 65 536 and 2^20 devices with every optional attribute present
(workloads.dra_vf_vgpu_devices / dra_mdev_devices, and passthrough records carrying the same group, bdf, root, ids, NUMA
mask and product), untainted (taint_since NULL) and with every device carrying the first entry of the host's table.
The three calls alternate, 30 times each per case.  Kernel times come from the library's per-stage CUDA events
(KXPU_T_EMIT); a whole call is the host clock around one call with an output buffer large enough (the call ends in a
stream synchronisation).  Prints the card and its power limit and one JSON object (also written to argv[1] when
given)."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 30
T0 = 1767225600  # 2026-01-01T00:00:00Z


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    tab = (B.DraTaint * 1)(B.DraTaint(b"x.nvidia.com/unhealthy", b"vfio-device-missing", b"NoSchedule"))
    t = {}
    for n in (1 << 16, 1 << 20):
        vf = W.dra_vf_vgpu_devices(n)
        mdev = W.dra_mdev_devices(n)
        dra = np.zeros(n, B.DRADEV_DTYPE)
        for f in ("product", "bdf", "pcie_root", "vendor", "device", "numa_mask", "iommu_group", "product_len"):
            dra[f] = vf[f]
        layouts = (("dra_slices_vf_vgpu", kx.L.kxpu_dra_slices_vf_vgpu, vf),
                   ("dra_slices_taints", kx.L.kxpu_dra_slices_taints, dra),
                   ("dra_slices_mdev_taints", kx.L.kxpu_dra_slices_mdev_taints, mdev))
        for tainted in (False, True):
            since = np.full(n, T0, np.int64) if tainted else None
            sp = None if since is None else since.ctypes.data
            calls = []
            for name, fn, devs in layouts:
                ln, ns = C.c_size_t(0), C.c_size_t(0)
                rc = fn(kx.ctx, b"x.nvidia.com", b"node-a", b"node-a", 1, devs.ctypes.data, n, C.cast(tab, C.c_void_p), 1,
                        sp, None, 0, C.byref(ln), None, C.byref(ns))
                assert rc == B.E_NOSPACE, rc
                out, offs = np.empty(ln.value, np.uint8), np.empty(ns.value + 1, np.uint64)

                def call(fn=fn, devs=devs, out=out, offs=offs, need=ln.value):
                    got, s = C.c_size_t(0), C.c_size_t(0)
                    rc = fn(kx.ctx, b"x.nvidia.com", b"node-a", b"node-a", 1, devs.ctypes.data, n, C.cast(tab, C.c_void_p),
                            1, sp, out.ctypes.data, need, C.byref(got), offs.ctypes.data, C.byref(s))
                    assert rc == 0 and got.value == need
                calls.append((name, call, ln.value, [], []))
            for _ in range(3):  # warm-up
                for c in calls:
                    c[1]()
            for _ in range(REPS):
                for name, call, nbytes, k_ms, w_ms in calls:
                    t0 = time.perf_counter()
                    call()
                    w_ms.append((time.perf_counter() - t0) * 1e3)
                    k_ms.append(kx.timings()[B.T_EMIT])
            for name, call, nbytes, k_ms, w_ms in calls:
                key = "%s_%d_%s" % (name, n, "tainted" if tainted else "untainted")
                bps = nbytes / (float(np.median(k_ms)) * 1e-3)
                t[key] = {"kernel": stats(k_ms), "call": stats(w_ms), "out_bytes": nbytes,
                          "out_GB_per_s_of_kernel_time": round(bps / 1e9, 1)}
                print("%-24s n=%-8d %-9s kernel %.4f ms [%.4f, %.4f]  call %.3f ms  %d B  %.1f GB/s"
                      % (name, n, "tainted" if tainted else "untainted", np.median(k_ms), np.percentile(k_ms, 10),
                         np.percentile(k_ms, 90), np.median(w_ms), nbytes, bps / 1e9))
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "timings": t}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
