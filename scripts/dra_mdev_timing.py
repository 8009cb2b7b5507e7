"""Device and call time of kxpu_dra_slices_mdev (DESIGN.md K11, the vGPU layout) next to kxpu_dra_slices on the same
devices: 65 536 and 2^20 vGPUs with every optional attribute present (workloads.dra_mdev_devices; the passthrough
records carry the same group, parent as bdf, root, ids, NUMA mask and product), 40 alternating calls of each.  Kernel
times come from the library's per-stage CUDA events (KXPU_T_EMIT); a whole call is the host clock around one call with
an output buffer large enough (the call ends in a stream synchronisation).  Output bytes per second of kernel time are
printed against the 3.35 TB/s data-sheet HBM3 figure.  Prints the card and its power limit and one JSON object (also
written to argv[1] when given)."""
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

REPS = 40
HBM_BPS = 3.35e12  # H100 SXM data sheet, HBM3


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    t = {}
    for n in (1 << 16, 1 << 20):
        mdev = W.dra_mdev_devices(n)
        dra = np.zeros(n, B.DRADEV_DTYPE)
        for f in ("product", "pcie_root", "vendor", "device", "numa_mask", "iommu_group", "product_len"):
            dra[f] = mdev[f]
        dra["bdf"] = mdev["parent"]
        mdev_len = len(kx.dra_slices_mdev("vgpu.nvidia.com", "node-a", "node-a", 1, mdev)[0])
        dra_len = len(kx.dra_slices("vfio.nvidia.com", "node-a", "node-a", 1, dra)[0])
        out_m, out_d = np.empty(mdev_len, np.uint8), np.empty(dra_len, np.uint8)
        offs = np.empty(n // 128 + 2, np.uint64)
        ln, ns = C.c_size_t(0), C.c_size_t(0)

        def call_mdev():
            rc = kx.L.kxpu_dra_slices_mdev(kx.ctx, b"vgpu.nvidia.com", b"node-a", b"node-a", 1, mdev.ctypes.data, n,
                                           out_m.ctypes.data, mdev_len, C.byref(ln), offs.ctypes.data, C.byref(ns))
            assert rc == 0 and ln.value == mdev_len

        def call_dra():
            rc = kx.L.kxpu_dra_slices(kx.ctx, b"vfio.nvidia.com", b"node-a", b"node-a", 1, dra.ctypes.data, n,
                                      out_d.ctypes.data, dra_len, C.byref(ln), offs.ctypes.data, C.byref(ns))
            assert rc == 0 and ln.value == dra_len

        for _ in range(3):  # warm-up
            call_mdev(); call_dra()
        k_m, k_d, w_m, w_d = [], [], [], []
        for _ in range(REPS):
            for fn, k_ms, w_ms in ((call_mdev, k_m, w_m), (call_dra, k_d, w_d)):
                t0 = time.perf_counter()
                fn()
                w_ms.append((time.perf_counter() - t0) * 1e3)
                k_ms.append(kx.timings()[B.T_EMIT])
        for name, nbytes, k_ms, w_ms in (("dra_slices_mdev", mdev_len, k_m, w_m), ("dra_slices", dra_len, k_d, w_d)):
            bps = nbytes / (float(np.median(k_ms)) * 1e-3)
            t["%s_%d" % (name, n)] = {"kernel": stats(k_ms), "call": stats(w_ms), "out_bytes": nbytes,
                                      "out_bytes_per_s": round(bps / 1e9, 1), "share_of_3.35TBps": round(bps / HBM_BPS, 4)}
            print("%-22s n=%-8d kernel %.4f ms [%.4f, %.4f]  call %.3f ms  %d B  %.1f GB/s of kernel time (%.1f %% of 3.35 TB/s)"
                  % (name, n, np.median(k_ms), np.percentile(k_ms, 10), np.percentile(k_ms, 90), np.median(w_ms), nbytes,
                     bps / 1e9, 100 * bps / HBM_BPS))
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "timings": t}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
