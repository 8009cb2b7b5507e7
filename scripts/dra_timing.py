"""Device and call time of kxpu_dra_slices (DESIGN.md K11) next to kxpu_cdi_emit_kind JSON on the same devices: 65 536
and 2^20 devices with every optional attribute present (workloads.dra_devices), 40 alternating calls of each.  Kernel
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
    kind = b"nvidia.com/gpu"
    t = {}
    for n in (1 << 16, 1 << 20):
        dra = W.dra_devices(n)
        cdi = np.zeros(n, B.CDIDEV_DTYPE)
        cdi["bdf"], cdi["iommu_group"], cdi["index"] = dra["bdf"], dra["iommu_group"], np.arange(n)
        dra_len = len(kx.dra_slices("vfio.nvidia.com", "node-a", "node-a", 1, dra)[0])
        cdi_len = len(kx.cdi_emit(B.FMT_JSON, cdi, kind))
        out_d, out_c = np.empty(dra_len, np.uint8), np.empty(cdi_len, np.uint8)
        offs = np.empty(n // 128 + 2, np.uint64)
        ln, ns = C.c_size_t(0), C.c_size_t(0)

        def call_dra():
            rc = kx.L.kxpu_dra_slices(kx.ctx, b"vfio.nvidia.com", b"node-a", b"node-a", 1, dra.ctypes.data, n,
                                      out_d.ctypes.data, dra_len, C.byref(ln), offs.ctypes.data, C.byref(ns))
            assert rc == 0 and ln.value == dra_len

        def call_cdi():
            rc = kx.L.kxpu_cdi_emit_kind(kx.ctx, B.FMT_JSON, kind, cdi.ctypes.data, n, out_c.ctypes.data, cdi_len, C.byref(ln))
            assert rc == 0 and ln.value == cdi_len

        for _ in range(3):  # warm-up
            call_dra(); call_cdi()
        k_d, k_c, w_d, w_c = [], [], [], []
        for _ in range(REPS):
            for fn, k_ms, w_ms in ((call_dra, k_d, w_d), (call_cdi, k_c, w_c)):
                t0 = time.perf_counter()
                fn()
                w_ms.append((time.perf_counter() - t0) * 1e3)
                k_ms.append(kx.timings()[B.T_EMIT])
        for name, nbytes, k_ms, w_ms in (("dra_slices", dra_len, k_d, w_d), ("cdi_emit_kind_json", cdi_len, k_c, w_c)):
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
