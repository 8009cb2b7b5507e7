"""Kernel time of kxpu_dra_slices_taint / kxpu_dra_slices_mdev_taint (DESIGN.md K11, taints) against the untainted
kxpu_dra_slices / kxpu_dra_slices_mdev on the same records: 65 536 and 2^20 devices of both layouts with every optional
attribute present (workloads.dra_devices / dra_mdev_devices), 0 %, 1 % and 100 % of them tainted with the longest key
(127 bytes) and value (63 bytes), 40 calls of each taint share alternating with the untainted call.  Kernel times come
from the library's per-stage CUDA events (KXPU_T_EMIT): median [p10, p90].  Prints the card and its power limit and one
JSON object (also written to argv[1] when given), with the SHA-256 of each call's output and slice offsets, so that two
builds can be checked for identical bytes."""
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
LONG_KEY = "p" * 30 + "." + "q" * 32 + "/" + "N" + ("a-b_c.d" * 9)[:61] + "Z"
LONG_VALUE = "V" + ("x_y-z.w" * 9)[:61] + "0"
SHARES = (0.0, 0.01, 1.0)


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def digest(out, length, offs, n_slices):
    """SHA-256 of a call's output bytes and its slice offsets"""
    h = hashlib.sha256(memoryview(out[:length]))
    h.update(memoryview(offs[:n_slices + 1]))
    return h.hexdigest()


def since_of(n, share, seed=5):
    """int64 taint times: `share` of the n devices tainted, spread over the pool, at times across the whole range"""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, B.DRA_TAINT_SINCE_MAX + 1, n, dtype=np.int64)
    return np.where(rng.random(n) < share, t, -1).astype(np.int64) if share < 1.0 else t


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    t = {}
    key, value = LONG_KEY.encode(), LONG_VALUE.encode()
    for layout, devs_of, plain, taint in (("pci", W.dra_devices, "kxpu_dra_slices", "kxpu_dra_slices_taint"),
                                          ("mdev", W.dra_mdev_devices, "kxpu_dra_slices_mdev", "kxpu_dra_slices_mdev_taint")):
        for n in (1 << 16, 1 << 20):
            devs = devs_of(n)
            ln, ns = C.c_size_t(0), C.c_size_t(0)
            offs = np.empty(n // 64 + 2, np.uint64)
            base = (kx.ctx, b"vfio.nvidia.com", b"node-a", b"node-a", 1, devs.ctypes.data, n)
            getattr(kx.L, plain)(*base, None, 0, C.byref(ln), None, C.byref(ns))
            plain_len = ln.value
            out = np.empty(plain_len + n * 300, np.uint8)

            def call_plain():
                rc = getattr(kx.L, plain)(*base, out.ctypes.data, out.size, C.byref(ln), offs.ctypes.data, C.byref(ns))
                assert rc == 0 and ln.value == plain_len

            for share in SHARES:
                since = since_of(n, share)

                def call_taint():
                    rc = getattr(kx.L, taint)(*base, key, value, b"NoSchedule", since.ctypes.data, out.ctypes.data, out.size,
                                              C.byref(ln), offs.ctypes.data, C.byref(ns))
                    assert rc == 0
                    return ln.value

                for _ in range(3):  # warm-up
                    call_taint(); call_plain()
                taint_len = call_taint()
                taint_sha = digest(out, taint_len, offs, ns.value)
                call_plain()
                plain_sha = digest(out, plain_len, offs, ns.value)
                k_t, k_p = [], []
                for _ in range(REPS):
                    call_taint()
                    k_t.append(kx.timings()[B.T_EMIT])
                    call_plain()
                    k_p.append(kx.timings()[B.T_EMIT])
                name = "%s_%d_taint%g" % (layout, n, 100 * share)
                t[name] = {"taint_kernel": stats(k_t), "untainted_kernel": stats(k_p), "taint_out_bytes": taint_len,
                           "untainted_out_bytes": plain_len, "taint_sha256": taint_sha, "untainted_sha256": plain_sha,
                           "ratio_median": round(float(np.median(k_t) / np.median(k_p)), 3)}
                print("%-4s n=%-8d %5.1f %% tainted: taint kernel %.4f ms [%.4f, %.4f] %d B | untainted %.4f ms [%.4f, %.4f] "
                      "%d B | x%.2f" % (layout, n, 100 * share, np.median(k_t), np.percentile(k_t, 10), np.percentile(k_t, 90),
                                       taint_len, np.median(k_p), np.percentile(k_p, 10), np.percentile(k_p, 90), plain_len,
                                       np.median(k_t) / np.median(k_p)))
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "timings": t}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
