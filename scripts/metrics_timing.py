"""Device time of kxpu_metrics_devices (DESIGN.md K17) on metrics_devices(2^20) -- 2^20 devices, 1 in 8 with one reason,
1 in 64 with three, details of about 80 bytes, 1 in 256 of them with a non-ASCII or escaped byte, every device with both
AER values -- next to kxpu_lw_encode_topo over the same devices' groups, health and a two-node NUMA mask, the two
alternated.  40 calls each; kernel times from the library's per-stage CUDA events (KXPU_T_EMIT: size pass, scan and
write pass of one call with a large enough buffer), median [p10, p90], and the bytes each call wrote.  The card's name,
power limit and SM clock are read in the same run.  Prints one JSON object (and writes it to argv[1] when given)."""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 40


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "min_ms": round(float(v.min()), 4),
            "max_ms": round(float(v.max()), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    kx = K.Kxpu(0)
    devs, strings, reasons = W.metrics_devices(1 << 20)
    rc, need = kx.metrics_devices_raw(devs, strings, reasons, None, 0)
    assert rc == B.E_NOSPACE, rc
    out = np.empty(need, np.uint8)
    groups = np.ascontiguousarray(devs["group"])
    healthy = np.ascontiguousarray(devs["healthy"].astype(np.uint8))
    masks = np.where(np.arange(len(devs)) % 2 == 0, 1, 2).astype(np.uint64)

    def metrics():
        kx.timer_begin()
        rc, got = kx.metrics_devices_raw(devs, strings, reasons, out, need)
        call = kx.timer_end()
        assert rc == B.KXPU_OK and got == need
        return call, kx.timings()[B.T_EMIT]

    lw_len = []

    def lw():
        kx.timer_begin()
        lw_len.append(len(kx.lw_encode_topo(groups, healthy, masks)))
        return kx.timer_end()

    for _ in range(3):
        metrics(); lw()
    a, k, b = [], [], []
    for _ in range(REPS):
        call, kern = metrics()
        a.append(call)
        k.append(kern)
        b.append(lw())
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "n_devices": len(devs), "n_reasons": len(reasons),
           "metrics_devices": {"bytes": int(need), "call": stats(a), "kernels": stats(k)},
           "lw_encode_topo": {"bytes": lw_len[-1], "call": stats(b)}}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
