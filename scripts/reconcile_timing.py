"""Device time of kxpu_reconcile (DESIGN.md K9) on reconcile_pair(2^20) (PCI keys), 40 calls alternating with
kxpu_classify on cfg3 (2^20 records) in the same process:
  - kernels: the library's per-stage CUDA events (table reset, insert, probe + scan for reconcile; every classify kernel);
  - call: the whole call on the ctx stream (uploads, kernels, downloads), from the library's device stopwatch
    (kxpu_timer_begin / _end).
Prints the card and its power limit, read in the same run, and one JSON object (also written to argv[1] when given)."""
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
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    keys = kx.table_export(kx.pciids_load(W.load_pci_ids()))[0]
    recs = W.cfg3_records(keys)
    prev, cur, ni = W.reconcile_pair(3, 1 << 20)
    out = B.reconcile_outputs(len(prev), len(cur))

    def rc():
        kx.reconcile_raw(prev, cur, ni, out)

    def cl():
        kx.classify(recs)

    for _ in range(3):  # warm-up
        rc(); cl()
    samples = {"reconcile_kernels": [], "reconcile_call": [], "classify_kernels": [], "classify_call": []}
    for _ in range(REPS):
        for name, fn in (("reconcile", rc), ("classify", cl)):
            kx.timer_begin()
            fn()
            samples[name + "_call"].append(kx.timer_end())
            samples[name + "_kernels"].append(kx.timings()[B.T_CLASSIFY])
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "n_prev": len(prev), "n_cur": len(cur),
           "counts": B.reconcile_result(out)["counts"], "timings": {k: stats(v) for k, v in samples.items()}}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
