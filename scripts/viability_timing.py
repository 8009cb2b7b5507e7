"""Device time of kxpu_classify_viable next to kxpu_classify_rules (DESIGN.md K5): 40 alternating calls of each on
viab_records(2^20), kernel times from the library's per-stage CUDA events, median [p10, p90].  The card's name and power
limit are read in the same run.  Prints one JSON object (and writes it to argv[1] when given)."""
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
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    kx = K.Kxpu(0)
    recs = W.viab_records(1 << 20)
    rules = W.VIAB_RULES

    def kernel_ms(fn):
        fn()
        return kx.timings()[B.T_CLASSIFY]
    for _ in range(3):  # warm-up
        kx.classify_rules(rules, recs); kx.classify_viable(rules, recs)
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(lambda: kx.classify_rules(rules, recs)))
        b.append(kernel_ms(lambda: kx.classify_viable(rules, recs)))
    res = kx.classify_viable(rules, recs)
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "n_records": len(recs), "n_groups": int(res["n_groups"]),
           "n_blockers": int(((recs["flags"] & B.REC_BLOCKS) != 0).sum()),
           "timings": {"classify_rules": stats(a), "classify_viable": stats(b)}}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
