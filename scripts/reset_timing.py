"""Device time of kxpu_reset_check (DESIGN.md K16) on reset_walk(2^20) -- 2^20 functions in 2^20 groups, 8 per down port,
70 % with "flr bus", 15 % bus only, 2 % pm only, 1 % a kernel without reset_method, 12 % with no method -- over the CSR
of kxpu_classify_viable on the same records, next to that classify call, the two alternated.  40 calls each; kernel times
from the library's per-stage CUDA events (KXPU_T_CLASSIFY), median [p10, p90].  The card's name and power limit are read
in the same run.  Prints one JSON object (and writes it to argv[1] when given)."""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 40
RULES = [(b"10de", b"vfio-pci")]


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "min_ms": round(float(v.min()), 4),
            "max_ms": round(float(v.max()), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    kx = K.Kxpu(0)

    def kernel_ms(fn):
        fn()
        return kx.timings()[B.T_CLASSIFY]

    recs, paths, rrs = W.reset_walk(1 << 20)
    c = kx.classify_viable(RULES, recs)
    viable = lambda: kx.classify_viable(RULES, recs)  # noqa: E731
    check = lambda: kx.reset_check(RULES, recs, paths, rrs, B.RM_ALL, c["group_off"], c["group_members"])  # noqa: E731
    for _ in range(3):
        viable(); check()
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(viable))
        b.append(kernel_ms(check))
    res = check()
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "n_records": len(recs), "n_groups": int(c["n_groups"]),
           "reset_check": {"n_withheld": int((res["group_reset"] != B.VIABLE).sum()),
                           "n_set_ok": int((res["set_verdict"] == B.RESET_SET_OK).sum()), "device": stats(b)},
           "classify_viable": {"device": stats(a)}}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
