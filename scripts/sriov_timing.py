"""Device time of kxpu_sriov (DESIGN.md K14) on sriov_walk(2^20) -- 1 record in 8 a PF carrying 7 VFs -- over the CSR of
kxpu_classify_rules, and of kxpu_pcie_tree_sriov next to kxpu_pcie_tree on pcie_walk(2^20) with functions 1..7 of every
device naming function 0 as PF, the two tree calls alternated.  40 calls each; kernel times from the library's per-stage
CUDA events (KXPU_T_CLASSIFY), median [p10, p90].  The card's name and power limit are read in the same run.  Prints one
JSON object (and writes it to argv[1] when given)."""
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

    recs, srs = W.sriov_walk(1 << 20)
    c = kx.classify_rules(RULES, recs)
    call = lambda: kx.sriov(RULES, recs, srs, c["group_ids"], c["group_off"], c["group_members"])  # noqa: E731
    for _ in range(3):
        call()
    sr = [kernel_ms(call) for _ in range(REPS)]
    res = call()

    precs, ppaths, poff, pmem = W.pcie_walk(1 << 20)
    i = np.arange(len(precs), dtype=np.uint64)
    pf_of = np.where(i & 7, i & ~np.uint64(7), B.NO_PF).astype(np.uint32)
    plain = lambda: kx.pcie_tree(precs, ppaths, poff, pmem)  # noqa: E731
    vf = lambda: kx.pcie_tree(precs, ppaths, poff, pmem, pf_of)  # noqa: E731
    for _ in range(3):
        plain(); vf()
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(plain))
        b.append(kernel_ms(vf))
    t0, t1 = plain(), vf()
    out = {"gpu": smi.stdout.strip(), "reps": REPS,
           "sriov": {"n_records": len(recs), "n_groups": int(c["n_groups"]),
                     "n_withheld": int((res["group_sriov"] != B.VIABLE).sum()),
                     "n_vfs_resolved": int((res["pf_of"] != B.NO_PF).sum()), "device": stats(sr)},
           "pcie_tree": {"n_records": len(precs), "n_groups": len(poff) - 1, "nodes": len(t0["key"]), "device": stats(a)},
           "pcie_tree_sriov": {"nodes": len(t1["key"]), "device": stats(b)}}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
