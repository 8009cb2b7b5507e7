"""Device time of kxpu_pcie_tree_mdev (DESIGN.md K10) on pcie_mdev_walk(2^20) -- 32 vGPUs per parent GPU, the parents
scattered over the walk order -- next to kxpu_pcie_tree on the walk's PCI twin (the same forest), the two calls
alternated over 40 calls: kernel time from the library's per-stage CUDA events (KXPU_T_CLASSIFY).  Then
kxpu_preferred_allocation_pcie on the forest of a 4096-vGPU walk for 4096 requests of 4 of 32 vGPUs, alternated with
kxpu_preferred_allocation on the same requests: whole-call time between CUDA events.  Median [p10, p90].  The card's name and power limit are read in the same run.  Prints one JSON object (and writes it to
argv[1] when given)."""
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

    def kernel_ms(fn):
        fn()
        return kx.timings()[B.T_CLASSIFY]

    recs, paths, off, mem, twin, twin_paths = W.pcie_mdev_walk(1 << 20)
    mdev = lambda: kx.pcie_tree_mdev(recs, paths, off, mem)  # noqa: E731
    plain = lambda: kx.pcie_tree(twin, twin_paths, off, mem)  # noqa: E731
    for _ in range(3):
        mdev(); plain()
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(mdev))
        b.append(kernel_ms(plain))
    t0, t1 = mdev(), plain()
    same = all(np.array_equal(t0[k], t1[k]) for k in t0)

    # 4096 requests of 4 out of 32 available vGPUs, over the forest of a 4096-vGPU walk (128 parent GPUs)
    r2, p2, o2, g2, _, _ = W.pcie_mdev_walk(4096, seed=31)
    f = kx.pcie_tree_mdev(r2, p2, o2, g2)
    dn = W.topo_dev_numa(4096, nodes=4)
    reqs = B.pref_requests(W.topo_requests(dn, n_req=4096, avail=32, size=4))
    out_a, off_a = np.empty(int(reqs["size"].sum()), np.uint32), np.empty(4097, np.uint32)
    alloc = lambda: kx.preferred_allocation_pcie_raw(dn, f["group_node"], f["parent"], f["depth"], reqs, out_a, off_a)  # noqa: E731
    numa = lambda: kx.preferred_allocation_raw(dn, reqs, out_a, off_a)  # noqa: E731

    def call_ms(fn):
        kx.timer_begin()
        fn()
        return kx.timer_end()

    for _ in range(3):
        alloc(); numa()
    c, d = [], []
    for _ in range(REPS):
        c.append(call_ms(alloc))
        d.append(call_ms(numa))
    out = {"gpu": smi.stdout.strip(), "reps": REPS,
           "pcie_tree_mdev": {"n_records": len(recs), "n_groups": len(off) - 1, "nodes": len(t0["key"]), "device": stats(a)},
           "pcie_tree_twin": {"nodes": len(t1["key"]), "same_forest": bool(same), "device": stats(b)},
           "preferred_allocation_pcie_4096x_4_of_32": {"nodes": len(f["key"]), "call": stats(c)},
           "preferred_allocation_4096x_4_of_32": {"call": stats(d)}}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
