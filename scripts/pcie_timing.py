"""Device time of the PCIe topology calls (DESIGN.md K10), 40 alternating calls each:
  - kxpu_pcie_tree vs kxpu_classify_topo on the same 2^20 records (pcie_walk: groups of 1..4 records): the kernels,
    from the library's per-stage CUDA events (both report in the classify slot);
  - kxpu_preferred_allocation_pcie vs kxpu_preferred_allocation for 4096 requests of 8 of 16 devices and for one request
    of 2^19 of 2^20: the whole call on the ctx stream (uploads, kernels, download), from the library's device stopwatch
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
NV = [(b"10de", b"vfio-pci")]


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    t = {}

    def stage_ms(fn):
        fn()
        return kx.timings()[B.T_CLASSIFY]

    def call_ms(fn):
        kx.timer_begin()
        fn()
        return kx.timer_end()

    def alternate(name_a, fa, name_b, fb, measure):
        for _ in range(3):  # warm-up
            fa(); fb()
        a, b = [], []
        for _ in range(REPS):
            a.append(measure(fa))
            b.append(measure(fb))
        t[name_a], t[name_b] = stats(a), stats(b)

    n = 1 << 20
    recs, paths, off, mem = W.pcie_walk(n)
    alternate("pcie_tree_2^20", lambda: kx.pcie_tree(recs, paths, off, mem),
              "classify_topo_2^20", lambda: kx.classify_topo(NV, recs), stage_ms)

    def forest(m, seed):
        r, p, o, g = W.pcie_walk(m + m // 8, seed=seed, group_max=1)
        f = kx.pcie_tree(r, p, o, g)
        return f["group_node"][:m].copy(), f["parent"], f["depth"]

    node_s, par_s, dep_s = forest(4096, 31)
    dn_small = W.topo_dev_numa(4096, nodes=4)
    small = B.pref_requests(W.topo_requests(dn_small, n_req=4096, avail=16, size=8))
    out_s, off_s = np.empty(int(small["size"].sum()), np.uint32), np.empty(4097, np.uint32)
    alternate("preferred_allocation_pcie_4096x_8_of_16",
              lambda: kx.preferred_allocation_pcie_raw(dn_small, node_s, par_s, dep_s, small, out_s, off_s),
              "preferred_allocation_4096x_8_of_16", lambda: kx.preferred_allocation_raw(dn_small, small, out_s, off_s),
              call_ms)
    node_b, par_b, dep_b = forest(n, 41)
    dn_big = W.topo_dev_numa(n, nodes=4)
    big = B.pref_requests(W.topo_requests(dn_big, n_req=1, avail=n, size=n // 2, must_max=3, seed=10))
    out_b, off_b = np.empty(n // 2, np.uint32), np.empty(2, np.uint32)
    alternate("preferred_allocation_pcie_1x_2^19_of_2^20",
              lambda: kx.preferred_allocation_pcie_raw(dn_big, node_b, par_b, dep_b, big, out_b, off_b),
              "preferred_allocation_1x_2^19_of_2^20", lambda: kx.preferred_allocation_raw(dn_big, big, out_b, off_b),
              call_ms)
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "nodes_2^20": int(len(par_b)), "timings": t}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
