"""Device time of the NUMA topology calls (DESIGN.md K5, K6, K8), 40 alternating calls each:
  - kxpu_classify_topo vs kxpu_classify_rules on topo_records (2^20 records, rule {10de, vfio-pci}): classify kernels,
    from the library's per-stage CUDA events;
  - kxpu_lw_encode_topo vs kxpu_lw_encode on 2^20 groups (masks of 1-2 nodes, 20 % without topology): the whole call
    on the ctx stream (uploads, kernels, download), from the library's device stopwatch (kxpu_timer_begin / _end);
  - kxpu_preferred_allocation for 4096 requests of 8 of 16 and for one request of 2^19 of 2^20: the whole call, same
    stopwatch.
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
    keys = kx.table_export(kx.pciids_load(W.load_pci_ids()))[0]
    recs = W.topo_records(keys)
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

    alternate("classify_topo_2^20", lambda: kx.classify_topo(NV, recs),
              "classify_rules_2^20", lambda: kx.classify_rules(NV, recs), stage_ms)
    n = 1 << 20
    rng = np.random.default_rng(5)
    groups = rng.integers(0, 2**32 - 1, n, dtype=np.uint64).astype(np.uint32)
    healthy = np.ones(n, np.uint8)
    masks = W.topo_dev_numa(n, nodes=4)
    masks[rng.random(n) < 0.2] = 0
    alternate("lw_encode_topo_2^20", lambda: kx.lw_encode_topo(groups, healthy, masks),
              "lw_encode_2^20", lambda: kx.lw_encode(groups, healthy), call_ms)
    dn_small = W.topo_dev_numa(4096, nodes=4)
    small = B.pref_requests(W.topo_requests(dn_small, n_req=4096, avail=16, size=8))
    out_s, off_s = np.empty(int(small["size"].sum()), np.uint32), np.empty(4097, np.uint32)
    dn_big = W.topo_dev_numa(n, nodes=4)
    big = B.pref_requests(W.topo_requests(dn_big, n_req=1, avail=n, size=n // 2, must_max=3, seed=10))
    out_b, off_b = np.empty(n // 2, np.uint32), np.empty(2, np.uint32)
    alternate("preferred_allocation_4096x_8_of_16", lambda: kx.preferred_allocation_raw(dn_small, small, out_s, off_s),
              "preferred_allocation_1x_2^19_of_2^20", lambda: kx.preferred_allocation_raw(dn_big, big, out_b, off_b), call_ms)
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "timings": t}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
