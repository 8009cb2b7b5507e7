"""Device time of kxpu_dra_slices_pcie (DESIGN.md K11) next to kxpu_dra_slices_pf on the same 2^20 passthrough devices
(workloads.dra_pcie_devices: one in eight a VF, a root port on every device and a switch on three in four), untainted
and with a three-entry taint table, and of kxpu_pcie_ports (K10) next to kxpu_pcie_tree on the same walk of 2^20
functions (workloads.pcie_ports_walk), each pair alternated.  40 calls each; kernel times from the library's per-stage
CUDA events (KXPU_T_EMIT, KXPU_T_CLASSIFY), median [p10, p90].  The card's name and power limit are read in the same
run.  Prints one JSON object (and writes it to argv[1] when given)."""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 40
TAINTS = [("vfio.nvidia.com/unhealthy", "vfio-device-missing", "NoSchedule"),
          ("vfio.nvidia.com/pcie-aer", "fatal", "NoSchedule"), ("vfio.nvidia.com/pcie-aer", "nonfatal", "NoSchedule")]
DOMAIN = "pcie.example.com"


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def pair(kx, slot, fa, fb):
    """alternated device times of two calls"""
    for _ in range(3):
        fa(); fb()
    a, b = [], []
    for _ in range(REPS):
        fa(); a.append(kx.timings()[slot])
        fb(); b.append(kx.timings()[slot])
    return stats(a), stats(b)


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    kx = K.Kxpu(0)
    n = 1 << 20
    devs = W.dra_pcie_devices(n)
    since = np.where(np.arange(3 * n).reshape(n, 3) % 97 == 0, 1767225600, -1).astype(np.int64)
    since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    out = {}
    for name, s in (("untainted", None), ("tainted", since)):
        fa = lambda: kx.dra_slices_pcie("vfio.nvidia.com", "node-a", "node-a", 1, DOMAIN, devs, TAINTS, s)  # noqa: E731
        fb = lambda: kx.dra_slices_pf("vfio.nvidia.com", "node-a", "node-a", 1, devs["pf"], TAINTS, s)  # noqa: E731
        (ta, tb), blen = pair(kx, B.T_EMIT, fa, fb), (len(fa()[0]), len(fb()[0]))
        out[name] = {"pcie": dict(ta, bytes=blen[0]), "pf": dict(tb, bytes=blen[1]),
                     "ratio": round(ta["median_ms"] / tb["median_ms"], 3)}
    recs, paths, off, mem = W.pcie_ports_walk(n)
    fa = lambda: kx.pcie_ports(recs, paths, off, mem)  # noqa: E731
    fb = lambda: kx.pcie_tree(recs, paths, off, mem)  # noqa: E731
    ta, tb = pair(kx, B.T_CLASSIFY, fa, fb)
    rp, sw = fa()
    ports = {"pcie_ports": ta, "pcie_tree": tb, "ratio": round(ta["median_ms"] / tb["median_ms"], 3),
             "n_groups": n, "with_switch": int((sw != B.PCIE_NO_KEY).sum())}
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "n_devices": n,
           "n_vfs": int((devs["pf"]["physfn"] != b"").sum()), "dra_slices": out, "ports": ports}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
