"""Device time of the vGPU PCIe calls next to their parents, each pair alternated, 40 calls each: kxpu_pcie_ports_mdev
(K10) next to kxpu_pcie_tree_mdev on the same walk of 2^20 mdevs (workloads.pcie_ports_mdev_walk: parents below root
ports and switches, one in four a VF), kxpu_dra_slices_mdev_pcie (K11) next to kxpu_dra_slices_mdev_pf and
kxpu_dra_slices_vf_vgpu_pcie next to kxpu_dra_slices_vf_vgpu on the same 2^20 devices, each slice pair untainted and
with a three-entry taint table.  Kernel times from the library's per-stage CUDA events (KXPU_T_CLASSIFY, KXPU_T_EMIT),
median [p10, p90].  The card's name and power limit are read in the same run.  Prints one JSON object (and writes it
to argv[1] when given)."""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 40
TAINTS = [("vgpu.example.com/unhealthy", "vfio-device-missing", "NoSchedule"),
          ("vgpu.example.com/pcie-aer", "fatal", "NoSchedule"), ("vgpu.example.com/pcie-aer", "nonfatal", "NoSchedule")]
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
    since = np.where(np.arange(3 * n).reshape(n, 3) % 97 == 0, 1767225600, -1).astype(np.int64)
    since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    mdevs, vfs = W.dra_mdev_pcie_devices(n), W.dra_vf_vgpu_pcie_devices(n)
    out = {}
    for layout, devs, fpcie, fbase, sub in (
            ("mdev", mdevs, kx.dra_slices_mdev_pcie, kx.dra_slices_mdev_pf, "pf"),
            ("vf_vgpu", vfs, kx.dra_slices_vf_vgpu_pcie, kx.dra_slices_vf_vgpu, "dev")):
        for name, s in (("untainted", None), ("tainted", since)):
            fa = lambda: fpcie("vgpu.example.com", "node-a", "node-a", 1, DOMAIN, devs, TAINTS, s)  # noqa: E731
            fb = lambda: fbase("vgpu.example.com", "node-a", "node-a", 1, devs[sub], TAINTS, s)  # noqa: E731
            (ta, tb), blen = pair(kx, B.T_EMIT, fa, fb), (len(fa()[0]), len(fb()[0]))
            out["%s_%s" % (layout, name)] = {"pcie": dict(ta, bytes=blen[0]), "base": dict(tb, bytes=blen[1]),
                                             "ratio": round(ta["median_ms"] / tb["median_ms"], 3)}
    recs, paths, off, mem = W.pcie_ports_mdev_walk(n)
    fa = lambda: kx.pcie_ports_mdev(recs, paths, off, mem)  # noqa: E731
    fb = lambda: kx.pcie_tree_mdev(recs, paths, off, mem)  # noqa: E731
    ta, tb = pair(kx, B.T_CLASSIFY, fa, fb)
    rp, sw = fa()
    ports = {"pcie_ports_mdev": ta, "pcie_tree_mdev": tb, "ratio": round(ta["median_ms"] / tb["median_ms"], 3),
             "n_groups": n, "with_root_port": int((rp != B.PCIE_NO_KEY).sum()),
             "with_switch": int((sw != B.PCIE_NO_KEY).sum())}
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "n_devices": n, "dra_slices": out, "ports": ports}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
