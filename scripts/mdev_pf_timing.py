"""Device time of kxpu_mdev_pf (DESIGN.md K18) on mdev_pf_walk -- 2^20 mdevs on the VFs of 2^15 PFs among 2^20 PCI
records, 1 in 16 on a PF and 1 in 16 with a link that cannot resolve -- next to kxpu_sriov on sriov_walk(2^20), a walk of
the same size; and of kxpu_dra_slices_mdev_pf next to kxpu_dra_slices_mdev_taints on 2^20 vGPUs (untainted, and with a
three-entry taint table), the calls of each pair alternated.  40 calls each; kernel times from the library's per-stage
CUDA events (KXPU_T_CLASSIFY / KXPU_T_EMIT), median [p10, p90].  The card's name and power limit are read in the same
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
RULES = [(b"10de", b"vfio-pci")]
TAINTS = [("vgpu.nvidia.com/unhealthy", "vfio-device-missing", "NoSchedule"),
          ("vgpu.nvidia.com/pcie-aer", "fatal", "NoSchedule"), ("vgpu.nvidia.com/pcie-aer", "nonfatal", "NoSchedule")]


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
    recs, mrecs, msrs, want = W.mdev_pf_walk()
    pf_of = np.empty(len(mrecs), np.uint32)
    mp = lambda: kx.mdev_pf_raw(recs, mrecs, msrs, pf_of)  # noqa: E731
    mp()
    assert np.array_equal(pf_of, want)
    srecs, ssrs = W.sriov_walk(1 << 20)
    c = kx.classify_rules(RULES, srecs)
    sr = lambda: kx.sriov(RULES, srecs, ssrs, c["group_ids"], c["group_off"], c["group_members"])  # noqa: E731
    t_mp, t_sr = pair(kx, B.T_CLASSIFY, mp, sr)

    n = 1 << 20
    devs = np.zeros(n, B.DRAMDEVPF_DTYPE)
    devs["dev"] = W.dra_mdev_devices(n)
    vf = np.arange(n) % 16 != 0  # 15 in 16 vGPUs on a VF of a PF with a known device id
    devs["physfn"] = np.where(vf, b"0000:41:00.0", b"")
    devs["physfn_device"] = np.where(vf, b"2330", b"")
    since = np.where(np.arange(3 * n).reshape(n, 3) % 97 == 0, 1767225600, -1).astype(np.int64)
    since[:, 2] = np.where(since[:, 1] >= 0, -1, since[:, 2])
    out = {}
    for name, s in (("untainted", None), ("tainted", since)):
        fa = lambda: kx.dra_slices_mdev_pf("vgpu.nvidia.com", "node-a", "node-a", 1, devs, TAINTS, s)  # noqa: E731
        fb = lambda: kx.dra_slices_mdev_taints("vgpu.nvidia.com", "node-a", "node-a", 1, devs["dev"], TAINTS, s)  # noqa: E731
        (ta, tb), blen = pair(kx, B.T_EMIT, fa, fb), (len(fa()[0]), len(fb()[0]))
        out[name] = {"mdev_pf": dict(ta, bytes=blen[0]), "mdev_taints": dict(tb, bytes=blen[1])}
    res = {"gpu": smi.stdout.strip(), "reps": REPS,
           "mdev_pf": {"n_records": len(recs), "n_mdevs": len(mrecs), "n_resolved": int((pf_of != B.NO_PF).sum()),
                       "device": t_mp},
           "sriov": {"n_records": len(srecs), "device": t_sr},
           "dra_slices": dict(out, n_devices=n)}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
