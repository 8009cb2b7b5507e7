"""Device time of the vGPU-on-VF calls (DESIGN.md K15) on vf_vgpu_walk(2^20) -- a PF and 31 VFs per GPU on the vGPU
manager's driver, 1 VF in 4 free and listing the 14-line H100 type table: kxpu_vf_vgpu_types over those tables, and
kxpu_classify_vf_vgpu with the walk's key rows next to kxpu_classify_rules on the same records, the two classify calls
alternated.  40 calls each; kernel times from the library's per-stage CUDA events (KXPU_T_CLASSIFY), median [p10, p90].
The card's name and power limit are read in the same run.  Prints one JSON object (and writes it to argv[1] when
given)."""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 40
RULES = [(b"10de", b"nvidia")]


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

    recs, vts, tables = W.vf_vgpu_walk(1 << 20)
    blob, toff = B.vgpu_tables(tables)
    types = lambda: kx.vf_vgpu_types(vts, (blob, toff))  # noqa: E731
    for _ in range(3):
        types()
    l0 = kx.launch_count()
    types()
    reruns = (kx.launch_count() - l0) // 2 - 1  # two launches per run: a rerun of the join shows as four
    t = [kernel_ms(types) for _ in range(REPS)]
    res = types()
    keys = res["keys"]
    vf = lambda: kx.classify_vf_vgpu(RULES, 1, recs, keys)  # noqa: E731
    plain = lambda: kx.classify_rules(RULES, recs)  # noqa: E731
    for _ in range(3):
        vf(); plain()
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(plain))
        b.append(kernel_ms(vf))
    c0, c1 = plain(), vf()
    st = res["status"]
    out = {"gpu": smi.stdout.strip(), "reps": REPS,
           "vf_vgpu_types": {"n_records": len(vts), "n_tables": len(tables), "blob_bytes": int(toff[-1]),
                             "named": int((st == B.VT_NAMED).sum()), "unnamed": int((st == B.VT_UNNAMED).sum()),
                             "bad": int((st == B.VT_BAD).sum()), "reruns": reruns, "device": stats(t)},
           "classify_rules": {"n_groups": int(c0["n_groups"]), "n_devids": int(c0["n_devids"]), "device": stats(a)},
           "classify_vf_vgpu": {"n_groups": int(c1["n_groups"]), "n_devids": int(c1["n_devids"]), "device": stats(b)}}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
