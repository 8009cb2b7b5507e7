"""Device time of kxpu_vf_vgpu_drift (DESIGN.md K15) over 2^20 re-read VF records and 2^20 one-member groups, about 1 in
64 of them drifted (cleared, changed or unreadable), beside kxpu_vf_vgpu_types on the same records and the walk's name
tables (vf_vgpu_walk(2^20)), the two calls alternated.  40 calls each; kernel times from the library's per-stage CUDA
events (KXPU_T_CLASSIFY), median [p10, p90].  The card's name and power limit are read in the same run.  Prints one
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
N = 1 << 20


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

    _, vts, tables = W.vf_vgpu_walk(N)
    blob, toff = B.vgpu_tables(tables)
    was = kx.vf_vgpu_types(vts, (blob, toff))["type_id"].copy()
    # the re-read: about 1 in 64 records drifted, a third each cleared, changed and unreadable
    rng = np.random.default_rng(64)
    now = vts.copy()
    d = np.flatnonzero(rng.random(N) < 1.0 / 64)
    kind = rng.integers(0, 3, len(d))
    for i, k in zip(d, kind):
        txt = [b"0\n", b"4294967295\n", b"0557\n"][k]
        now["cur_txt"][i] = np.frombuffer(txt.ljust(16, b"\0"), np.uint8)
        now["cur_len"][i] = len(txt)
    now["flags"][d] |= B.VT_READ
    goff, gmem = np.arange(N + 1, dtype=np.uint32), np.arange(N, dtype=np.uint32)
    drift = lambda: kx.vf_vgpu_drift(now, was, goff, gmem)  # noqa: E731
    types = lambda: kx.vf_vgpu_types(now, (blob, toff))  # noqa: E731
    for _ in range(3):
        drift(); types()
    l0 = kx.launch_count()
    drift()
    launches = kx.launch_count() - l0
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(drift))
        b.append(kernel_ms(types))
    res = drift()
    first = res["group_first"]
    out = {"gpu": smi.stdout.strip(), "reps": REPS,
           "vf_vgpu_drift": {"n_records": N, "n_groups": N, "launches": launches,
                             "drifted_groups": int((first != B.VD_STEADY).sum()),
                             "by_status": {s: int((res["status_now"] == v).sum())
                                           for s, v in (("same", B.VD_SAME), ("cleared", B.VD_CLEARED),
                                                        ("changed", B.VD_CHANGED), ("bad", B.VD_BAD))},
                             "device": stats(a)},
           "vf_vgpu_types": {"n_records": N, "n_tables": len(tables), "blob_bytes": int(toff[-1]), "device": stats(b)}}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
