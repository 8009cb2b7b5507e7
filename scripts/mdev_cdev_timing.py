"""Times of the CDI spec of a vGPU class served through VFIO cdevs (DESIGN.md K6 / K13) beside the vGPU group layout's.
  - kxpu_cdi_emit_mdev_cdev and kxpu_cdi_emit_mdev on the same records (kind nvidia.com/vgpu), 2^16 and 2^20 vGPUs,
    YAML and JSON: the device time under KXPU_T_EMIT and the whole call on the host clock;
  - kxpu_cdi_parse_mdev_cdev and kxpu_cdi_parse_mdev on those documents: the same two times.
Before any timing, every document is checked against the oracle (the cdev one: the C oracle's vGPU document with each
node replaced, mdev_cdev_cases.oracle_doc) and every parse against the records.  The two layouts alternate call by call
in one process, 20 calls of each after two warm-up rounds.  Median [p10, p90].  Prints the card and its power limit, a
SHA-256 of every output, and one JSON object (also written to argv[1] when given)."""
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B  # noqa: E402
import mdev_cdev_cases as MC  # noqa: E402
from oracle import mdev_oracle as MO  # noqa: E402

REPS = 20
SIZES = [1 << 16, 1 << 20]
KIND = b"nvidia.com/vgpu"


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "kind": KIND.decode(), "rows": {}}
    for n in SIZES:
        recs = MC.records(n, seed=11)
        dev_recs = np.ascontiguousarray(recs["dev"])
        for fmt, fname in ((B.FMT_YAML, "yaml"), (B.FMT_JSON, "json")):
            calls = {
                "cdev_emit": lambda: kx.cdi_emit_mdev_cdev(fmt, recs, KIND),
                "group_emit": lambda: kx.cdi_emit_mdev(fmt, dev_recs, KIND),
            }
            docs = {"cdev": calls["cdev_emit"](), "group": calls["group_emit"]()}
            assert docs["cdev"] == MC.oracle_doc(fmt, KIND, recs), "mdev cdev document differs from the oracle"
            assert docs["group"] == MO.cdi_emit_mdev(fmt, KIND, dev_recs), "mdev document differs from the oracle"
            calls["cdev_parse"] = lambda: kx.cdi_parse_mdev_cdev(fmt, docs["cdev"], KIND)
            calls["group_parse"] = lambda: kx.cdi_parse_mdev(fmt, docs["group"], KIND)
            parsed = {"cdev": calls["cdev_parse"](), "group": calls["group_parse"]()}
            assert parsed["cdev"].tobytes() == recs.tobytes()
            assert parsed["group"].tobytes() == dev_recs.tobytes()
            for _ in range(2):
                for f in calls.values():
                    f()
            dev = {k: [] for k in calls}
            wall = {k: [] for k in calls}
            for _ in range(REPS):
                for k, f in calls.items():  # alternating: cdev emit, group emit, cdev parse, group parse
                    t = time.perf_counter()
                    f()
                    wall[k].append((time.perf_counter() - t) * 1e3)
                    dev[k].append(kx.timings()[B.T_EMIT])
            for k in calls:
                layout, op = k.split("_")
                name = "%s_%s_%d" % (k, fname, n)
                out = docs[layout] if op == "emit" else parsed[layout]
                res["rows"][name] = {"doc_bytes": len(docs[layout]), "sha256": sha(out), "device": stats(dev[k]),
                                     "call": stats(wall[k])}
                print(name, json.dumps(res["rows"][name]))
            for op in ("emit", "parse"):
                r = np.median(dev["cdev_" + op]) / np.median(dev["group_" + op])
                res["rows"]["%s_%s_%d_cdev_over_group" % (op, fname, n)] = round(float(r), 4)
                print("%s %s %d: cdev / group device time %.3f, bytes %.3f" % (op, fname, n, r,
                                                                                len(docs["cdev"]) / len(docs["group"])))
    out = json.dumps(res)
    print(out)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(out)
    kx.close()


if __name__ == "__main__":
    main()
