"""Times of the typed CDI layouts of a class that serves vGPUs on SR-IOV VFs (DESIGN.md K6 / K13) beside the plain
layouts they extend.
  - kxpu_cdi_emit_vf_vgpu against kxpu_cdi_emit_kind, and kxpu_cdi_emit_vf_vgpu_cdev against kxpu_cdi_emit_cdev, on the
    same 2^20 VFs (workloads.vf_vgpu_cdi_devices, kind nvidia.com/vgpu), YAML and JSON: the device time under
    KXPU_T_EMIT and the whole call on the host clock;
  - the four parse calls on those documents: the same two times.
Before any timing, every typed document is checked against the C oracle (tests/vf_vgpu_cdi_oracle.c) and every parse
against the records.  The four layouts alternate call by call in one process, 20 calls of each after two warm-up
rounds.  Median [p10, p90].  Prints the card and its power limit, a SHA-256 of every output, and one JSON object (also
written to argv[1] when given)."""
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
from kxpu_b200 import binding as B, workloads as W  # noqa: E402
import vf_vgpu_cdi_oracle as VO  # noqa: E402

REPS = 20
N = 1 << 20
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
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "kind": KIND.decode(), "n": N, "rows": {}}
    recs = W.vf_vgpu_cdi_devices(N)
    plain = np.ascontiguousarray(recs["dev"])
    group_recs = recs.copy()
    group_recs["dev"][B.CDEV_FIELD] = 0
    for fmt, fname in ((B.FMT_YAML, "yaml"), (B.FMT_JSON, "json")):
        calls = {
            "typed_emit": lambda: kx.cdi_emit_vf_vgpu(fmt, recs, KIND),
            "plain_emit": lambda: kx.cdi_emit(fmt, plain, KIND),
            "typedcdev_emit": lambda: kx.cdi_emit_vf_vgpu(fmt, recs, KIND, cdev=True),
            "plaincdev_emit": lambda: kx.cdi_emit_cdev(fmt, plain, KIND),
        }
        docs = {k.split("_")[0]: f() for k, f in calls.items()}
        assert docs["typed"] == VO.emit(fmt, KIND, recs), "typed document differs from the oracle"
        assert docs["typedcdev"] == VO.emit(fmt, KIND, recs, cdev=True), "typed cdev document differs from the oracle"
        calls["typed_parse"] = lambda: kx.cdi_parse_vf_vgpu(fmt, docs["typed"], KIND)
        calls["plain_parse"] = lambda: kx.cdi_parse(fmt, docs["plain"], KIND)
        calls["typedcdev_parse"] = lambda: kx.cdi_parse_vf_vgpu(fmt, docs["typedcdev"], KIND, cdev=True)
        calls["plaincdev_parse"] = lambda: kx.cdi_parse_cdev(fmt, docs["plaincdev"], KIND)
        parsed = {k.split("_")[0]: f() for k, f in calls.items() if k.endswith("_parse")}
        assert parsed["typed"].tobytes() == group_recs.tobytes()
        assert parsed["typedcdev"].tobytes() == recs.tobytes()
        assert parsed["plaincdev"].tobytes() == plain.tobytes()
        for _ in range(2):
            for f in calls.values():
                f()
        dev = {k: [] for k in calls}
        wall = {k: [] for k in calls}
        for _ in range(REPS):
            for k, f in calls.items():  # alternating: the four emits, then the four parses
                t = time.perf_counter()
                f()
                wall[k].append((time.perf_counter() - t) * 1e3)
                dev[k].append(kx.timings()[B.T_EMIT])
        for k in calls:
            layout, op = k.split("_")
            name = "%s_%s" % (k, fname)
            out = docs[layout] if op == "emit" else parsed[layout]
            res["rows"][name] = {"doc_bytes": len(docs[layout]), "sha256": sha(out), "device": stats(dev[k]),
                                 "call": stats(wall[k])}
            print(name, json.dumps(res["rows"][name]))
        for op in ("emit", "parse"):
            for t, p in (("typed", "plain"), ("typedcdev", "plaincdev")):
                r = np.median(dev["%s_%s" % (t, op)]) / np.median(dev["%s_%s" % (p, op)])
                res["rows"]["%s_%s_%s_over_%s" % (op, fname, t, p)] = round(float(r), 4)
                print("%s %s: %s / %s device time %.3f, bytes %.3f" % (op, fname, t, p, r, len(docs[t]) / len(docs[p])))
    out = json.dumps(res)
    print(out)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(out)
    kx.close()


if __name__ == "__main__":
    main()
