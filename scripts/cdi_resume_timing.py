"""Times of the CDI spec parse that a restart with resumeIndices runs (DESIGN.md K13).
  - kxpu_cdi_parse / kxpu_cdi_parse_mdev on the documents of 65 536 and 2^20 devices, YAML and JSON, kind
    nvidia.com/gpu (vGPUs: nvidia.com/vgpu): the device time under KXPU_T_EMIT (decode, re-emit and compare, with the one
    host read of the device count between them) and the whole call on the host clock (upload of the document included);
  - kxpu_cdi_emit_kind / kxpu_cdi_emit_mdev on the same records: KXPU_T_EMIT and the whole call;
  - reading the document back from a file in the page cache, the start-up's host step before the parse.
20 calls of each, alternating parse and emit.  Median [p10, p90].  Prints the card and its power limit, and one JSON
object (also written to argv[1] when given)."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B  # noqa: E402
import cdi_parse_cases as CC  # noqa: E402

REPS = 20


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "rows": {}}
    for n in (1 << 16, 1 << 20):
        for mdev in (False, True):
            recs = CC.records(n, mdev, seed=11)
            kind = b"nvidia.com/vgpu" if mdev else b"nvidia.com/gpu"
            for fmt, fname in ((B.FMT_YAML, "yaml"), (B.FMT_JSON, "json")):
                emit = (lambda: kx.cdi_emit_mdev(fmt, recs, kind)) if mdev else (lambda: kx.cdi_emit(fmt, recs, kind))
                doc = emit()
                parse = (lambda: kx.cdi_parse_mdev(fmt, doc, kind)) if mdev else (lambda: kx.cdi_parse(fmt, doc, kind))
                got = parse()
                assert got.tobytes() == recs.tobytes()
                for _ in range(2):
                    parse(); emit()
                pd, pw, ed, ew = [], [], [], []
                for _ in range(REPS):
                    t = time.perf_counter(); parse(); pw.append((time.perf_counter() - t) * 1e3)
                    pd.append(kx.timings()[B.T_EMIT])
                    t = time.perf_counter(); emit(); ew.append((time.perf_counter() - t) * 1e3)
                    ed.append(kx.timings()[B.T_EMIT])
                with tempfile.NamedTemporaryFile() as f:
                    f.write(doc); f.flush()
                    rd = []
                    for _ in range(5):
                        t = time.perf_counter()
                        with open(f.name, "rb") as g:
                            g.read()
                        rd.append((time.perf_counter() - t) * 1e3)
                name = "%s_%s_%d" % ("mdev" if mdev else "pci", fname, n)
                res["rows"][name] = {"doc_bytes": len(doc), "parse_device": stats(pd), "parse_call": stats(pw),
                                     "emit_device": stats(ed), "emit_call": stats(ew), "file_read": stats(rd),
                                     "parse_GBps": round(len(doc) / (np.median(pd) * 1e-3) / 1e9, 1)}
                print(name, json.dumps(res["rows"][name]))
    out = json.dumps(res)
    print(out)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(out)
    kx.close()


if __name__ == "__main__":
    main()
