"""Device time of the vGPU discovery calls next to the PCI ones (DESIGN.md K5 / K6): kxpu_classify_mdev on
mdev_records (2^20 records, four rules) alternating with kxpu_classify on cfg3, and kxpu_cdi_emit_mdev alternating
with kxpu_cdi_emit_kind on 65 536 devices, 40 calls each.  Kernel times come from the library's per-stage CUDA
events.  Prints the card and its power limit and one JSON object (also written to argv[1] when given)."""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import kxpu_b200 as K  # noqa: E402
from kxpu_b200 import binding as B, workloads as W  # noqa: E402

REPS = 40


def stats(v):
    v = np.asarray(v)
    return {"median_ms": round(float(np.median(v)), 4), "p10_ms": round(float(np.percentile(v, 10)), 4),
            "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("card:", smi.stdout.strip())
    kx = K.Kxpu(0)
    keys = kx.table_export(kx.pciids_load(W.load_pci_ids()))[0]
    cfg3 = W.cfg3_records(keys)
    mrecs = W.mdev_records()
    cfg5 = W.cfg5_devices()
    mdevs = W.mdev_devices()
    t = {}

    def kernel_ms(stage, fn):
        fn()
        return kx.timings()[stage]
    for _ in range(3):  # warm-up
        kx.classify(cfg3); kx.classify_mdev(W.MDEV_RULES, mrecs)
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(B.T_CLASSIFY, lambda: kx.classify(cfg3)))
        b.append(kernel_ms(B.T_CLASSIFY, lambda: kx.classify_mdev(W.MDEV_RULES, mrecs)))
    t["classify_cfg3"] = stats(a)
    t["classify_mdev_4_rules_mdev_records"] = stats(b)
    for fmt, name in ((B.FMT_JSON, "json"), (B.FMT_YAML, "yaml")):
        for kind in ("nvidia.com/gpu", "v" + "e" * 22 + ".example/" + "c" + "l" * 29 + "9"):
            for _ in range(3):
                kx.cdi_emit(fmt, cfg5, kind=kind); kx.cdi_emit_mdev(fmt, mdevs, kind)
            e0, e1 = [], []
            for _ in range(REPS):
                e0.append(kernel_ms(B.T_EMIT, lambda: kx.cdi_emit(fmt, cfg5, kind=kind)))
                e1.append(kernel_ms(B.T_EMIT, lambda: kx.cdi_emit_mdev(fmt, mdevs, kind)))
            tag = "%dB_%s" % (len(kind), name)
            t["cdi_emit_kind_%s_65536" % tag] = stats(e0)
            t["cdi_emit_mdev_%s_65536" % tag] = stats(e1)
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "timings": t}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
