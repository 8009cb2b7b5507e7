"""Device time of the any-vendor discovery calls next to the NVIDIA-only ones (DESIGN.md K5 / K6):
kxpu_classify vs kxpu_classify_rules([10de/vfio-pci]) on cfg3, alternating; kxpu_classify_rules with five rules
on xpu_records; kxpu_cdi_emit vs kxpu_cdi_emit_kind on cfg5 with a short and a 63-byte kind.  Kernel times come
from the library's per-stage CUDA events.  Prints one JSON object (and writes it to argv[1] when given)."""
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
    return {"median_ms": round(float(np.median(v)), 4), "min_ms": round(float(v.min()), 4), "max_ms": round(float(v.max()), 4),
            "p10_ms": round(float(np.percentile(v, 10)), 4), "p90_ms": round(float(np.percentile(v, 90)), 4), "n": len(v)}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    kx = K.Kxpu(0)
    keys = kx.table_export(kx.pciids_load(W.load_pci_ids()))[0]
    cfg3 = W.cfg3_records(keys)
    xpu = W.xpu_records(keys)
    cfg5 = W.cfg5_devices()
    nv = [(b"10de", b"vfio-pci")]
    t = {}

    def kernel_ms(stage, fn):
        fn()
        return kx.timings()[stage]
    for _ in range(3):  # warm-up
        kx.classify(cfg3); kx.classify_rules(nv, cfg3); kx.classify_rules(W.XPU_RULES, xpu)
    a, b = [], []
    for _ in range(REPS):
        a.append(kernel_ms(B.T_CLASSIFY, lambda: kx.classify(cfg3)))
        b.append(kernel_ms(B.T_CLASSIFY, lambda: kx.classify_rules(nv, cfg3)))
    t["classify_cfg3"] = stats(a)
    t["classify_rules_nvidia_cfg3"] = stats(b)
    t["classify_rules_5_xpu_records"] = stats([kernel_ms(B.T_CLASSIFY, lambda: kx.classify_rules(W.XPU_RULES, xpu)) for _ in range(REPS)])
    kind63 = "v" + "e" * 22 + ".example/" + "c" + "l" * 29 + "9"
    for fmt, name in ((B.FMT_JSON, "json"), (B.FMT_YAML, "yaml")):
        for _ in range(3):
            kx.cdi_emit(fmt, cfg5); kx.cdi_emit(fmt, cfg5, kind="amd.com/gpu"); kx.cdi_emit(fmt, cfg5, kind=kind63)
        e0, e1, e2 = [], [], []
        for _ in range(REPS):
            e0.append(kernel_ms(B.T_EMIT, lambda: kx.cdi_emit(fmt, cfg5)))
            e1.append(kernel_ms(B.T_EMIT, lambda: kx.cdi_emit(fmt, cfg5, kind="amd.com/gpu")))
            e2.append(kernel_ms(B.T_EMIT, lambda: kx.cdi_emit(fmt, cfg5, kind=kind63)))
        t["cdi_emit_%s_cfg5" % name] = stats(e0)
        t["cdi_emit_kind_amd_%s_cfg5" % name] = stats(e1)
        t["cdi_emit_kind_63B_%s_cfg5" % name] = stats(e2)
    out = {"gpu": smi.stdout.strip(), "reps": REPS, "timings": t}
    s = json.dumps(out, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
