"""Device time of kxpu_classify_named (DESIGN.md K5) on xpu_records(2^20) -- several device ids under five vendors --
with a name table of a "*" entry and listed ids, alternated with kxpu_classify_rules and kxpu_classify_vf_vgpu (no
vGPU rule) on the same records.  40 calls each; kernel times from the library's per-stage CUDA events (KXPU_T_CLASSIFY),
median [p10, p90].  The card's name and power limit are read in the same run.  Prints one JSON object (and writes it to
argv[1] when given)."""
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
    kx = K.Kxpu(0)
    keys = kx.table_export(kx.pciids_load(W.load_pci_ids()))[0]  # the (vendor, device) keys pci.ids lists
    recs, rules = W.xpu_records(keys, 1 << 20), W.XPU_RULES
    # listed ids: the first eight 4-digit ids of rules 0 and 1 in the walk, two per name; "*" for the rest of rule 0
    ids = []
    for r in recs[:1 << 14]:
        v, d = bytes(r["vendor_txt"])[2:6], bytes(r["device_txt"])[2:6]
        rule = [k for k, (rv, _) in enumerate(rules) if rv == v]
        if rule and rule[0] < 2 and int(r["device_len"]) == 7 and (rule[0], d) not in ids:
            ids.append((rule[0], d))
        if len(ids) == 8:
            break
    table = [(r, d, k // 2) for k, (r, d) in enumerate(ids)] + [(0, b"*", 4)]
    fns = {"named": lambda: kx.classify_named(rules, 0, recs, None, table),
           "rules": lambda: kx.classify_rules(rules, recs),
           "vf_vgpu": lambda: kx.classify_vf_vgpu(rules, 0, recs, None)}
    for f in fns.values():
        f()
    t = {k: [] for k in fns}
    for _ in range(REPS):
        for k, f in fns.items():
            f()
            t[k].append(kx.timings()[B.T_CLASSIFY])
    c = fns["named"]()
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "n_records": len(recs), "n_names": len(table),
           "n_devids": {"named": int(c["n_devids"]), "rules": int(fns["rules"]()["n_devids"])},
           "device": {k: stats(v) for k, v in t.items()}}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
