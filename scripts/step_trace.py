"""Kernel trace of the N = 1 bench step (bench.py): one kxpu_pciids_join_device call on the x1000 pci.ids text with
the 2^20 cfg4 keys (make_queries(present, 2^20, 2)), then the table's free.  Stage timing is off, so the trace holds
the step exactly as bench.py times it.  torch.profiler (CUDA activities) records the library's kernels; printed:
  - per kernel: launches, mean / min device time;
  - per step: first kernel start -> last kernel end (arena_reset_kernel, enqueued by the free, is not part of it);
  - the gaps between a step's kernels, and from one step's last kernel to the next step's first.
usage: python scripts/step_trace.py [--steps 50] [--warmup 10] [--out DIR]"""
import argparse
import collections
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

COPIES = 1000
NQ = 1 << 20
PREFIXES = ("kxparse", "kxsmall")  # namespaces of libkxpu.so's pci.ids kernels
RESET = "arena_reset_kernel"


def short(name):
    return name.split("(")[0].split("<")[0].replace("void ", "").strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for the chrome trace and summary.json (default: a new temporary one)")
    args = ap.parse_args()
    if args.out is None:
        args.out = tempfile.mkdtemp(prefix="kxpu_step_trace_")

    import torch
    from torch.profiler import ProfilerActivity, profile
    import kxpu_b200 as K
    from kxpu_b200 import workloads as W

    kx = K.Kxpu(0)  # raises without an H100
    torch.zeros(1, device="cuda")  # a CUDA context for the profiler's activity tracing
    text = W.load_pci_ids()
    t1 = kx.pciids_load(np.frombuffer(text, np.uint8))
    present, _, _ = kx.table_export(t1)
    t1.free()
    keys = W.make_queries(present, NQ, 2)
    n = len(text) * COPIES
    d_text = kx.dev_alloc(n)
    kx.upload(d_text, np.tile(np.frombuffer(text, np.uint8), COPIES))
    d_keys = kx.dev_alloc(NQ * 4)
    kx.upload(d_keys, keys)
    d_rows = kx.dev_alloc(NQ * 4)

    kx.set_stage_timing(False)
    for _ in range(args.warmup):
        kx.pciids_join_device(d_text, n, d_keys, NQ, d_rows).free()
    kx.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            kx.pciids_join_device(d_text, n, d_keys, NQ, d_rows).free()
        kx.sync()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "step.pt.trace.json")
    prof.export_chrome_trace(path)
    for p in (d_text, d_keys, d_rows):
        kx.dev_free(p)
    kx.close()

    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    ks = sorted(((float(e["ts"]), float(e["dur"]), short(e["name"])) for e in ev
                 if e.get("cat") == "kernel" and short(e["name"]).startswith(PREFIXES)), key=lambda k: k[0])
    if not ks:
        sys.exit("step_trace: the profiler recorded none of libkxpu.so's kernels")
    # a step = the kernels from one parse to the next arena reset (the free after the call)
    steps, cur = [], []
    for k in ks:
        if k[2].endswith(RESET):
            if cur:
                steps.append(cur)
            cur = []
        else:
            cur.append(k)
    if cur:
        steps.append(cur)
    if len(steps) != args.steps:
        sys.exit("step_trace: found %d steps in the trace, expected %d" % (len(steps), args.steps))

    per = collections.OrderedDict()
    for ts, dur, name in ks:
        per.setdefault(name, []).append(dur)
    print("# N = 1 bench step: kxpu_pciids_join_device, x1000 text (%d B), %d keys; %d steps, stage timing off" % (n, NQ, args.steps))
    print("%-48s %7s %10s %10s" % ("kernel", "count", "mean_us", "min_us"))
    for name, d in per.items():
        print("%-48s %7d %10.2f %10.2f" % (name[:48], len(d), np.mean(d), np.min(d)))
    span = [s[-1][0] + s[-1][1] - s[0][0] for s in steps]
    print("step (first kernel start -> last kernel end): mean %.2f us, min %.2f us, max %.2f us"
          % (np.mean(span), np.min(span), np.max(span)))
    names = [k[2] for k in steps[0]]
    same = all([k[2] for k in s] == names for s in steps)
    if same:
        print("gaps inside a step (previous kernel end -> kernel start), mean / min us:")
        for i in range(1, len(names)):
            g = [s[i][0] - (s[i - 1][0] + s[i - 1][1]) for s in steps]
            print("  %-44s %8.2f %8.2f" % ("-> " + names[i][:41], np.mean(g), np.min(g)))
    else:
        print("steps differ in their kernel sequence (retries): no per-position gaps")
    between = [steps[i + 1][0][0] - (steps[i][-1][0] + steps[i][-1][1]) for i in range(len(steps) - 1)]
    if between:
        print("step end -> next step start (host round trip, arena_reset_kernel): mean %.2f us, min %.2f us"
              % (np.mean(between), np.min(between)))
    summary = {"steps": args.steps, "kernels": {k: {"count": len(v), "mean_us": float(np.mean(v)), "min_us": float(np.min(v))}
                                                for k, v in per.items()},
               "step_us": {"mean": float(np.mean(span)), "min": float(np.min(span))},
               "between_steps_us": float(np.mean(between)) if between else None, "sequence": names if same else None}
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print("trace and summary.json in %s" % args.out)


if __name__ == "__main__":
    main()
