"""Device time of kxpu_aer_ports (DESIGN.md K19) next to kxpu_pcie_ports (one group per record) on the same walk of 2^20
functions, and of kxpu_aer_health with and without the ports as members, each pair alternated.  Walks
(workloads.aer_port_walk): switch trees two levels deep with fan-out 8, every chain end in turn (a function below the
host bridge, the root port, a switch upstream and a switch downstream port: "mixed"), and three levels deep with fan-out
4 (every function below a downstream port: seven ports each).  The AER files are workloads.aer_records' for the
functions and zero-count files for the ports; a group is one function, with its ports after it.  40 calls each; kernel
times from the library's KXPU_T_CLASSIFY CUDA events, median [p10, p90].  The card's name and power limit are read in
the same run.  Prints one JSON object (and writes it to argv[1] when given)."""
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


def pair(kx, fa, fb):
    """alternated device times of two calls"""
    for _ in range(3):
        fa(); fb()
    a, b = [], []
    for _ in range(REPS):
        fa(); a.append(kx.timings()[B.T_CLASSIFY])
        fb(); b.append(kx.timings()[B.T_CLASSIFY])
    return stats(a), stats(b)


def health_inputs(n, off, of, n_ports):
    """kxpu_aer_health's inputs for n functions and n_ports ports: (text, file_off, file_len, groups without ports,
    groups with them)"""
    a = W.aer_records(n)
    zf, zn = W.aer_file("TOTAL_ERR_FATAL", [0] * 18), W.aer_file("TOTAL_ERR_NONFATAL", [0] * 18)
    base = len(a["text"])
    text = a["text"] + zf + zn
    file_off = np.concatenate([a["file_off"], np.tile(np.array([base, base + len(zf)], np.uint64), n_ports)])
    file_len = np.concatenate([a["file_len"], np.tile(np.array([len(zf), len(zn)], np.uint32), n_ports)])
    plain = (np.arange(n + 1, dtype=np.uint32), np.arange(n, dtype=np.uint32))
    cnt = np.diff(off).astype(np.int64) + 1
    goff = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
    mem = np.empty(int(goff[-1]), np.uint32)
    mem[goff[:-1]] = np.arange(n, dtype=np.uint32)
    rest = np.ones(len(mem), bool)
    rest[goff[:-1]] = False
    mem[rest] = n + of
    return text, file_off, file_len, plain, (goff, mem)


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    kx = K.Kxpu(0)
    n = 1 << 20
    res = {"gpu": smi.stdout.strip(), "reps": REPS, "n_records": n, "walks": {}}
    for name, depth, fanout, mixed in (("mixed_depth2_fanout8", 2, 8, True), ("depth3_fanout4", 3, 4, False)):
        recs, paths = W.aer_port_walk(n, depth=depth, fanout=fanout, mixed=mixed)
        goff, gmem = np.arange(n + 1, dtype=np.uint32), np.arange(n, dtype=np.uint32)
        ta, tb = pair(kx, lambda: kx.aer_ports(recs, paths), lambda: kx.pcie_ports(recs, paths, goff, gmem))
        off, of, key = kx.aer_ports(recs, paths)
        text, fo, fl, plain, ported = health_inputs(n, off, of, len(key))
        ha, hb = pair(kx, lambda: kx.aer_health(text, fo, fl, 0, 0, *ported), lambda: kx.aer_health(text, fo, fl, 0, 0, *plain))
        res["walks"][name] = {
            "aer_ports": ta, "pcie_ports": tb, "ratio": round(ta["median_ms"] / tb["median_ms"], 3),
            "positions": int(off[-1]), "distinct_ports": int(len(key)),
            "aer_health_with_ports": ha, "aer_health_members_only": hb,
            "health_ratio": round(ha["median_ms"] / hb["median_ms"], 3), "health_members": int(len(ported[1]))}
    s = json.dumps(res, indent=1)
    print(s)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(s)
    kx.close()


if __name__ == "__main__":
    main()
