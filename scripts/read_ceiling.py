"""Read ceiling of the H100 for the pci.ids parse: how fast the parse kernel's own copy pattern reads the x1000 text
(cfg4, 1 458 186 000 B in HBM) when it does no parse work, how fast variants of it read (one change at a time), and
how fast a plain grid-stride LDG.128 read does.  The kernels are in scripts/read_ceiling.cu, compiled here with nvcc
for sm_90a into a temporary directory.  Every variant is warmed up, then the variants are launched in turn, one
launch each per round, timed with CUDA events.  Prints one JSON line: the card (name, power limit, SM clock, read in
this run) and per variant the CTAs/SM it runs at, bytes read and GB/s (median and best over the rounds).
Compare `a_parse_staging` with `kernel_ms.parse` of bench.py (what the per-chunk work costs) and with the best of
the others (what restaging can win).
usage: python scripts/read_ceiling.py [--rounds 30] [--warmup 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

COPIES = 1000
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))


def build(tmp):
    so = os.path.join(tmp, "libread_ceiling.so")
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared",
                           "-Xcompiler", "-fPIC", "-o", so, os.path.join(ROOT, "scripts", "read_ceiling.cu")])
    L = C.CDLL(so)
    L.rc_variant_name.restype = C.c_char_p
    L.rc_variant_name.argtypes = [C.c_int]
    L.rc_ctas_per_sm.argtypes = [C.c_int]
    L.rc_setup.argtypes = [C.c_void_p, C.c_ulonglong]
    L.rc_bytes.restype = C.c_ulonglong
    L.rc_bytes.argtypes = [C.c_int]
    L.rc_time.restype = C.c_float
    L.rc_time.argtypes = [C.c_int]
    L.rc_last_error.restype = C.c_char_p
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30, help="timed launches per variant (variants alternate)")
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    from kxpu_b200 import workloads as W
    text = np.tile(np.frombuffer(W.load_pci_ids(), np.uint8), COPIES)
    before = card()
    with tempfile.TemporaryDirectory(prefix="kxpu_read_ceiling_") as tmp:
        L = build(tmp)
        rc = L.rc_setup(text.ctypes.data, len(text))
        if rc != 0:
            sys.exit("read_ceiling: set-up failed (%d): no GPU?" % rc)
        nv = L.rc_num_variants()
        names = [L.rc_variant_name(v).decode() for v in range(nv)]
        for v in range(nv):
            for _ in range(args.warmup):
                if L.rc_time(v) < 0:
                    sys.exit("read_ceiling: %s failed: %s" % (names[v], L.rc_last_error().decode()))
        ms = [[] for _ in range(nv)]
        for _ in range(args.rounds):
            for v in range(nv):
                t = L.rc_time(v)
                if t < 0:
                    sys.exit("read_ceiling: %s failed: %s" % (names[v], L.rc_last_error().decode()))
                ms[v].append(t)
        res = {}
        for v in range(nv):
            b = L.rc_bytes(v)
            gbs = sorted(b / (t * 1e-3) / 1e9 for t in ms[v])
            res[names[v]] = {"ctas_per_sm": L.rc_ctas_per_sm(v), "bytes": b, "launches": len(ms[v]),
                             "ms_median": float(np.median(ms[v])), "gbs_median": float(np.median(gbs)),
                             "gbs_best": gbs[-1], "gbs_spread": gbs[-1] - gbs[0]}
        L.rc_teardown()
    after = card()
    print(json.dumps({"card": before, "sm_clock_after": after["clocks.sm"], "text_bytes": len(text),
                      "rounds": args.rounds, "variants": res}))


if __name__ == "__main__":
    main()
