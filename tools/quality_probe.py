#!/usr/bin/env python3
"""Stage times and results of encoding to a target quality on the 8192x8192x3 12-bit frame (a real GPU only).

For 5/3 + RCT and 9/7 + ICT q90, at 40, 45 and 50 dB PSNR (peak 4095), and for 9/7 also at 30, 33 and 35.5 dB (this
frame's 9/7 q90 quantisation floor lies near 36.6 dB, so the higher targets end on the floor path): resident encodes (the
frame in device memory, the codestream copied back), after --warmup frames, --reps timed frames.  Per target it prints
the measured rounds, the median CUDA-event stage times (candidates: distortion + candidate lengths; rounds: hull,
bracket and every measured round; final block coding: the code-block encoder on the chosen selection -- packet headers
and layout are not in it), the median whole call (host clock around a call that ends in a device synchronise), the PSNR and bytes of the stream, and what the model alone gave: the measured PSNR of round 1's
selection (the model's proposal before any correction) and the PSNR the model predicted for it.  The unconstrained
encode of each configuration is timed the same way.  The card's name, power limit and maximum SM clock come from the
same run.  --json writes every number to a file.
usage: python tools/quality_probe.py [--size 8192] [--reps 5] [--warmup 2] [--json out.json]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [_ROOT, os.path.join(_ROOT, "tests")]
import openjph_b200 as ob                          # noqa: E402
from openjph_b200 import codestream as cs         # noqa: E402
import images                                      # noqa: E402


def psnr(sse, n, peak):
    return float("inf") if sse == 0 else 10.0 * math.log10(peak * peak * n / float(sse))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print("card (name, power limit, max SM clock):", card[0] if card else "nvidia-smi unavailable")
    n = a.size
    frame = images.synth_frame(n, n, 3, 12, 1234)
    peak = 4095.0
    out = dict(card=card[0] if card else None, size=n, reps=a.reps, warmup=a.warmup, results=[])
    for name, kw in (("5/3+RCT", dict(reversible=True)), ("9/7+ICT q90", dict(reversible=False, qfactor=90))):
        p = ob.make_params(n, n, 3, 12, num_decomps=5, color_transform=True, **kw)
        enc = cs.Encoder(p)
        enc.upload(frame)
        for _ in range(a.warmup):
            enc.encode_resident()
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter(); full = enc.encode_resident(); ts.append((time.perf_counter() - t0) * 1e3)
        base = dict(config=name, target_db=None, bytes=len(full), call_ms=float(np.median(ts)))
        print("%-12s unconstrained: %d bytes, call %.2f ms" % (name, len(full), base["call_ms"]))
        out["results"].append(base)
        for db in (40.0, 45.0, 50.0) + (() if kw["reversible"] else (30.0, 33.0, 35.5)):
            enc.set_target_psnr(db)
            for _ in range(a.warmup):
                enc.encode_resident()
            ts, st, rounds = [], [], []
            for _ in range(a.reps):
                t0 = time.perf_counter(); j2c = enc.encode_resident(); ts.append((time.perf_counter() - t0) * 1e3)
                q = enc.quality_info()
                st.append([q["ms"]["candidates"], q["ms"]["rounds"], q["ms"]["final_encode"]])
                rounds.append(len(q["rounds"]))
            med = np.median(np.array(st), axis=0)
            N = q["num_samples"]
            r1 = q["rounds"][0] if q["rounds"] else None
            res = dict(config=name, target_db=db, bytes=len(j2c), reached=q["reached"], psnr=psnr(q["sse"], N, peak),
                       rounds=rounds, keys=[r["key"] for r in q["rounds"]], call_ms=float(np.median(ts)),
                       candidates_ms=float(med[0]), rounds_ms=float(med[1]), final_ms=float(med[2]),
                       round1_psnr=psnr(r1["sse"], N, peak) if r1 else None, round1_bytes=r1["body"] if r1 else None,
                       round1_model_psnr=psnr(q["model_round1"], N, peak) if r1 else None)
            out["results"].append(res)
            print("%-12s %4.1f dB: %s %.3f dB, %d bytes, rounds %s | candidates %.2f ms, rounds %.2f ms, final block coding %.2f ms, "
                  "call %.2f ms | round 1 (model only): %.3f dB measured, %.3f dB predicted, %s body bytes"
                  % (name, db, "reached" if q["reached"] else "NOT reached", res["psnr"], len(j2c), rounds,
                     res["candidates_ms"], res["rounds_ms"], res["final_ms"], res["call_ms"],
                     res["round1_psnr"] or 0, res["round1_model_psnr"] or 0, res["round1_bytes"]))
        enc.close()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
