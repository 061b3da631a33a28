#!/usr/bin/env python3
"""Stage times of encoding to a target size on the 8192x8192x3 12-bit headline frame (a real GPU only).

For 5/3 + RCT and 9/7 + ICT: an unconstrained resident encode, then encodes at 1/4, 1/16 and 1/64 of the lossless
(5/3) size, each with its stage times (distortion, candidate lengths, selection rounds, final block coding; CUDA events),
the whole encode call (host clock around a call that ends in a device synchronise), the stream size, the selection
rounds, the share of blocks left out, and the decode time of the stream.  Whether truncated blocks still take the fast
decoder (missing MSBs + 2 <= 16) is printed as the largest missing-MSB count in the stream.
usage: python tools/rate_probe.py [--size 8192] [--reps 5]
"""
import argparse
import json
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


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); r = fn(); ts.append((time.perf_counter() - t0) * 1e3)
    return r, float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    n = a.size
    frame = images.synth_frame(n, n, 3, 12, 1234)
    lossless = None
    for name, kw in (("5/3+RCT", dict(reversible=True)), ("9/7+ICT", dict(reversible=False))):
        p = ob.make_params(n, n, 3, 12, num_decomps=5, color_transform=True, **kw)
        enc = cs.Encoder(p)
        enc.upload(frame)
        full, ms_full = timed(enc.encode_resident, a.reps)
        if lossless is None:
            lossless = len(full)
        dec = cs.Decoder()
        _, ms_dec = timed(lambda: dec.decode(full), a.reps)
        print(json.dumps(dict(config=name, target="none", bytes=len(full), encode_ms=round(ms_full, 3), decode_ms=round(ms_dec, 3),
                              stages=enc.timings())))
        for div in (4, 16, 64):
            T = lossless // div
            if T >= len(full):
                continue
            enc.set_target_size(T)
            j2c, ms = timed(enc.encode_resident, a.reps)
            info = enc.rate_info()
            _, ms_d = timed(lambda: dec.decode(j2c), a.reps)
            mm = max(int(b.missing_msbs) for b in dec.list_blocks() if b.len1)
            print(json.dumps(dict(config=name, target="lossless/%d" % div, T=T, bytes=len(j2c), encode_ms=round(ms, 3),
                                  decode_ms=round(ms_d, 3), rounds=info["rounds"],
                                  left_out=round(float(np.mean(info["k"] == info["kmax"])), 4), max_missing_msbs=mm,
                                  rate_ms={k: round(v, 3) for k, v in info["ms"].items()})))
        enc.set_target_size(0)
        enc.close(); dec.close()


if __name__ == "__main__":
    main()
