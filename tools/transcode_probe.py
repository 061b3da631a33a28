"""Transcode against decode + encode-to-target, on the GPU.

For the 8K 12-bit 5/3 + RCT frame (its lossless stream) and the 4K 9/7 q90 frame (its stream), with input and output
resident in device memory (CUDA tensors): transcodes to 1/4, 1/16 and 1/64 of the lossless size and at 40, 45 and 50 dB,
and in the same run encodes of the image with the same targets.  Medians after warm-up of the whole call (host clock
around a call that ends in a device synchronise) and of the stages (CUDA events): parse (host), input block decode
(the transform's place; the forward DWT for an encode), candidates, selection or rounds, final coding, headers.  For the
lossless input the two paths must give byte-identical streams.  Prints the GPU's name, power limit and clock next to
the numbers.

    python tools/transcode_probe.py [--reps 7] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import cases  # noqa: E402
from openjph_b200 import codestream as cs  # noqa: E402

FRAMES = [
    ("8k_rev_rct", dict(width=8192, height=8192, num_comps=3, bit_depth=12, num_decomps=5, reversible=True, color_transform=True)),
    ("4k_irv_q90", dict(width=4096, height=4096, num_comps=3, bit_depth=12, num_decomps=5, reversible=False, color_transform=True, qfactor=90)),
]


def stages(enc, quality):
    t = enc.timings()
    st = dict(parse_host=t["host_ms"], block_decode_or_dwt=t["dwt"], headers=t["assemble"])
    if quality:
        q = enc.quality_info()["ms"]
        st.update(candidates=q["candidates"], rounds=q["rounds"], final_coding=q["final_encode"])
    else:
        r = enc.rate_info()["ms"]
        st.update(candidates=r["distortion"] + r["candidates"], selection=r["selection"], final_coding=r["final_encode"])
    return st


def timed(call, enc, quality, reps, warmup):
    import torch
    wall, st, out = [], [], None
    for i in range(warmup + reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = call()
        torch.cuda.synchronize()
        if i >= warmup:
            wall.append((time.perf_counter() - t0) * 1e3)
            st.append(stages(enc, quality))
    med = {k: float(np.median([s[k] for s in st])) for k in st[0]}
    return float(np.median(wall)), med, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip())
    for name, kw in FRAMES:
        p = cases.make(kw)
        frame = cases.frame_for(p)
        img = torch.stack([torch.from_numpy(np.ascontiguousarray(f, np.int32)) for f in frame]).cuda()
        base = cs.Encoder(p).encode(frame)
        lossless = bool(p.reversible)
        src = torch.from_numpy(np.frombuffer(base, np.uint8).copy()).cuda()
        targets = [("size", len(base) // d) for d in (4, 16, 64)] + [("psnr", db) for db in (40.0, 45.0, 50.0)]
        for kind, v in targets:
            q = kind == "psnr"
            kwargs = dict(target_psnr=v) if q else dict(target_bytes=v)
            e = cs.Encoder(p, **kwargs)
            t = cs.Encoder.from_codestream(src, **kwargs)
            we, se, oe = timed(lambda: e.encode_tensor(img), e, q, a.reps, a.warmup)
            wt, stt, ot = timed(lambda: t.transcode(src), t, q, a.reps, a.warmup)
            same = bool(torch.equal(oe, ot)) if oe.numel() == ot.numel() else False
            if lossless:
                assert same, (name, kind, v)
            print(json.dumps(dict(frame=name, input_bytes=len(base), target=kind, value=v, encode_ms=round(we, 3),
                                  transcode_ms=round(wt, 3), encode_bytes=int(oe.numel()), transcode_bytes=int(ot.numel()),
                                  identical=same, encode_stages={k: round(x, 3) for k, x in se.items()},
                                  transcode_stages={k: round(x, 3) for k, x in stt.items()})), flush=True)
            e.close()
            t.close()


if __name__ == "__main__":
    main()
