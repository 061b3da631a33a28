"""Reduced-resolution transcode against restricted decode + encode, on the GPU.

For the 8K 12-bit 5/3 + RCT lossless stream at skipped_res 1 and 2, and the 4K 12-bit 9/7 q90 stream at skipped_res 1,
with input and output resident in device memory (CUDA tensors): Encoder.from_codestream(src, skipped_res=r).transcode
without a target and with 1/4 and 1/16 of the reduced output's size as targets; in the same run the alternative path,
a Decoder restricted to (r, r) decoding into a CUDA tensor, then an Encoder (the input's coding parameters with r fewer
levels, on the reduced image) encoding that tensor with the same target.  Medians after warm-up of the whole call
(host clock around a call that ends in a device synchronise) and of the stages (CUDA events).  Prints the GPU's name,
power limit and SM clocks, read in the same run, next to the numbers.

    python tools/reduce_probe.py [--reps 7] [--warmup 2]
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
    ("8k_rev_rct", dict(width=8192, height=8192, num_comps=3, bit_depth=12, num_decomps=5, reversible=True, color_transform=True), (1, 2)),
    ("4k_irv_q90", dict(width=4096, height=4096, num_comps=3, bit_depth=12, num_decomps=5, reversible=False, color_transform=True, qfactor=90), (1,)),
]


def _ms(x):
    return round(float(x), 3)


def timed(call, stage_of, reps, warmup):
    import torch
    wall, st, out = [], [], None
    for i in range(warmup + reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = call()
        torch.cuda.synchronize()
        if i >= warmup:
            wall.append((time.perf_counter() - t0) * 1e3)
            st.append(stage_of())
    med = {k: _ms(np.median([s[k] for s in st])) for k in st[0]}
    return _ms(np.median(wall)), med, out


def enc_stages(enc, target):
    t = enc.timings()
    st = dict(parse_host=t["host_ms"], block_decode_or_dwt=t["dwt"], headers=t["assemble"])
    if target:
        r = enc.rate_info()["ms"]
        st.update(candidates=r["distortion"] + r["candidates"], selection=r["selection"], final_coding=r["final_encode"])
    else:
        st.update(block_coding=t["ht_encode"])
    return st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card (name, power limit, SM clock, max SM clock):", card, flush=True)
    for name, kw, rs in FRAMES:
        p = cases.make(kw)
        base = cs.Encoder(p).encode(cases.frame_for(p))
        src = torch.from_numpy(np.frombuffer(base, np.uint8).copy()).cuda()
        for r in rs:
            t = cs.Encoder.from_codestream(src, skipped_res=r)
            plain = t.transcode(src)
            rkw = dict(kw, width=-(-kw["width"] // (1 << r)), height=-(-kw["height"] // (1 << r)), num_decomps=kw["num_decomps"] - r)
            rp = cases.make(rkw)
            e = cs.Encoder(rp)
            d = cs.Decoder()
            img = torch.empty((p.num_comps, rkw["height"], rkw["width"]), dtype=torch.int32, device="cuda")
            view = cs._tensor_image(img, "chw", cs.I32, e.dims)

            def decode_encode():
                d.read_headers_device(src.data_ptr(), src.numel(), cs.I32)
                d.restrict_input_resolution(r, r)
                d.decode_device(view, torch.cuda.current_stream().cuda_stream)
                return e.encode_tensor(img)

            for label, T in (("none", 0), ("1/4", plain.numel() // 4), ("1/16", plain.numel() // 16)):
                t.set_target_size(T)
                e.set_target_size(T)
                wt, stt, ot = timed(lambda: t.transcode(src), lambda: enc_stages(t, T), a.reps, a.warmup)
                wd, std, od = timed(decode_encode, lambda: dict(decode=sum(d.timings()[k] for k in ("h2d", "host_parse", "ht_decode", "dwt_inv")),
                                                                **{"encode_" + k: v for k, v in enc_stages(e, T).items()}), a.reps, a.warmup)
                print(json.dumps(dict(frame=name, skipped_res=r, input_bytes=len(base), target=label, target_bytes=int(T),
                                      transcode_ms=wt, decode_encode_ms=wd, transcode_bytes=int(ot.numel()),
                                      decode_encode_bytes=int(od.numel()), identical=bool(ot.numel() == od.numel() and torch.equal(ot, od)),
                                      transcode_stages=stt, decode_encode_stages=std, card=card)), flush=True)
            t.close()
            e.close()
            d.close()


if __name__ == "__main__":
    main()
