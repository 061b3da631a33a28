"""Per-frame time of the device-image entry points against the copy + resident forms they replace, on one GPU.

Encode:  A = copy a CHW tensor into the encoder's image buffer (ojb_enc_device_plane) + ojb_enc_encode_resident;
         B = ojb_enc_encode_device from the CHW tensor;  C = the same from an HWC tensor.
Decode:  A = ojb_dec_decode_resident + a device-to-device copy into a CHW tensor;
         B = ojb_dec_decode_device into a CHW tensor;  C = the same into an HWC tensor.
The codestream stays in device memory throughout.  Every call returns with its output complete, so a host clock
around it times the frame.  A, B and C alternate inside one run; each figure is the median over --reps frames after
--warmup frames of each.  Prints the card, its power limit and SM clock from the same run, and one JSON line.

  python tools/device_image_probe.py [--size 8192] [--reps 9] [--warmup 3] [--irv]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


class _Raw:
    """a device pointer as a tensor (the codec's own image planes)"""
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = dict(shape=shape, typestr=typestr, data=(ptr, False), version=3, strides=None)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--irv", action="store_true", help="9/7 + ICT q90 instead of 5/3 + RCT")
    a = ap.parse_args()
    import torch
    import images
    import openjph_b200 as ob
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this probe measures on the GPU only")
    W = H = a.size
    kw = dict(num_decomps=5, reversible=not a.irv, color_transform=True)
    if a.irv:
        kw["qfactor"] = 90
    p = ob.make_params(W, H, 3, 12, **kw)
    frame = [f.astype(np.uint16) for f in images.synth_frame(W, H, 3, 12, 5)]
    chw16 = torch.stack([torch.from_numpy(f.view(np.int16)).cuda() for f in frame])
    chw = chw16.view(torch.uint16)
    hwc = chw16.permute(1, 2, 0).contiguous().view(torch.uint16)
    enc, dec = ob.Encoder(p, ob.U16), ob.Decoder()
    L = enc.L
    cap = enc._out.size
    dev_cs = torch.empty(cap + 64, dtype=torch.uint8, device="cuda")
    own = [torch.as_tensor(_Raw(L.ojb_enc_device_plane(enc.h, c), (H, W), "<i2"), device="cuda") for c in range(3)]
    n = C.c_uint64()

    def enc_a():
        for c in range(3):
            own[c].copy_(chw16[c])
        torch.cuda.current_stream().synchronize()
        assert L.ojb_enc_encode_resident(enc.h, dev_cs.data_ptr(), cap, C.byref(n), 1) == 0, L.ojb_last_error()
        return int(n.value)

    def enc_b():
        return enc.encode_tensor(chw, out=dev_cs)

    def enc_c():
        return enc.encode_tensor(hwc, layout="hwc", out=dev_cs)

    nbytes = enc_b()
    ref_cs = dev_cs[:nbytes].cpu().numpy().tobytes()
    for f in (enc_a, enc_c):
        assert f() == nbytes and dev_cs[:nbytes].cpu().numpy().tobytes() == ref_cs, f.__name__
    dec.read_headers_device(dev_cs.data_ptr(), nbytes, ob.U16)
    dplanes = [torch.as_tensor(_Raw(L.ojb_dec_device_plane(dec.h, c), (H, W), "<i2"), device="cuda") for c in range(3)]
    out_chw = torch.empty((3, H, W), dtype=torch.int16, device="cuda")
    out_hwc = torch.empty((H, W, 3), dtype=torch.int16, device="cuda")
    cs_img = ob.codestream._tensor_image(out_chw.view(torch.uint16), "chw", ob.U16, [(W, H)] * 3)
    hwc_img = ob.codestream._tensor_image(out_hwc.view(torch.uint16), "hwc", ob.U16, [(W, H)] * 3)
    sh = torch.cuda.current_stream().cuda_stream

    def dec_a():
        assert L.ojb_dec_decode_resident(dec.h) == 0, L.ojb_last_error()
        for c in range(3):
            out_chw[c].copy_(dplanes[c])
        torch.cuda.current_stream().synchronize()

    def dec_b():
        dec.decode_device(cs_img, sh)

    def dec_c():
        dec.decode_device(hwc_img, sh)

    dec_b()
    ref = out_chw.clone()
    dec_c()
    assert torch.equal(out_hwc.permute(2, 0, 1), ref)
    dec_a()
    assert torch.equal(out_chw, ref)

    fns = dict(enc_copy_resident=enc_a, enc_device_chw=enc_b, enc_device_hwc=enc_c,
               dec_resident_copy=dec_a, dec_device_chw=dec_b, dec_device_hwc=dec_c)
    times = {k: [] for k in fns}
    for i in range(a.warmup + a.reps):
        for k, f in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            if i >= a.warmup:
                times[k].append((time.perf_counter() - t0) * 1e3)
    card = _card()
    res = dict(card=card, torch_device=torch.cuda.get_device_name(0), frame="%dx%dx3 12-bit %s" % (W, H, "9/7 ICT q90" if a.irv else "5/3 RCT"),
               codestream_bytes=nbytes, reps=a.reps, warmup=a.warmup,
               median_ms={k: round(float(np.median(v)), 3) for k, v in times.items()},
               min_ms={k: round(float(np.min(v)), 3) for k, v in times.items()})
    print("card (name, power limit, SM clock, max SM clock):", card)
    for k in fns:
        print("%-20s median %8.3f ms  min %8.3f ms" % (k, res["median_ms"][k], res["min_ms"][k]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
