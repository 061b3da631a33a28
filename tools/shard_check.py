#!/usr/bin/env python3
"""torchrun entry: tile-sharded encode/decode over NCCL (sharding.NativeShard with the tile partition; BASELINE
configs[3]: 8192x8192x3 16-bit, reversible 5/3, 4 tiles of 4096^2 sharded over the ranks).  Checks on rank 0 that the
gathered codestream is identical to the one-GPU codestream (and, at 2048^2 tiles, to the reference's) and that the
sharded decode is lossless."""
import os, sys, time, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist
import openjph_b200 as ob
from openjph_b200 import sharding, _lib
from openjph_b200.codestream import comp_dims
import images

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
L = _lib.lib(); assert L.ojb_set_device(local) == 0
res = {}
for name, W, T, bd, vs_ref in (("4k_2048tiles_ref", 4096, 2048, 12, True), ("cfg4_8k16_4tiles", 8192, 4096, 16, False)):
    p = ob.make_params(W, W, 3, bd, num_decomps=5, reversible=True, color_transform=True, tile=(T, T), tlm=True)
    frame = [f.astype(np.uint16) for f in images.synth_frame(W, W, 3, bd, 77)]
    sh = sharding.NativeShard()
    sh.set_partition("tiles")
    sh.configure(p, ob.U16, writer=0)
    cs = sh.encode(frame)                                       # first frame: arenas, descriptor tables
    dist.barrier(); torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(3):
        cs = sh.encode(frame)
    torch.cuda.synchronize(); dist.barrier(); t1 = time.perf_counter()
    t2 = time.perf_counter()
    planes = sh.decode(cs, dims=comp_dims(p), sample_type=ob.U16, writer=0)   # the codestream is needed on the writer only
    dist.barrier(); t3 = time.perf_counter()
    sh.close()
    if rank == 0:
        one = ob.Encoder(p, ob.U16).encode(frame)
        ok = cs == one and all(np.array_equal(a, b) for a, b in zip(planes, frame))
        if vs_ref:
            import refharness
            if refharness.available():
                ok = ok and cs == refharness.encode(p, [f.astype(np.int32) for f in frame])
        res[name] = dict(identical=bool(ok), bytes=len(cs), encode_s=round((t1 - t0) / 3, 3), decode_s=round(t3 - t2, 3), ranks=world)
if rank == 0:
    print(json.dumps(res))
dist.destroy_process_group()
sys.exit(0 if rank != 0 or all(v["identical"] for v in res.values()) else 1)
