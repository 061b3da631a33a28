"""Tile sharding of one image over ranks (SURVEY §8(e)): the C++ of ojb_shard.cpp -- every rank keeps one encoder /
decoder with the whole image's geometry and a tile mask, the transport is behind callbacks.  CPU tier: world_size 2
over gloo, kernels under the SIMT emulator, against the reference's codestream and decode.  GPU tier: the same worker
with the nvcc-built library and two processes on one device (tests/test_zz_regions_gpu.py); tools/shard_check.py runs
larger frames over NCCL under torchrun."""
import os
import sys
import numpy as np
import cases
import openjph_b200 as ob
from openjph_b200 import sharding
from test_regions import _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TILED = dict(width=300, height=200, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, color_transform=True,
             tile=(128, 128), tlm=True)
TILED_OFF = dict(width=300, height=200, num_comps=1, bit_depth=8, num_decomps=3, reversible=True, tile=(128, 100),
                 offset=(7, 5), tile_offset=(3, 2), tilepart_div=1)
TILED_SUB = dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=2, reversible=True, tile=(96, 64),
                 subsampling=[(1, 1), (2, 2), (2, 2)], planar=1)

# (parameters, writer rank); the last one (six 256x256 tiles of a 12-bit frame) runs on the GPU tier only
TILE_CASES = [
    (TILED, 0),
    (TILED_OFF, 1),
    (TILED_SUB, 0),
    (dict(width=256, height=192, num_comps=3, bit_depth=12, num_decomps=3, reversible=False, color_transform=True,
          qstep=0.002, tile=(128, 96)), 0),
    (dict(width=700, height=500, num_comps=3, bit_depth=12, num_decomps=4, reversible=True, color_transform=True,
          tile=(256, 256), tlm=True), 0),
]


def _native_worker(rank, world, port, q, which, gpu=False):
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), OJB_EMU_THREADS="2")
    import ctypes
    import torch.distributed as dist
    import refharness
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        if gpu:
            # the nvcc-built library on cuda:0, both processes on the one device; the transport callbacks stage device
            # buffers through host memory and gloo
            L = None
        else:
            import emu
            L = emu.emu_lib(build=False)
        ok, notes = True, []
        for ci in which:
            kw, writer = TILE_CASES[ci]
            p = cases.make(kw)
            frame = cases.frame_for(p)
            if rank == writer:
                print("tile case %d: %dx%dx%d %d-bit, %d levels, %s, tiles %dx%d, writer %d" % (
                    ci, p.width, p.height, p.num_comps, p.bit_depth[0], p.num_decomps,
                    "5/3" if p.reversible else "9/7", p.tile_w, p.tile_h, writer), flush=True)
            sh = sharding.NativeShard(lib=L, transport="callbacks" if gpu else None)
            sh.configure(p, ob.I32, writer=writer)
            for rep in range(2):                   # a second frame through the same objects
                fr = frame if rep == 0 else [np.ascontiguousarray(a[::-1]) for a in frame]
                cs = sh.encode(fr)
                want = refharness.encode(p, fr) if rank == writer else None
                if rank == writer:
                    if p.reversible:
                        good = cs == want
                    else:
                        good = len(cs) == len(want) and cs[:cs.index(b"\xff\x90")] == want[:want.index(b"\xff\x90")]
                    if not good:
                        notes.append("case %d rep %d: encode differs (%d vs %d bytes)" % (ci, rep, len(cs), len(want)))
                    ok = ok and good
                else:
                    ok = ok and cs is None
                planes = sh.decode(want, sample_type=ob.I32, writer=writer)
                if rank == writer:
                    ref_planes, _ = refharness.decode(want)
                    tol = 0 if p.reversible else 1
                    err = max(int(np.abs(a.astype(np.int64) - b).max()) for a, b in zip(planes, ref_planes))
                    if p.reversible:                # lossless: the input frame itself
                        err = max([err] + [int(np.abs(a.astype(np.int64) - b).max()) for a, b in zip(planes, fr)])
                    if err > tol:
                        notes.append("case %d rep %d: decode off by %d" % (ci, rep, err))
                    ok = ok and err <= tol
                else:
                    ok = ok and planes is None
            # device-resident forms (under the emulator "device" memory is host memory: read it back directly)
            sh.upload(frame)
            addr, n = sh.encode_resident()
            want = refharness.encode(p, frame) if rank == writer else None
            if rank == writer and p.reversible:
                good = (n == len(want)) if gpu else (ctypes.string_at(addr, n) == want)
                if not good:
                    notes.append("case %d: resident encode differs" % ci)
                ok = ok and good
            lens = [n]
            dist.broadcast_object_list(lens, src=writer)
            sh.decode_resident(addr, lens[0], ob.I32, writer)
            if rank == writer and not gpu:       # (device memory on a GPU: the host-buffer forms above already compared samples)
                ref_planes, _ = refharness.decode(want if p.reversible else ctypes.string_at(addr, n))
                for c, rp in enumerate(ref_planes):
                    got = np.frombuffer(ctypes.string_at(sh.device_plane(c), rp.size * 4), np.int32).reshape(rp.shape)
                    good = np.abs(got.astype(np.int64) - rp).max() <= (0 if p.reversible else 1)
                    if not good:
                        notes.append("case %d: resident decode differs in component %d" % (ci, c))
                    ok = ok and good
            sh.close()
        q.put((rank, bool(ok), notes))
    except BaseException as e:              # the parent must hear about it instead of waiting for its timeout
        import traceback
        q.put((rank, False, ["rank %d: %r\n%s" % (rank, e, traceback.format_exc()[-1500:])]))
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_gloo_world2_native_shard(emu_lib, ref):
    """world_size 2 over gloo: the C++ sharded encoder / decoder (tile masks, size allgather, tile-part and sample
    gathers through the transport callbacks) against the reference's codestream and decode"""
    _run(2, [0, 1, 2, 3], worker=_native_worker)
