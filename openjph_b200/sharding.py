"""One image across the GPUs of a box (one process per GPU, torch.distributed): the ctypes wrapper of ojb_shard.cpp.

Every rank keeps ONE encoder / decoder with the geometry of the whole image, so canvas coordinates, Isot and packet
contents are those of a single encoder and the codestream on the writer rank is byte-identical to the one-GPU stream.
Two partitions (NativeShard.set_partition):
  "tiles"    rank r codes the tiles t with t % world == r (a tile mask).  Tiles are independent through colour
             transform, DWT, quantisation, block coding and packet formation -- the reference gives every tile its own
             component / resolution tree (src/core/codestream/ojph_codestream_local.cpp:132-168) and concatenates the
             tile-parts in tile-index order at flush (:1148-1164).  Encode gathers the tile-parts to the writer, which
             adds the main header (+TLM) and EOC; decode sends each rank's tile samples to the writer.
  "regions"  every tile-component is cut into `world` row slabs, each rank reading its slab plus a halo, so a
             single-tile image is split too; the code-block bytes go to the writer, which writes packet headers and
             markers as one encoder does (DESIGN.md §5).

Transport: NCCL inside the library, or callbacks over a torch.distributed process group (gloo) -- the CPU test tier's
emulator build, and two processes on one GPU in the GPU test tier.
"""
import ctypes as C
import struct
import numpy as np
from . import _lib
from . import codestream as cs_mod

SIZ = 0xFF51


def siz_params(header):
    """image / tile geometry and sub-sampling out of the SIZ segment (enough for comp_dims)"""
    if struct.unpack(">H", header[2:4])[0] != SIZ:
        raise cs_mod.OjphError("SIZ must follow SOC")
    x1, y1, x0, y0, tw, th, gx, gy, nc = struct.unpack(">IIIIIIIIH", header[8:42])
    p = _lib.Params()
    p.width, p.height, p.off_x, p.off_y = x1, y1, x0, y0
    p.tile_w, p.tile_h, p.tile_off_x, p.tile_off_y = tw, th, gx, gy
    p.num_comps = nc
    for c in range(nc):
        ss, dx, dy = struct.unpack(">BBB", header[42 + 3 * c:45 + 3 * c])
        p.bit_depth[c] = (ss & 0x7F) + 1
        p.is_signed[c] = ss >> 7
        p.dx[c], p.dy[c] = dx, dy
    return p


def _dist():
    import torch.distributed as dist
    return dist


class NativeShard:
    """One per rank.  Wraps ojb_shard: every rank keeps one encoder / decoder with the geometry of the whole image
    and a tile mask; tile-parts (encode) and decoded tile samples (decode) go device to device to the writer rank.
    Transport: NCCL inside the library (product path: the unique id is handed out through torch.distributed), or --
    when `lib` is the SIMT-emulator build of the CPU test tier, which has no NCCL -- callbacks over the process
    group (gloo), where "device" memory is host memory."""

    def __init__(self, group=None, lib=None, transport=None):
        """transport: None = NCCL inside the library (callbacks when `lib` is the emulator build); "callbacks" = the
        callback transport over the process group also with the product library -- device buffers are staged through
        host memory (cudaMemcpy), which lets two processes on ONE GPU run the sharded paths over gloo (GPU test tier)"""
        import torch
        dist = _dist()
        self.L = lib if lib is not None else _lib.lib()
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self._keep = None
        self._staged = lib is None and transport == "callbacks"
        if lib is None and transport != "callbacks":
            uid = torch.zeros(128, dtype=torch.uint8)
            if self.rank == 0:
                buf = (C.c_uint8 * 128)()
                if self.L.ojb_shard_unique_id(buf) != 0:
                    raise cs_mod.OjphError(self.L.ojb_shard_last_error().decode(errors="replace"))
                uid = torch.tensor(list(buf), dtype=torch.uint8)
            dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
            uid = uid.to(dev)
            dist.broadcast(uid, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
            ub = (C.c_uint8 * 128)(*uid.cpu().tolist())
            self.h = self.L.ojb_shard_create_nccl(self.rank, self.world, ub)
        else:
            self._keep = self._gloo_callbacks()
            self.h = self.L.ojb_shard_create(self.rank, self.world, C.byref(self._keep[0]))
        if not self.h:
            raise cs_mod.OjphError(self.L.ojb_shard_last_error().decode(errors="replace"))
        self.info = None

    def _gloo_callbacks(self):
        import torch
        dist = _dist()
        group = self.group

        def view(ptr, n):
            return torch.from_numpy(np.frombuffer((C.c_uint8 * n).from_address(ptr), np.uint8)) if n else torch.zeros(0, dtype=torch.uint8)

        cudart = None
        if self._staged:
            cudart = C.CDLL("libcudart.so.12")
            cudart.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
            cudart.cudaMemcpy.restype = C.c_int

        def pull(ptr, n):            # device (or, under the emulator, host) buffer -> host tensor
            if not self._staged:
                return view(ptr, n).clone()
            t = torch.empty(n, dtype=torch.uint8)
            if n and cudart.cudaMemcpy(t.data_ptr(), ptr, n, 2) != 0:
                raise RuntimeError("cudaMemcpy D2H")
            return t

        def push(ptr, t):            # host tensor -> device buffer
            if t.numel() and cudart.cudaMemcpy(ptr, t.data_ptr(), t.numel(), 1) != 0:
                raise RuntimeError("cudaMemcpy H2D")
            # a copy from pageable memory returns once the bytes are staged, not once they are on the device, and the
            # library reads them on its own non-blocking stream
            if cudart.cudaDeviceSynchronize() != 0:
                raise RuntimeError("cudaDeviceSynchronize")

        def grank(r):
            return dist.get_global_rank(group, r) if group is not None else r

        def allgather(ctx, send, recv, n):
            try:
                out = list(view(recv, n * self.world).split(n))
                dist.all_gather(out, view(send, n).clone(), group=group)
                return 0
            except Exception:
                return 1

        def bcast(ctx, buf, n, root):
            try:
                if not self._staged:
                    dist.broadcast(view(buf, n), src=grank(root), group=group)
                else:
                    t = pull(buf, n) if self.rank == root else torch.empty(n, dtype=torch.uint8)
                    dist.broadcast(t, src=grank(root), group=group)
                    if self.rank != root:
                        push(buf, t)
                return 0
            except Exception:
                return 1

        def send(ctx, buf, n, peer):
            try:
                dist.send(pull(buf, n), dst=grank(peer), group=group)
                return 0
            except Exception:
                return 1

        def recv(ctx, buf, n, peer):
            try:
                if not self._staged:
                    dist.recv(view(buf, n), src=grank(peer), group=group)
                else:
                    t = torch.empty(n, dtype=torch.uint8)
                    dist.recv(t, src=grank(peer), group=group)
                    push(buf, t)
                return 0
            except Exception:
                return 1

        fns = (_lib.CB_ALLGATHER(allgather), _lib.CB_BCAST(bcast), _lib.CB_SENDRECV(send), _lib.CB_SENDRECV(recv))
        cb = _lib.CommCallbacks(None, *fns)
        return cb, fns

    def _check(self, rc):
        if rc != 0:
            raise cs_mod.OjphError(self.L.ojb_shard_last_error().decode(errors="replace"))

    def close(self):
        if self.h:
            self.L.ojb_shard_destroy(self.h)
            self.h = None

    def set_partition(self, kind):
        """0 / "tiles": rank r codes the tiles t % world == r (default); 1 / "regions": every tile-component is cut into
        `world` row slabs (input halo, no mid-pipeline exchange) -- this also splits a single-tile image.  Call it on
        every rank before configure() / decode()."""
        k = {"tiles": 0, "regions": 1}.get(kind, kind)
        self._check(self.L.ojb_shard_set_partition(self.h, int(k)))

    def region_rows(self, comp=0):
        """row regions, after configure(): image rows [lo, hi) of component comp this rank's encoder reads"""
        lo, hi = C.c_uint32(), C.c_uint32()
        if not self.L.ojb_shard_region_rows(self.h, comp, C.byref(lo), C.byref(hi)):
            return None
        return int(lo.value), int(hi.value)

    def configure(self, p, sample_type=cs_mod.I32, writer=0):
        self.p, self.sample_type, self.writer = p, sample_type, writer
        self._check(self.L.ojb_shard_enc_configure(self.h, C.byref(p), sample_type, writer))
        dims = cs_mod.comp_dims(p)
        self._out = np.empty(sum(w * h for w, h in dims) * 5 + (1 << 20), np.uint8) if self.rank == writer else np.empty(16, np.uint8)

    def encode(self, planes):
        """planes: the whole image (every rank); returns the codestream on the writer, None elsewhere"""
        arrs = [np.ascontiguousarray(a, cs_mod._NP[self.sample_type]) for a in planes]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        n = C.c_uint64()
        self._check(self.L.ojb_shard_enc_encode(self.h, ptrs, None, self._out.ctypes.data, self._out.size, C.byref(n)))
        return self._out[:n.value].tobytes() if self.rank == self.writer else None

    def decode(self, cs, dims=None, sample_type=cs_mod.I32, writer=0):
        """cs: the codestream (needed on the writer only); dims: [(w, h)] of the components when known, else read
        from the headers by a first call; returns the planes on the writer, None elsewhere"""
        fi = _lib.FrameInfo()
        buf = np.frombuffer(cs, np.uint8) if (cs is not None and self.rank == writer) else np.zeros(1, np.uint8)
        n = buf.size if self.rank == writer else 0
        if dims is None:
            # geometry first (every rank needs its plane sizes on the writer only; a header-only decode would do, the
            # call is collective so all ranks take this path together)
            hdr = [None]
            if self.rank == writer:
                hdr[0] = bytes(cs[:1 << 16])
            _dist().broadcast_object_list(hdr, src=_dist().get_global_rank(self.group, writer) if self.group is not None else writer, group=self.group)
            dims = cs_mod.comp_dims(siz_params(hdr[0]))
        planes = [np.zeros((h, w), cs_mod._NP[sample_type]) for w, h in dims] if self.rank == writer else None
        ptrs = (C.c_void_p * len(dims))(*[a.ctypes.data for a in planes]) if planes is not None else None
        self._check(self.L.ojb_shard_dec_decode(self.h, buf.ctypes.data, n, sample_type, writer, ptrs, None, C.byref(fi)))
        self.info = fi
        return planes

    # ---- device-resident forms (tiles uploaded once per rank; codestream and decoded image stay on the writer's device)
    def upload(self, planes):
        arrs = [np.ascontiguousarray(a, cs_mod._NP[self.sample_type]) for a in planes]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        self._check(self.L.ojb_shard_enc_upload(self.h, ptrs, None))

    def encode_resident(self):
        """-> (device address of the codestream on the writer, length); (None, 0) elsewhere"""
        n = C.c_uint64()
        self._check(self.L.ojb_shard_enc_encode_resident(self.h, C.byref(n)))
        return (self.L.ojb_shard_device_codestream(self.h), int(n.value)) if self.rank == self.writer else (None, 0)

    def decode_resident(self, dev_ptr, length, sample_type=cs_mod.I32, writer=0):
        """codestream at dev_ptr on the writer; decoded planes stay in the writer's device image buffer
        (device_plane(c)); returns the frame info"""
        fi = _lib.FrameInfo()
        self._check(self.L.ojb_shard_dec_decode_resident(self.h, dev_ptr, length, sample_type, writer, C.byref(fi)))
        self.info = fi
        return fi

    def device_plane(self, comp):
        return self.L.ojb_shard_device_plane(self.h, comp)

    @property
    def timings(self):
        t = (C.c_float * 2)()
        self.L.ojb_shard_timings(self.h, t)
        return {"codec_ms": t[0], "gather_ms": t[1]}
