"""Host-side mirror of the reference's encode / decode interface for the GPU path.

`Encoder` follows ojph::codestream's write side (access_siz/cod/qcd setters -> write_headers ->
exchange loop -> flush; src/core/openjph/ojph_codestream.h:88-383) and `Decoder` its read side
(read_headers -> create -> pull loop); both also expose the frame-at-once calls the C-ABI adds.
Argument meaning and error behaviour follow the reference: invalid settings raise
`OjphError` carrying the reference's error code where it has one.
"""
import ctypes as C
import numpy as np
from . import _lib

U8, U16, I32 = 0, 1, 2
_NP = {U8: np.uint8, U16: np.uint16, I32: np.int32}
PROG = {"LRCP": 0, "RLCP": 1, "RPCL": 2, "PCRL": 3, "CPRL": 4}


RASTER = {"pnm": 0, "yuv": 1, "dpx_be": 2, "dpx_le": 3}


class OjphError(RuntimeError):
    pass


def make_params(width, height, num_comps=1, bit_depth=8, is_signed=False, num_decomps=5, block=(64, 64),
                reversible=True, color_transform=False, prog_order="RPCL", qstep=-1.0, qfactor=0,
                tile=(0, 0), offset=(0, 0), tile_offset=(0, 0), precincts=None, subsampling=None,
                tlm=False, tilepart_div=0, planar=-1, coc=None, nlt=None, profile=None, qcc=None, decomp=None, atk=None):
    p = _lib.Params()
    p.width, p.height = width, height
    p.off_x, p.off_y = offset
    p.tile_w, p.tile_h = tile
    p.tile_off_x, p.tile_off_y = tile_offset
    p.num_comps = num_comps
    bds = bit_depth if isinstance(bit_depth, (list, tuple)) else [bit_depth] * num_comps
    sgs = is_signed if isinstance(is_signed, (list, tuple)) else [is_signed] * num_comps
    for c in range(num_comps):
        p.bit_depth[c] = bds[c]
        p.is_signed[c] = 1 if sgs[c] else 0
        p.dx[c], p.dy[c] = (subsampling[c] if subsampling else (1, 1))
    p.num_decomps = num_decomps
    p.block_w, p.block_h = block
    if precincts:
        p.num_precincts = len(precincts)
        for i, (w, h) in enumerate(precincts):
            p.precinct_w[i], p.precinct_h[i] = w, h
    p.reversible = 1 if reversible else 0
    p.color_transform = 1 if color_transform else 0
    p.prog_order = PROG[prog_order] if isinstance(prog_order, str) else prog_order
    p.qstep = qstep
    p.qfactor = qfactor
    p.tlm = 1 if tlm else 0
    p.tilepart_div = tilepart_div
    p.planar = planar
    # per-component coding styles: {comp: dict(reversible=, num_decomps=, block=)}; as in the reference a
    # component's COC starts from the library defaults (5 levels, 64x64, irreversible)
    for c in range(16):
        p.coc_num_decomps[c], p.coc_block_w[c], p.coc_block_h[c] = 5, 64, 64
    for c, st in (coc or {}).items():
        p.coc_present[c] = 1
        p.coc_reversible[c] = 1 if st.get("reversible", False) else 0
        p.coc_num_decomps[c] = st.get("num_decomps", 5)
        p.coc_block_w[c], p.coc_block_h[c] = st.get("block", (64, 64))
        for i, (pw, ph) in enumerate(st.get("precincts", [])):
            p.coc_precinct_w[c][i], p.coc_precinct_h[c][i] = pw, ph
        p.coc_num_precincts[c] = len(st.get("precincts", []))
    p.profile = {None: 0, "IMF": 1, "BROADCAST": 2}[profile]          # codestream::set_profile
    # per-component quantisation calls in order: [("qstep", comp, delta) | ("qfactor", comp, ctype, q), ...]
    for seq, call in enumerate(qcc or [], start=1):
        c = call[1]
        if call[0] == "qstep":
            p.qcc_calls[c] |= 1; p.qcc_qstep[c] = call[2]; p.qcc_qstep_seq[c] = seq
        else:
            p.qcc_calls[c] |= 2; p.qcc_ctype[c], p.qcc_qfactor[c] = call[2], call[3]; p.qcc_qfactor_seq[c] = seq
    # Part 2 structures (encoder extension; the reference only reads them): decomp = "BHVHB" or [1, 2, 3, ...] per
    # level, finest first (B both ways, H horizontal only, V vertical only); atk = dict(reversible=False, K=..., A=[...])
    # or dict(reversible=True, steps=[(a, b, e), ...]), lifting steps in synthesis order
    if decomp:
        kinds = [{"X": 0, "B": 1, "H": 2, "V": 3}[d] if isinstance(d, str) else int(d) for d in decomp]
        p.dfs_num_levels = len(kinds)
        for i, k in enumerate(kinds):
            p.dfs_type[i] = k
    if atk:
        if atk.get("reversible", False):
            p.atk_reversible = 1
            p.atk_num_steps = len(atk["steps"])
            for i, (a, b, e) in enumerate(atk["steps"]):
                p.atk_a[i], p.atk_b[i], p.atk_e[i] = a, b, e
        else:
            p.atk_num_steps = len(atk["A"])
            p.atk_K = atk["K"]
            for i, a in enumerate(atk["A"]):
                p.atk_A[i] = a
    # param_nlt::set_nonlinear_transform calls, in order: {"all": 3, 1: 0, ...} (types 0 and 3)
    for seq, (c, t) in enumerate((nlt or {}).items()):
        if c == "all":
            p.nlt_all = 1 + t
        else:
            p.nlt_comp[c], p.nlt_seq[c] = 1 + t, seq
    return p


def device_image(comps):
    """an ojb_device_image from [(address, row_pitch_bytes, col_stride), ...], one entry per component"""
    img = _lib.DeviceImage()
    for c, (addr, pitch, col) in enumerate(comps):
        img.base[c], img.row_pitch[c], img.col_stride[c] = addr, pitch, col
    return img


_TORCH_DTYPE = {U8: "uint8", U16: "uint16", I32: "int32"}


def _tensor_image(t, layout, sample_type, dims):
    """the ojb_device_image of a CUDA tensor: (C, H, W) for "chw", (H, W, C) for "hwc", any strides (a channels_last
    view, batch[i], a window of a larger canvas); or a list of 2-D tensors, one per component (sub-sampled
    components).  Components past the coded ones (an alpha channel) are left alone."""
    import torch
    want = getattr(torch, _TORCH_DTYPE[sample_type])
    if isinstance(t, (list, tuple)):
        planes = list(t)
    else:
        if layout not in ("chw", "hwc"):
            raise ValueError("layout is 'chw' or 'hwc', not %r" % (layout,))
        if t.dim() != 3:
            raise ValueError("a %s image tensor has 3 dimensions, this one has %d" % (layout, t.dim()))
        v = t.permute(2, 0, 1) if layout == "hwc" else t
        planes = [v[c] for c in range(v.shape[0])]
    if len(planes) < len(dims):
        raise ValueError("%d components coded, the tensor holds %d" % (len(dims), len(planes)))
    comps = []
    for c, (w, h) in enumerate(dims):
        p = planes[c]
        if not p.is_cuda:
            raise ValueError("component %d is not a CUDA tensor" % c)
        if p.dtype != want:
            raise ValueError("component %d is %s; the codec's sample container is %s" % (c, p.dtype, want))
        if tuple(p.shape) != (h, w):
            raise ValueError("component %d is %s, the codestream's is (%d, %d)" % (c, tuple(p.shape), h, w))
        comps.append((p.data_ptr(), p.stride(0) * p.element_size(), p.stride(1)))
    return device_image(comps)


def comp_dims(p):
    def dc(a, b):
        return (a + b - 1) // b
    return [(dc(p.width, p.dx[c]) - dc(p.off_x, p.dx[c]), dc(p.height, p.dy[c]) - dc(p.off_y, p.dy[c]))
            for c in range(p.num_comps)]


def _siz_of(head):
    """(component sizes [(w, h)], bit depths) from a codestream's SIZ segment, which follows SOC"""
    b = bytes(head)
    if len(b) < 42 or b[0:4] != b"\xff\x4f\xff\x51":
        raise OjphError("not a codestream: no SOC and SIZ at its start")
    u32 = lambda o: int.from_bytes(b[o:o + 4], "big")
    X, Y, XO, YO = u32(8), u32(12), u32(16), u32(20)
    nc = int.from_bytes(b[40:42], "big")
    dims, depths = [], []
    for c in range(nc):
        s, dx, dy = b[42 + 3 * c], b[43 + 3 * c], b[44 + 3 * c]
        dims.append((-(-X // dx) - -(-XO // dx), -(-Y // dy) - -(-YO // dy)))
        depths.append((s & 0x7F) + 1)
    return dims, depths


class _Base:
    def __init__(self, lib=None):
        self.L = lib if lib is not None else _lib.lib()

    def _check(self, rc):
        if rc != 0:
            raise OjphError(self.L.ojb_last_error().decode(errors="replace"))


class Encoder(_Base):
    def __init__(self, params, sample_type=I32, lib=None, comments=None, target_bytes=None, target_mse=None,
                 target_psnr=None):
        """comments: the extra COM segments of write_headers(file, comments, n): bytes (binary) or str (text);
        target_bytes: every frame call returns a codestream of at most this many bytes (see set_target_size);
        target_mse / target_psnr: every frame call returns a codestream whose decoded error is within this mean squared
        error / at least this PSNR (see set_target_mse, set_target_psnr)"""
        super().__init__(lib)
        self.h = self.L.ojb_enc_create()
        if not self.h:
            raise OjphError(self.L.ojb_last_error().decode(errors="replace"))
        self.params = params
        self.sample_type = sample_type
        if comments:
            keep = [c.encode("latin-1") if isinstance(c, str) else bytes(c) for c in comments]
            arr = (_lib.Comment * len(keep))()
            bufs = [C.create_string_buffer(k, len(k)) for k in keep]
            for i, c in enumerate(comments):
                arr[i].data, arr[i].len, arr[i].rcom = C.addressof(bufs[i]), len(keep[i]), 1 if isinstance(c, str) else 0
            self._check(self.L.ojb_enc_set_comments(self.h, arr, len(keep)))
        self._check(self.L.ojb_enc_configure(self.h, C.byref(params), sample_type))
        self.dims = comp_dims(params)
        cap = sum(w * h for w, h in self.dims) * 4 + (1 << 20)
        self._out = np.empty(cap, np.uint8)
        if target_bytes:
            self.set_target_size(target_bytes)
        if target_mse is not None:
            self.set_target_mse(target_mse)
        if target_psnr is not None:
            self.set_target_psnr(target_psnr)

    def set_target_size(self, nbytes):
        """cap every following codestream at nbytes (0: no target).  Each code-block is coded at the bit-plane a
        rate-distortion selection on the GPU chooses; a target at or above the unconstrained size changes nothing."""
        self._check(self.L.ojb_enc_set_target_size(self.h, int(nbytes)))

    @property
    def min_size(self):
        """the smallest codestream of this geometry (every code-block left out): the lowest target accepted"""
        n = C.c_uint64()
        self._check(self.L.ojb_enc_min_size(self.h, C.byref(n)))
        return int(n.value)

    def set_target_mse(self, mse):
        """bound the decoded error of every following codestream (0: no target): the squared error of the decoded
        samples against the source, summed over every sample of every component, is at most floor(mse * N), N the
        number of samples.  The search measures each candidate selection by reconstructing it on the GPU as the decoder
        would; it returns the smallest stream it finds within the limit.  Below the quantisation floor of an
        irreversible configuration, the unconstrained stream comes back with quality_info()["reached"] False."""
        self._check(self.L.ojb_enc_set_target_mse(self.h, float(mse)))

    def set_target_psnr(self, db):
        """set_target_mse for a PSNR in dB, peak 2^B - 1; every component must have the same bit depth B (a
        transcoder takes B from the codestream's headers)"""
        if self.params is None:
            depths = set(self._depths)
        else:
            depths = {int(self.params.bit_depth[c]) for c in range(self.params.num_comps)}
        if len(depths) != 1:
            raise ValueError("a PSNR target needs one bit depth for every component (have %s)" % sorted(depths))
        peak = float((1 << depths.pop()) - 1)
        self.set_target_mse(peak * peak / 10.0 ** (float(db) / 10.0))

    @classmethod
    def from_codestream(cls, j2c, sample_type=I32, target_bytes=None, target_mse=None, target_psnr=None, lib=None,
                        skipped_res=0):
        """an encoder configured from a codestream's headers and tile-parts (bytes or a uint8 array in host memory, or
        a 1-D CUDA uint8 tensor), which transcodes: transcode() re-codes such a codestream from its code-blocks,
        single-layer and cleanup-only, with the input's geometry, coding parameters, main header (less TLM / PLM) and
        tile-parts, to the targets given here or set later.  The source of a quality target is the input as the
        Decoder returns it in `sample_type`; target_psnr takes the bit depth from the headers.

        skipped_res=r > 0 drops the input's top r resolution levels (as ojph_expand -skip_res r): the output is the
        reduced-resolution codestream the kept code-blocks make, whose decode equals the input's decode restricted to
        (r, r), and a quality target's source is that restricted decode.  `dims` are the output's component sizes."""
        self = cls.__new__(cls)
        _Base.__init__(self, lib)
        self.h = self.L.ojb_enc_create()
        if not self.h:
            raise OjphError(self.L.ojb_last_error().decode(errors="replace"))
        self.params = None
        self.sample_type = sample_type
        ptr, n, dev, head = self._codestream(j2c)
        if skipped_res == 0:
            self._check(self.L.ojb_enc_transcode_headers(self.h, ptr, n, dev, sample_type))
            self.dims, self._depths = _siz_of(head)
        else:
            info = _lib.FrameInfo()
            self._check(self.L.ojb_enc_transcode_headers_reduced(self.h, ptr, n, dev, sample_type, int(skipped_res),
                                                                 C.byref(info)))
            self.dims = [(int(info.comp_w[c]), int(info.comp_h[c])) for c in range(info.num_comps)]
            self._depths = [int(info.bit_depth[c]) for c in range(info.num_comps)]
        self._out = np.empty(sum(w * h for w, h in self.dims) * 4 + (1 << 20), np.uint8)
        if target_bytes:
            self.set_target_size(target_bytes)
        if target_mse is not None:
            self.set_target_mse(target_mse)
        if target_psnr is not None:
            self.set_target_psnr(target_psnr)
        return self

    def _codestream(self, j2c):
        """(address, length, on device, its first bytes) of a codestream in host memory or in a CUDA uint8 tensor"""
        try:
            import torch
            is_tensor = isinstance(j2c, torch.Tensor)
        except ImportError:
            is_tensor = False
        if is_tensor:
            if not (j2c.is_cuda and j2c.dtype == torch.uint8 and j2c.dim() == 1 and j2c.is_contiguous()):
                raise ValueError("a codestream tensor is a contiguous 1-D CUDA uint8 tensor")
            n = j2c.numel()
            if j2c.untyped_storage().nbytes() - j2c.storage_offset() - n < 32:      # the reader wants 32 bytes of slack
                pad = torch.zeros(n + 32, dtype=torch.uint8, device=j2c.device)
                pad[:n].copy_(j2c)
                j2c = pad[:n]
            # the headers are read on the host: the bytes must be complete before the call
            torch.cuda.current_stream(j2c.device).synchronize()
            self._cs_keep = j2c
            return j2c.data_ptr(), n, 1, j2c[:min(n, 1 << 16)].cpu().numpy().tobytes()
        buf = np.frombuffer(j2c, np.uint8) if not isinstance(j2c, np.ndarray) else np.ascontiguousarray(j2c, np.uint8)
        self._cs_keep = buf
        return buf.ctypes.data, buf.size, 0, buf[:1 << 16].tobytes()

    def transcode(self, j2c, out=None):
        """re-code a codestream (see from_codestream) to the encoder's target.  Host bytes / array in: the codestream
        bytes out.  A CUDA uint8 tensor in: the codestream as a CUDA uint8 tensor, or, with `out` (a CUDA uint8 tensor),
        written there and its length returned; it never leaves the device.  The call returns with the bytes in place."""
        ptr, n, dev, _ = self._codestream(j2c)
        m = C.c_uint64()
        if not dev:
            self._check(self.L.ojb_enc_transcode(self.h, ptr, n, 0, self._out.ctypes.data, self._out.size, C.byref(m), 0))
            return self._out[:m.value].tobytes()
        import torch
        where = j2c.device
        if out is not None:
            if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()):
                raise ValueError("out is a contiguous CUDA uint8 tensor")
            self._check(self.L.ojb_enc_transcode(self.h, ptr, n, 1, out.data_ptr(), out.numel(), C.byref(m), 1))
            return int(m.value)
        stage = getattr(self, "_dev_out", None)
        if stage is None or stage.device != where:
            stage = self._dev_out = torch.empty(self._out.size, dtype=torch.uint8, device=where)
        self._check(self.L.ojb_enc_transcode(self.h, ptr, n, 1, stage.data_ptr(), stage.numel(), C.byref(m), 1))
        res = torch.empty(m.value + 32, dtype=torch.uint8, device=where)     # 32 readable bytes past the end
        res[:m.value].copy_(stage[:m.value])
        return res[:m.value]

    def quality_info(self):
        """the search of the last frame encoded with a target quality: N, the limit floor(mse * N), the exact squared
        error of the returned stream (sse, an int) and per component, reached, the rounds (slope key, measured squared
        error, code-block bytes), the final bracket, the model's prediction for round 1 and the stage times (ms)"""
        q = _lib.QualityInfo()
        self._check(self.L.ojb_enc_quality_info(self.h, C.byref(q)))
        n = q.rounds
        rounds = [dict(key=int(q.round_key[i]), sse=(int(q.round_sse_hi[i]) << 64) | int(q.round_sse_lo[i]),
                       body=int(q.round_body[i])) for i in range(n)]
        return dict(num_samples=int(q.num_samples), limit=int(q.limit), sse=(int(q.sse_hi) << 64) | int(q.sse_lo),
                    comp_sse=list(q.comp_sse)[:q.num_comps], reached=bool(q.reached), rounds=rounds,
                    pass_key=int(q.pass_key), fail_key=int(q.fail_key), pass_body=int(q.pass_body),
                    fail_body=int(q.fail_body), pass_measured=bool(q.pass_measured), fail_measured=bool(q.fail_measured), body0=int(q.body0),
                    model_round1=float(q.model_round1),
                    ms=dict(candidates=q.ms_candidates, rounds=q.ms_rounds, final_encode=q.ms_final))

    def rate_info(self):
        """the selection of the last frame encoded with a target: K_max, chosen k (k == K_max: left out), R[b, k]
        (cleanup bytes; 0xFFFFFFFF: not codable), D[b, k] (weighted squared error, k <= K_max), the final body budget,
        the selection rounds, the header and marker bytes, the stream bytes, the slope-key threshold and the stage
        times (ms)"""
        nb, kc = C.c_uint32(), C.c_uint32()
        self._check(self.L.ojb_enc_rate_info(self.h, C.byref(nb), C.byref(kc), None, None, None, None, None, None))
        n, m = nb.value, kc.value
        kmax, k = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        R, D = np.zeros((n, m), np.uint32), np.zeros((n, m), np.float64)
        info, ms = (C.c_uint64 * 5)(), (C.c_float * 4)()
        self._check(self.L.ojb_enc_rate_info(self.h, C.byref(nb), C.byref(kc), kmax.ctypes.data, k.ctypes.data,
                                             R.ctypes.data, D.ctypes.data, info, ms))
        return dict(kmax=kmax, k=k, R=R, D=D, budget=int(info[0]), rounds=int(info[1]), header_bytes=int(info[2]),
                    total=int(info[3]), threshold=int(info[4]), ms=dict(zip(("distortion", "candidates", "selection", "final_encode"), list(ms))))

    def close(self):
        if self.h:
            self.L.ojb_enc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _planes(self, planes):
        arrs = []
        for c, a in enumerate(planes):
            a = np.ascontiguousarray(a, dtype=_NP[self.sample_type])
            w, h = self.dims[c]
            assert a.shape == (h, w), (a.shape, (h, w))
            arrs.append(a)
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        return arrs, ptrs

    def encode(self, planes):
        """frame-at-once: planes[c] is a (h, w) array; returns the codestream bytes."""
        arrs, ptrs = self._planes(planes)
        n = C.c_uint64()
        self._check(self.L.ojb_enc_encode_frame(self.h, ptrs, None, self._out.ctypes.data, self._out.size, C.byref(n)))
        return self._out[:n.value].tobytes()

    def encode_raster(self, payload, layout="pnm"):
        """a file payload as the reference's apps read it: 'pnm' = interleaved, big-endian 16-bit / 8-bit
        (.pgm / .ppm after the header); 'yuv' = planes one after the other, little-endian (.yuv / .raw)"""
        buf = np.frombuffer(payload, np.uint8)
        n = C.c_uint64()
        self._check(self.L.ojb_enc_encode_raster(self.h, RASTER[layout], buf.ctypes.data, buf.size,
                                                 self._out.ctypes.data, self._out.size, C.byref(n)))
        return self._out[:n.value].tobytes()

    def upload(self, planes):
        arrs, ptrs = self._planes(planes)
        self._check(self.L.ojb_enc_upload_frame(self.h, ptrs, None))

    def encode_resident(self):
        n = C.c_uint64()
        self._check(self.L.ojb_enc_encode_resident(self.h, self._out.ctypes.data, self._out.size, C.byref(n), 0))
        return self._out[:n.value].tobytes()

    def encode_resident_to_device(self, dev_ptr, cap):
        """encode the uploaded frame; the codestream is written to device memory at dev_ptr; returns its length"""
        n = C.c_uint64()
        self._check(self.L.ojb_enc_encode_resident(self.h, dev_ptr, cap, C.byref(n), 1))
        return int(n.value)

    def encode_device(self, image, stream=0, out_ptr=None, out_cap=0):
        """encode from device memory described by `image` (see device_image) after the work queued on the CUDA stream
        handle `stream` (0: the legacy default stream); the codestream comes back as bytes, or goes to device memory
        at out_ptr (capacity out_cap) and its length is returned"""
        n = C.c_uint64()
        if out_ptr is None:
            self._check(self.L.ojb_enc_encode_device(self.h, C.byref(image), stream, self._out.ctypes.data, self._out.size,
                                                     C.byref(n), 0))
            return self._out[:n.value].tobytes()
        self._check(self.L.ojb_enc_encode_device(self.h, C.byref(image), stream, out_ptr, out_cap, C.byref(n), 1))
        return int(n.value)

    def encode_tensor(self, t, layout="chw", stream=None, out=None):
        """encode a frame that is a CUDA tensor (see _tensor_image for the shapes; dtype uint8 / uint16 / int32 as the
        sample container) once the work queued on `stream` (default: torch's current stream) is done.  Returns the
        codestream as a CUDA uint8 tensor, or, with `out` (a CUDA uint8 tensor), writes it there and returns its
        length.  The codestream never leaves the device.  The returned tensor belongs to `stream`: work queued there
        after the call sees it complete."""
        import torch
        img = _tensor_image(t, layout, self.sample_type, self.dims)
        where = (t[0] if isinstance(t, (list, tuple)) else t).device
        s = torch.cuda.current_stream(where) if stream is None else stream
        if out is not None:
            if not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()):
                raise ValueError("out is a contiguous CUDA uint8 tensor")
            return self.encode_device(img, s.cuda_stream, out.data_ptr(), out.numel())
        # one staging buffer per encoder: the same output address every call, so the frame's work replays as a graph.
        # The copy out of it runs on `s`; the next call, whatever stream it names, writes the buffer only after that copy
        dev = getattr(self, "_dev_out", None)
        if dev is None or dev.device != where:
            dev = self._dev_out = torch.empty(self._out.size, dtype=torch.uint8, device=where)
        copied = getattr(self, "_copied", None)
        if copied is not None:
            s.wait_event(copied)
        n = self.encode_device(img, s.cuda_stream, dev.data_ptr(), dev.numel())
        with torch.cuda.stream(s):
            res = torch.empty(n + 32, dtype=torch.uint8, device=where)     # 32 readable bytes past the end
            res[:n].copy_(dev[:n])
        self._copied = torch.cuda.Event()
        self._copied.record(s)
        return res[:n]

    def encode_lines(self, planes):
        """the reference's exchange() loop + flush()."""
        nc = C.c_uint32()
        rows = [0] * len(planes)
        line = self.L.ojb_enc_exchange(self.h, None, C.byref(nc))
        while line:
            c = nc.value
            w, h = self.dims[c]
            buf = np.ctypeslib.as_array(C.cast(line, C.POINTER(C.c_int32)), shape=(w,))
            buf[:] = planes[c][rows[c]]
            rows[c] += 1
            line = self.L.ojb_enc_exchange(self.h, line, C.byref(nc))
        n = C.c_uint64()
        self._check(self.L.ojb_enc_flush(self.h, self._out.ctypes.data, self._out.size, C.byref(n)))
        return self._out[:n.value].tobytes()

    def read_band(self, tile, comp, res, band):
        bw, bh = C.c_uint32(), C.c_uint32()
        self._check(self.L.ojb_enc_read_band(self.h, tile, comp, res, band, None, C.byref(bw), C.byref(bh)))
        out = np.zeros((bh.value, bw.value), np.uint32)
        if out.size:
            self._check(self.L.ojb_enc_read_band(self.h, tile, comp, res, band, out.ctypes.data, C.byref(bw), C.byref(bh)))
        return out

    @property
    def kernel_launches(self):
        return self.L.ojb_enc_kernel_launches(self.h)

    def band_info(self, tile, comp, res, band):
        i8 = (C.c_uint32 * 8)(); d2 = (C.c_float * 2)()
        self._check(self.L.ojb_enc_band_info(self.h, tile, comp, res, band, i8, d2))
        return dict(x0=i8[0], y0=i8[1], w=i8[2], h=i8[3], K_max=i8[4], res_x0=i8[5], res_y0=i8[6], nblocks=i8[7],
                    delta=d2[0], delta_inv=d2[1])

    def timings(self):
        t = (C.c_float * 8)()
        self.L.ojb_enc_timings(self.h, t)
        return dict(zip(("h2d", "dwt", "ht_encode", "d2h_lengths", "host_wait", "assemble", "d2h_out", "host_ms"), list(t)))


class Decoder(_Base):
    def __init__(self, resilient=False, lib=None):
        super().__init__(lib)
        self.h = self.L.ojb_dec_create()
        if not self.h:
            raise OjphError(self.L.ojb_last_error().decode(errors="replace"))
        if resilient:
            self.L.ojb_dec_enable_resilience(self.h)
        self.info = None

    def close(self):
        if self.h:
            self.L.ojb_dec_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def read_headers(self, j2c, sample_type=I32):
        self._buf = np.frombuffer(j2c, np.uint8) if not isinstance(j2c, np.ndarray) else j2c
        self.sample_type = sample_type
        fi = _lib.FrameInfo()
        self._check(self.L.ojb_dec_read_headers(self.h, self._buf.ctypes.data, self._buf.size, sample_type, C.byref(fi)))
        self.info = fi
        return fi

    def read_headers_device(self, dev_ptr, length, sample_type=I32):
        """read_headers for a codestream that is in device memory only (address, byte count)"""
        self.sample_type = sample_type
        fi = _lib.FrameInfo()
        self._check(self.L.ojb_dec_read_headers_device(self.h, dev_ptr, length, sample_type, C.byref(fi)))
        self.info = fi
        return fi

    def decode_device(self, image, stream=0):
        """decode (after read_headers or read_headers_device) into device memory described by `image` (see
        device_image), after the work queued on the CUDA stream handle `stream` (0: the legacy default stream)"""
        self._check(self.L.ojb_dec_decode_device(self.h, C.byref(image), stream))

    def decode_tensor(self, cs, out=None, layout="chw", stream=None, sample_type=None):
        """decode a codestream -- bytes / ndarray in host memory, or a CUDA uint8 tensor, whose body then never leaves
        the device (read_headers_device) -- into the CUDA tensor `out` (see _tensor_image for the shapes), or into a
        new one: (C, H, W) / (H, W, C) when the components share a size, else a list of 2-D tensors.  The container
        follows out's dtype, else sample_type (default I32).  Writing waits for the work queued on `stream` (default:
        torch's current stream); the call returns with the samples in place."""
        import torch
        if sample_type is None:
            sample_type = I32
            if out is not None:
                o = out[0] if isinstance(out, (list, tuple)) else out
                sample_type = {torch.uint8: U8, torch.uint16: U16, torch.int32: I32}.get(o.dtype, I32)
        if isinstance(cs, torch.Tensor):
            if not (cs.is_cuda and cs.dtype == torch.uint8 and cs.dim() == 1 and cs.is_contiguous()):
                raise ValueError("a codestream tensor is a contiguous 1-D CUDA uint8 tensor")
            n = cs.numel()
            if cs.untyped_storage().nbytes() - cs.storage_offset() - n < 32:      # the reader wants 32 bytes of slack
                pad = torch.zeros(n + 32, dtype=torch.uint8, device=cs.device)
                pad[:n].copy_(cs)
                cs = pad[:n]
            # the headers are read on the host: the bytes must be complete before the call
            torch.cuda.current_stream(cs.device).synchronize()
            if stream is not None:
                stream.synchronize()
            self._cs_keep = cs
            self.read_headers_device(cs.data_ptr(), n, sample_type)
        else:
            self.read_headers(cs, sample_type)
        fi = self.info
        dims = [(fi.comp_w[c], fi.comp_h[c]) for c in range(fi.num_comps)]
        s = torch.cuda.current_stream() if stream is None else stream
        if out is None:                    # allocated on `s`, the stream the decoder's writes are ordered after
            dt = getattr(torch, _TORCH_DTYPE[sample_type])
            dev = cs.device if isinstance(cs, torch.Tensor) else torch.device("cuda", torch.cuda.current_device())
            with torch.cuda.stream(s):
                if len(set(dims)) == 1:
                    w, h = dims[0]
                    shape = (len(dims), h, w) if layout == "chw" else (h, w, len(dims))
                    out = torch.empty(shape, dtype=dt, device=dev)
                else:
                    out = [torch.empty((h, w), dtype=dt, device=dev) for w, h in dims]
        self.decode_device(_tensor_image(out, layout, sample_type, dims), s.cuda_stream)
        return out

    @property
    def mirror_bytes(self):
        return int(self.L.ojb_dec_mirror_bytes(self.h))

    def coding_style(self, comp=0):
        """the read-side getters of ojph::param_cod / param_siz for one component (after read_headers)"""
        cs = _lib.CodingStyle()
        self._check(self.L.ojb_dec_get_coding_style(self.h, comp, C.byref(cs)))
        return cs

    def restrict_input_resolution(self, skipped_res_for_read, skipped_res_for_recon):
        """codestream::restrict_input_resolution: after read_headers, before decode"""
        self._check(self.L.ojb_dec_restrict_input_resolution(self.h, skipped_res_for_read, skipped_res_for_recon,
                                                             C.byref(self.info)))
        return self.info

    def decode(self, j2c=None, sample_type=I32, skip=None):
        if j2c is not None:
            self.read_headers(j2c, sample_type)
        if skip is not None:
            self.restrict_input_resolution(*skip)
        fi = self.info
        planes = [np.zeros((fi.comp_h[c], fi.comp_w[c]), _NP[self.sample_type]) for c in range(fi.num_comps)]
        ptrs = (C.c_void_p * fi.num_comps)(*[a.ctypes.data for a in planes])
        self._check(self.L.ojb_dec_decode_frame(self.h, ptrs, None))
        return planes

    def decode_raster(self, j2c=None, layout="pnm", sample_type=None, skip=None):
        """decode into a file payload (see Encoder.encode_raster); returns bytes"""
        if j2c is not None:
            if sample_type is None:                      # the container the file format implies
                fi = self.read_headers(j2c, I32)
                sample_type = U16 if max(fi.bit_depth[c] for c in range(fi.num_comps)) > 8 else U8
            self.read_headers(j2c, sample_type)
        if skip is not None:
            self.restrict_input_resolution(*skip)
        fi = self.info
        es = 2 if self.sample_type == U16 else 1
        cap = sum(fi.comp_w[c] * fi.comp_h[c] for c in range(fi.num_comps)) * es
        out = np.zeros(max(cap, 1), np.uint8)
        n = C.c_uint64()
        self._check(self.L.ojb_dec_decode_raster(self.h, RASTER[layout], out.ctypes.data, cap, C.byref(n)))
        return out[:n.value].tobytes()

    def pull_lines(self, j2c, planar=None):
        """the reference's read_headers() -> [set_planar] -> create() -> pull() loop; returns the planes
        rebuilt from the pulled lines and the order the components came in"""
        fi = self.read_headers(j2c, I32)
        if planar is not None:
            self._check(self.L.ojb_dec_set_planar(self.h, 1 if planar else 0))
        self._check(self.L.ojb_dec_begin_pull(self.h))
        planes = [np.zeros((fi.comp_h[c], fi.comp_w[c]), np.int32) for c in range(fi.num_comps)]
        rows = [0] * fi.num_comps
        order = []
        nc = C.c_uint32()
        line = self.L.ojb_dec_pull(self.h, C.byref(nc))
        while line:
            c = nc.value
            order.append(c)
            planes[c][rows[c]] = np.ctypeslib.as_array(C.cast(line, C.POINTER(C.c_int32)), shape=(fi.comp_w[c],))
            rows[c] += 1
            line = self.L.ojb_dec_pull(self.h, C.byref(nc))
        return planes, order

    def read_band(self, tile, comp, res, band):
        bw, bh = C.c_uint32(), C.c_uint32()
        self._check(self.L.ojb_dec_read_band(self.h, tile, comp, res, band, None, C.byref(bw), C.byref(bh)))
        out = np.zeros((bh.value, bw.value), np.uint32)
        if out.size:
            self._check(self.L.ojb_dec_read_band(self.h, tile, comp, res, band, out.ctypes.data, C.byref(bw), C.byref(bh)))
        return out

    def list_blocks(self):
        n = C.c_uint32()
        self._check(self.L.ojb_dec_list_blocks(self.h, None, 0, C.byref(n)))
        arr = (_lib.BlockDesc * max(1, n.value))()
        self._check(self.L.ojb_dec_list_blocks(self.h, arr, n.value, C.byref(n)))
        return [arr[i] for i in range(n.value)]

    @property
    def failed_blocks(self):
        return self.L.ojb_dec_failed_blocks(self.h)

    @property
    def kernel_launches(self):
        return self.L.ojb_dec_kernel_launches(self.h)

    def timings(self):
        t = (C.c_float * 8)()
        self.L.ojb_dec_timings(self.h, t)
        return dict(zip(("h2d", "host_parse", "ht_decode", "dwt_inv", "d2h_image", "_5", "_6", "host_ms"), list(t)))


def encode_blocks(samples, descs, lib=None):
    """batch ojph_encode_codeblock32: samples = flat uint32 sign-magnitude array, descs =
    list of (sample_off, stride, w, h, missing_msbs) -> list of bytes (b'' if not coded)."""
    L = lib if lib is not None else _lib.lib()
    n = len(descs)
    arr = (_lib.BlockDesc * n)()
    for i, (off, stride, w, h, mm) in enumerate(descs):
        arr[i].sample_off, arr[i].stride, arr[i].w, arr[i].h, arr[i].missing_msbs = off, stride, w, h, mm
    samples = np.ascontiguousarray(samples, np.uint32)
    cap = int(samples.size) * 5 + 4096 * n + 65536
    out = np.zeros(cap, np.uint8)
    used = C.c_uint64()
    rc = L.ojb_encode_blocks(samples.ctypes.data, samples.size, arr, n, out.ctypes.data, cap, C.byref(used))
    if rc != 0:
        raise OjphError(L.ojb_last_error().decode(errors="replace"))
    return [out[arr[i].byte_off:arr[i].byte_off + arr[i].len1].tobytes() for i in range(n)]


def decode_blocks(coded, geoms, lib=None, causal=False):
    """batch ojph_decode_codeblock32: coded = list of (bytes, len1, len2, missing_msbs, num_passes),
    geoms = list of (w, h) -> list of ((h, w) uint32 sign-magnitude arrays, ok flag); causal = the
    stripe_causal argument for every block."""
    L = lib if lib is not None else _lib.lib()
    n = len(coded)
    arr = (_lib.BlockDesc * n)()
    blob = bytearray()
    soff = 0
    for i, ((data, l1, l2, mm, npass), (w, h)) in enumerate(zip(coded, geoms)):
        stride = (w + 15) & ~15
        arr[i].sample_off, arr[i].stride, arr[i].w, arr[i].h = soff, stride, w, h
        arr[i].missing_msbs, arr[i].num_passes, arr[i].len1, arr[i].len2 = mm, npass, l1, l2
        arr[i].byte_off = len(blob)
        arr[i].causal = 1 if causal else 0
        blob += data
        soff += stride * h
    cs = np.frombuffer(bytes(blob) + b"\0" * 64, np.uint8).copy()
    samples = np.zeros(soff + 64, np.uint32)
    rc = L.ojb_decode_blocks(cs.ctypes.data, len(blob), arr, n, samples.ctypes.data, samples.size)
    if rc != 0:
        raise OjphError(L.ojb_last_error().decode(errors="replace"))
    res = []
    for i, (w, h) in enumerate(geoms):
        st = arr[i].stride
        a = samples[arr[i].sample_off:arr[i].sample_off + st * h].reshape(h, st)[:, :w].copy()
        res.append((a, arr[i].status == 0))
    return res
