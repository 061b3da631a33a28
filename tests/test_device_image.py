"""Frames read from, and decoded into, memory the caller owns (ojb_enc_encode_device / ojb_dec_decode_device): planar
rows at any pitch, interleaved pixels, a window of a larger canvas.  The DWT kernels address that memory directly, so
every layout must give the codestream of the host-plane encoder and the samples of the host-plane decoder, byte for
byte, and the decoder must not touch a byte outside the samples it writes.  CPU tier: numpy arrays stand in for device
memory under the SIMT emulator.  GPU tier: the torch methods (Encoder.encode_tensor / Decoder.decode_tensor)."""
import ctypes as C
import numpy as np
import pytest
import openjph_b200 as ob
from openjph_b200 import codestream as cs
import cases
import images

_ALL = dict(cases.SMALL_REV + cases.SMALL_IRV)
EXTRA = {
    "nlt_signed": dict(width=67, height=45, num_comps=3, bit_depth=8, is_signed=True, num_decomps=2, reversible=True,
                       nlt={"all": 3}),
    "dfs_atk": dict(width=80, height=60, num_comps=1, bit_depth=8, num_decomps=3, reversible=True, decomp="BHV",
                    atk=dict(reversible=True, steps=[(1, 2, 2), (-1, 1, 1)])),
    "wide64": dict(width=41, height=30, num_comps=3, bit_depth=30, num_decomps=3, reversible=True, color_transform=True),
    "rgb8_u8_rct": dict(width=300, height=70, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, color_transform=True),
    "irv_rgb12_u16": dict(width=263, height=66, num_comps=3, bit_depth=12, num_decomps=3, reversible=False,
                          color_transform=True, qfactor=90),
}
NAMES = cases.EMU_REV + cases.EMU_IRV + list(EXTRA)
SENTINEL = {ob.U8: 0xA5, ob.U16: 0xA5A5, ob.I32: -0x5A5A5A5B}


def _kw(name):
    return EXTRA.get(name) or _ALL[name]


def _container(p):
    """the narrowest container of the case: all three occur across NAMES"""
    bd = max(p.bit_depth[c] for c in range(p.num_comps))
    if any(p.is_signed[c] for c in range(p.num_comps)) or bd > 16:
        return ob.I32
    return ob.U8 if bd <= 8 else ob.U16


def _frame(name, p):
    if name == "wide64":
        rng = np.random.default_rng(77)
        return [rng.integers(0, 1 << 30, (p.height, p.width)).astype(np.int32) for _ in range(p.num_comps)]
    return cases.frame_for(p, "noise" if "noise" in name else "synth")


def _setup(lib, name):
    p = cases.make(_kw(name))
    st = _container(p)
    dt = cs._NP[st]
    frame = [np.asarray(f).astype(dt) for f in _frame(name, p)]
    want = ob.Encoder(p, st, lib=lib).encode(frame)
    return p, st, dt, frame, want


def _planar(dims, dt, fill, extra=3):
    """one canvas per component whose rows are padded to an odd number of samples"""
    bufs = []
    for w, h in dims:
        pitch = w + extra if (w + extra) % 2 else w + extra + 1
        bufs.append(np.full((max(h, 1), pitch), fill, dt))
    return bufs


def _img_planar(bufs, dims):
    return cs.device_image([(b.ctypes.data, b.strides[0], 1) for b, _ in zip(bufs, dims)])


def _img_interleaved(buf, nc, x0=0, y0=0):
    """buf (H, W, S): components 0 .. nc-1 of the pixel at (x0, y0) onwards"""
    es = buf.itemsize
    base = buf.ctypes.data + y0 * buf.strides[0] + x0 * buf.strides[1]
    return cs.device_image([(base + c * es, buf.strides[0], buf.shape[2]) for c in range(nc)])


def _shared_size(dims):
    return len(set(dims)) == 1 and dims[0][0] > 0 and dims[0][1] > 0


def _check_encode(lib, name):
    p, st, dt, frame, want = _setup(lib, name)
    dims = cs.comp_dims(p)
    enc = ob.Encoder(p, st, lib=lib)
    bufs = _planar(dims, dt, 0)
    for b, f, (w, h) in zip(bufs, frame, dims):
        b[:h, :w] = f
    assert enc.encode_device(_img_planar(bufs, dims)) == want, "padded planar rows"
    if _shared_size(dims):
        w, h = dims[0]
        nc = p.num_comps
        for s in (nc, nc + 1):                     # HWC, and one more channel the codec ignores
            buf = np.zeros((h, w, s), dt)
            for c in range(nc):
                buf[:, :, c] = frame[c]
            assert enc.encode_device(_img_interleaved(buf, nc)) == want, "interleaved, %d channels" % s


def _check_decode(lib, name):
    p, st, dt, frame, want = _setup(lib, name)
    ref = ob.Decoder(lib=lib).decode(want, st)
    dims = [(r.shape[1], r.shape[0]) for r in ref]
    fill = SENTINEL[st]
    dec = ob.Decoder(lib=lib)
    dec.read_headers(want, st)
    bufs = _planar(dims, dt, fill)
    dec.decode_device(_img_planar(bufs, dims))
    for b, r, (w, h) in zip(bufs, ref, dims):
        assert np.array_equal(b[:h, :w], r)
        assert (b[:, w:] == fill).all() and (b[h:] == fill).all()
    if _shared_size(dims):
        w, h = dims[0]
        nc = p.num_comps
        for s in (nc, nc + 1):
            buf = np.full((h, w, s), fill, dt)
            dec.decode_device(_img_interleaved(buf, nc))
            for c in range(nc):
                assert np.array_equal(buf[:, :, c], ref[c]), (s, c)
            assert (buf[:, :, nc:] == fill).all()
        # a window at an odd offset inside a larger canvas
        canvas = np.full((h + 5, w + 8, nc + 1), fill, dt)
        dec.decode_device(_img_interleaved(canvas, nc, x0=3, y0=1))
        mask = np.ones(canvas.shape, bool)
        mask[1:1 + h, 3:3 + w, :nc] = False
        assert (canvas[mask] == fill).all(), "a byte outside the window changed"
        for c in range(nc):
            assert np.array_equal(canvas[1:1 + h, 3:3 + w, c], ref[c])
    # reduced resolution
    if p.num_decomps >= 1 and name not in ("dfs_atk",):
        want_r = ob.Decoder(lib=lib).decode(want, st, skip=(1, 1))
        dec.read_headers(want, st)
        dec.restrict_input_resolution(1, 1)
        rd = [(r.shape[1], r.shape[0]) for r in want_r]
        bufs = _planar(rd, dt, fill)
        dec.decode_device(_img_planar(bufs, rd))
        for b, r, (w, h) in zip(bufs, want_r, rd):
            assert np.array_equal(b[:h, :w], r)


@pytest.mark.parametrize("name", NAMES)
def test_encode_from_device_image_emulator(name, emu_lib):
    _check_encode(emu_lib, name)


@pytest.mark.parametrize("name", NAMES)
def test_decode_into_device_image_emulator(name, emu_lib):
    _check_decode(emu_lib, name)


def test_stream_of_frames_from_different_buffers_emulator(emu_lib):
    """five different frames, each from and to its own buffers, through one encoder / decoder pair with the
    codestream in "device" memory on both sides"""
    lib = emu_lib
    w, h, nc, bd = 160, 96, 3, 10
    p = ob.make_params(w, h, nc, bd, num_decomps=3, reversible=True, color_transform=True, block=(32, 32))
    enc, dec = ob.Encoder(p, ob.U16, lib=lib), ob.Decoder(lib=lib)
    cap = w * h * nc * 4 + (1 << 16)
    csbuf = np.zeros(cap + 64, np.uint8)
    for k in range(5):
        fr = [f.astype(np.uint16) for f in images.synth_frame(w, h, nc, bd, 60 + k)]
        want = ob.Encoder(p, ob.U16, lib=lib).encode(fr)
        src = np.zeros((h, w, nc + (k % 2)), np.uint16)
        for c in range(nc):
            src[:, :, c] = fr[c]
        n = enc.encode_device(_img_interleaved(src, nc), 0, csbuf.ctypes.data, cap)
        assert csbuf[:n].tobytes() == want, k
        dec.read_headers_device(csbuf.ctypes.data, n, ob.U16)
        out = _planar([(w, h)] * nc, np.uint16, 0, extra=1 + 2 * k)
        dec.decode_device(_img_planar(out, [(w, h)] * nc))
        for c in range(nc):
            assert np.array_equal(out[c][:, :w], fr[c]), (k, c)


def _code(lib, fn):
    with pytest.raises(ob.OjphError) as e:
        fn()
    return str(e.value)


def test_refusals_emulator(emu_lib):
    lib = emu_lib
    w, h = 40, 30
    p = ob.make_params(w, h, 3, 8, num_decomps=2, reversible=True, color_transform=True)
    enc = ob.Encoder(p, ob.U8, lib=lib)
    cs_bytes = enc.encode([np.zeros((h, w), np.uint8)] * 3)
    dec = ob.Decoder(lib=lib)
    dec.read_headers(cs_bytes, ob.U8)
    buf = np.zeros((h, w, 3), np.uint8)
    good = [(buf.ctypes.data + c, buf.strides[0], 3) for c in range(3)]

    def with_comp1(**kw):
        comps = list(good)
        a, pitch, col = comps[1]
        comps[1] = (kw.get("base", a), kw.get("pitch", pitch), kw.get("col", col))
        return cs.device_image(comps)

    bad = {
        "0x000B003B": with_comp1(base=0),
        "0x000B003C": with_comp1(col=0),
        "0x000B003D": with_comp1(pitch=(w - 1) * 3),                   # one byte short of a row's footprint
        "0x000B003E": with_comp1(pitch=1 << 32),
    }
    for code, img in bad.items():
        assert code in _code(lib, lambda: enc.encode_device(img)), code
        assert code in _code(lib, lambda: dec.decode_device(img)), code
    assert (buf == 0).all()
    # misaligned 16-bit rows
    p16 = ob.make_params(w, h, 1, 12, num_decomps=2)
    e16 = ob.Encoder(p16, ob.U16, lib=lib)
    b16 = np.zeros((h, w + 1), np.uint16)
    assert "0x000B003B" in _code(lib, lambda: e16.encode_device(cs.device_image([(b16.ctypes.data + 1, b16.strides[0], 1)])))
    # before configure / read_headers
    raw = lib.ojb_enc_create()
    try:
        n = C.c_uint64()
        img = cs.device_image(good)
        out = np.zeros(1 << 16, np.uint8)
        assert lib.ojb_enc_encode_device(raw, C.byref(img), None, out.ctypes.data, out.size, C.byref(n), 0) != 0
        assert "0x000B003F" in lib.ojb_last_error().decode()
    finally:
        lib.ojb_enc_destroy(raw)
    fresh = ob.Decoder(lib=lib)
    assert "0x000B003F" in _code(lib, lambda: fresh.decode_device(cs.device_image(good)))


# ---- GPU tier: the torch methods ---------------------------------------------------------------------------------
# torch has few kernels for uint16: 16-bit samples are built and compared as int16 (the same bits) and handed to the
# codec as uint16 views
def _cu(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()


def _api(t, st):
    import torch
    return t.view(torch.uint16) if st == ob.U16 else t


def _host(t, st):
    import torch
    if t.dtype == torch.uint16:
        t = t.view(torch.int16)
    a = t.cpu().numpy()
    return a.view(np.uint16) if st == ob.U16 else a


def _fill(st):
    return -0x5A5B if st == ob.U16 else SENTINEL[st]


def _work_dtype(st):
    import torch
    return {ob.U8: torch.uint8, ob.U16: torch.int16, ob.I32: torch.int32}[st]


def _gpu_case(name):
    import torch
    p, st, dt, frame, want = _setup(None, name)
    ref = ob.Decoder().decode(want, st)
    dims = cs.comp_dims(p)
    wdt, fill = _work_dtype(st), _fill(st)
    enc, dec = ob.Encoder(p, st), ob.Decoder()
    planes = [_cu(f) for f in frame]
    # padded planar rows, one 2-D view per component
    views = []
    for t, (w, h) in zip(planes, dims):
        pitch = w + 3 if (w + 3) % 2 else w + 4
        canvas = torch.zeros((max(h, 1), pitch), dtype=wdt, device="cuda")
        canvas[:h, :w] = t
        views.append(_api(canvas[:h, :w], st))
    got = enc.encode_tensor(views)
    assert got.cpu().numpy().tobytes() == want
    outs = []
    for w, h in dims:
        pitch = w + 3 if (w + 3) % 2 else w + 4
        outs.append(torch.full((max(h, 1), pitch), fill, dtype=wdt, device="cuda"))
    dec.decode_tensor(got, out=[_api(o[:h, :w], st) for o, (w, h) in zip(outs, dims)])
    for o, r, (w, h) in zip(outs, ref, dims):
        assert np.array_equal(_host(o[:h, :w], st), r)
        assert (o[:, w:] == fill).all().item() and (o[h:] == fill).all().item()
    if _shared_size(dims):
        w, h = dims[0]
        nc = p.num_comps
        chw = torch.stack(planes)
        for s in (nc, nc + 1):
            hwc = torch.zeros((h, w, s), dtype=wdt, device="cuda")
            hwc[:, :, :nc] = chw.permute(1, 2, 0)
            assert enc.encode_tensor(_api(hwc, st)[:, :, :nc], layout="hwc").cpu().numpy().tobytes() == want
            out = torch.full((h, w, s), fill, dtype=wdt, device="cuda")
            dec.decode_tensor(want, out=_api(out, st)[:, :, :nc], layout="hwc")
            for c in range(nc):
                assert np.array_equal(_host(out[:, :, c], st), ref[c])
            assert (out[:, :, nc:] == fill).all().item()
        canvas = torch.full((nc, h + 5, w + 8), fill, dtype=wdt, device="cuda")
        dec.decode_tensor(got, out=_api(canvas, st)[:, 1:1 + h, 3:3 + w])
        mask = torch.ones(canvas.shape, dtype=torch.bool, device="cuda")
        mask[:, 1:1 + h, 3:3 + w] = False
        assert (canvas[mask] == fill).all().item()
        for c in range(nc):
            assert np.array_equal(_host(canvas[c, 1:1 + h, 3:3 + w], st), ref[c])
    if p.num_decomps >= 1 and name != "dfs_atk":
        want_r = ob.Decoder().decode(want, st, skip=(1, 1))
        d2 = ob.Decoder()
        d2.read_headers(want, st)
        d2.restrict_input_resolution(1, 1)
        outs = [torch.full((r.shape[0], r.shape[1] + 1), fill, dtype=wdt, device="cuda") for r in want_r]
        rd = [(r.shape[1], r.shape[0]) for r in want_r]
        d2.decode_device(cs._tensor_image([_api(o[:, :-1], st) for o in outs], "chw", st, rd), 0)
        for o, r in zip(outs, want_r):
            assert np.array_equal(_host(o[:, :-1], st), r)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_image_gpu(name, gpu_lib):
    _gpu_case(name)


@pytest.mark.gpu
@pytest.mark.parametrize("rev", [True, False], ids=["53_rct", "97_ict_q90"])
def test_headline_frame_tensors_gpu(rev, gpu_lib):
    """the 8192 x 8192 x 3 12-bit frame in and out as CHW, as HWC and as batch[1] of a (2, H, W, 3) tensor"""
    import torch
    W = H = 8192
    kw = dict(num_decomps=5, reversible=rev, color_transform=True)
    if not rev:
        kw["qfactor"] = 90
    p = ob.make_params(W, H, 3, 12, **kw)
    frame = [f.astype(np.uint16) for f in images.synth_frame(W, H, 3, 12, 5)]
    want = ob.Encoder(p, ob.U16).encode(frame)
    refc = torch.stack([_cu(r) for r in ob.Decoder().decode(want, ob.U16)])      # int16 bits
    enc, dec = ob.Encoder(p, ob.U16), ob.Decoder()
    chw = torch.stack([_cu(f) for f in frame])
    hwc = chw.permute(1, 2, 0).contiguous()
    batch = torch.zeros((2, H, W, 3), dtype=torch.int16, device="cuda")
    batch[0].fill_(0x1234)
    batch[1].copy_(hwc)
    for t, layout in ((chw, "chw"), (hwc, "hwc"), (batch[1], "hwc")):
        got = enc.encode_tensor(t.view(torch.uint16), layout=layout)
        assert got.numel() == len(want) and got.cpu().numpy().tobytes() == want, layout
    if rev:
        assert torch.equal(refc, chw)
    out = dec.decode_tensor(got, layout="chw", sample_type=ob.U16)
    assert torch.equal(out.view(torch.int16), refc)
    out = dec.decode_tensor(got, layout="hwc", sample_type=ob.U16)
    assert torch.equal(out.view(torch.int16), refc.permute(1, 2, 0))
    batch[1].zero_()
    dec.decode_tensor(got, out=batch.view(torch.uint16)[1], layout="hwc")
    assert torch.equal(batch[1], refc.permute(1, 2, 0))
    assert (batch[0] == 0x1234).all().item(), "batch[0] changed"


@pytest.mark.gpu
def test_ordering_against_the_callers_stream_gpu(gpu_lib):
    """input produced on a side stream behind a long kernel, no synchronise before the call; output consumed on the
    caller's stream straight after it"""
    import torch
    w, h = 1024, 768
    p = ob.make_params(w, h, 3, 8, num_decomps=5, reversible=True, color_transform=True)
    frames = [[f.astype(np.uint8) for f in images.synth_frame(w, h, 3, 8, s)] for s in (1, 2)]
    wants = [ob.Encoder(p, ob.U8).encode(f) for f in frames]
    enc, dec = ob.Encoder(p, ob.U8), ob.Decoder()
    srcs = [torch.stack([_cu(x) for x in f]) for f in frames]
    side = torch.cuda.Stream()
    t = srcs[0].clone()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)             # long enough that a missing wait reads frame 0
        t.copy_(srcs[1])
    got = enc.encode_tensor(t, stream=side)
    assert got.cpu().numpy().tobytes() == wants[1]
    # decode: the fill queued behind the sleep must land before the decoder writes
    out = torch.empty_like(srcs[0])
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        out.fill_(7)
    dec.decode_tensor(wants[1], out=out, stream=side)
    assert torch.equal(out, srcs[1])
    # consumed at once on the caller's stream
    out2 = dec.decode_tensor(wants[0], sample_type=ob.U8)
    assert torch.equal(out2.clone(), srcs[0])


@pytest.mark.gpu
def test_two_side_stream_encodes_with_a_busy_current_stream_gpu(gpu_lib):
    """the codestream tensor of one call must survive the next call on the same encoder, and be complete on the stream
    the caller named, while torch's current stream is still busy"""
    import torch
    w, h = 1024, 768
    p = ob.make_params(w, h, 3, 8, num_decomps=5, reversible=True, color_transform=True)
    frames = [[f.astype(np.uint8) for f in images.synth_frame(w, h, 3, 8, s)] for s in (3, 4)]
    wants = [ob.Encoder(p, ob.U8).encode(f) for f in frames]
    srcs = [torch.stack([_cu(x) for x in f]) for f in frames]
    enc = ob.Encoder(p, ob.U8)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    torch.cuda._sleep(400_000_000)                 # the current stream stays busy through both calls
    got = [enc.encode_tensor(srcs[i], stream=side) for i in range(2)]
    with torch.cuda.stream(side):
        copies = [g.clone() for g in got]          # consumed on the stream the calls named
    torch.cuda.synchronize()
    for g, c, want in zip(got, copies, wants):
        assert g.cpu().numpy().tobytes() == want
        assert c.cpu().numpy().tobytes() == want


@pytest.mark.gpu
def test_stream_of_frames_from_different_buffers_gpu(gpu_lib):
    """five different frames, each from and into its own tensors, through one encoder / decoder pair with the codestream
    in device memory on both sides: from the third call on each frame is a replayed graph"""
    import torch
    w, h, nc, bd = 640, 384, 3, 10
    p = ob.make_params(w, h, nc, bd, num_decomps=4, reversible=True, color_transform=True, block=(32, 32))
    enc, dec = ob.Encoder(p, ob.U16), ob.Decoder()
    cs_buf = torch.zeros(w * h * nc * 4 + (1 << 16), dtype=torch.uint8, device="cuda")
    for k in range(5):
        fr = [f.astype(np.uint16) for f in images.synth_frame(w, h, nc, bd, 80 + k)]
        want = ob.Encoder(p, ob.U16).encode(fr)
        chw = torch.stack([_cu(f) for f in fr])
        src = torch.zeros((h, w, nc + (k % 2)), dtype=torch.int16, device="cuda")
        src[:, :, :nc] = chw.permute(1, 2, 0)
        n = enc.encode_tensor(src.view(torch.uint16)[:, :, :nc], layout="hwc", out=cs_buf)
        assert cs_buf[:n].cpu().numpy().tobytes() == want, k
        out = torch.full((nc, h, w + 1 + 2 * k), 7, dtype=torch.int16, device="cuda")
        dec.decode_tensor(cs_buf[:n], out=out.view(torch.uint16)[:, :, :w], sample_type=ob.U16)
        assert torch.equal(out[:, :, :w], chw), k
        assert (out[:, :, w:] == 7).all().item(), k
