"""The irreversible (9/7) path held to a float64 model (tests/ref97.py), sample by sample, at the seams of the
streaming DWT kernels: warp strips of 120 columns, row chunks, mirrored odd edges, deep levels that fall to the general
kernels, tiles and sub-sampled components.  Runs under the emulator build on the CPU tier and on the H100 with -m gpu.

For every configuration:
  forward   every band's quantiser output (Encoder.read_band) against the model's unrounded quantiser input, and
            bit for bit against the float32 restatement that follows the reference's operation order (oracleport);
  inverse   the decoder's band planes (float bits) against the float32 de-quantisation of the encoder's words, and its
            samples against the model's synthesis of those words;
  cross     our decode against the reference's decode of the same codestream.

Tolerances.  u = 2^-24 is the unit round-off of float32.  Each lifting step of one direction is three float32
operations (a sum, a product, a sum), each off by at most u times its result; with the K scaling and two directions a
level rounds about 30 times, on values no larger than a few times M, the largest |sample| entering the level (M <= 1
in the normalised units the transform works in).  Errors of earlier levels pass through later ones with a gain near
one.  So after d levels the coefficient x is within C * d * u * M of the model, and the quantiser input v = x * delta_inv
within that times delta_inv, plus u * |v| for the product and 1/2 for its rounding.  The worst case (C about 60) is far
from what the arithmetic reaches: C_FWD = 40 is about three times the largest ratio |v - model| / (d u M delta_inv)
that the CPU-tier configurations reach (14.1, three levels of a 12-bit ICT frame; 5 to 10 elsewhere).
The quantiser input is a 2^(31-K_max)-scaled value whose float32 noise (hundreds of units at |v| ~ 2^30) is far above
its own rounding, so the rounding of v itself is pinned by the bit-exact comparison with the float32 restatement; the
rule compares what reaches the codestream: the coded magnitude floor(|v| / 2^(31-K_max)), with tie band
tau = e_v / 2^(31-K_max) around each quantisation threshold.
The inverse output is t = f * 2^B for a synthesised value f; the same count over D levels, the de-quantisation and the
inverse ICT gives |f - model| <= C_INV * D * u * M_syn, M_syn the largest |value| of the synthesised planes, so
tau = C_INV * D * u * M_syn * 2^B.  C_INV = 8: the library's rounding decisions that differ from the model's lie at
most 1.2 D u M_syn 2^B from the tie on the CPU tier.  The
reference itself is held to the same band: every sample where its decode differs from ours lies inside it.
Each check counts the samples inside its band and asserts that they stay a small fraction (TIE_FRACTION), so a
tolerance cannot pass by declaring every sample a tie."""
import os
import subprocess
import sys
import numpy as np
import pytest
import cases
import ref97 as M
import openjph_b200 as ob

C_FWD = 40.0
C_INV = 8.0
TIE_FRACTION = 0.03
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(w, h, nc=1, bd=10, x0=0, y0=0, st=ob.I32, **kw):
    """image of w x h samples at canvas offset (x0, y0)"""
    d = dict(width=w + x0, height=h + y0, num_comps=nc, bit_depth=bd, reversible=False, offset=(x0, y0), st=st)
    d.setdefault("num_decomps", 3)
    d.update(kw)
    return d


# CPU tier (emulator): widths either side of the 120-column strip boundaries at an even and an odd x0, heights either
# side of the 8-row chunk seams (small resolutions use 8-row chunks), and the edges of the transform
CPU_CASES = [
    ("w119_x0", _cfg(119, 23, x0=0)),
    ("w119_x1", _cfg(119, 25, x0=1, y0=1)),
    ("w120_x2", _cfg(120, 17, x0=2)),
    ("w120_x3", _cfg(120, 15, x0=3, y0=1)),
    ("w121_x0", _cfg(121, 24, x0=0, y0=1)),
    ("w121_x1", _cfg(121, 16, x0=1)),
    ("w241_x0", _cfg(241, 9, x0=0)),
    ("w241_x1", _cfg(241, 7, x0=1, y0=1)),
    ("w243_x4", _cfg(243, 17, x0=4, y0=3)),
    ("w243_x5", _cfg(243, 15, x0=5)),
    ("ict_u8", _cfg(125, 33, nc=3, bd=8, x0=1, y0=1, st=ob.U8, color_transform=True)),
    ("ict_u16_12bit", _cfg(131, 25, nc=3, bd=12, x0=2, y0=3, st=ob.U16, color_transform=True)),
    ("signed12_i32", _cfg(97, 31, bd=12, x0=3, y0=1, is_signed=True)),
    ("ict_signed12", _cfg(67, 19, nc=3, bd=12, x0=1, is_signed=True, color_transform=True)),
    ("levels5_deep", _cfg(67, 45, bd=12, x0=3, y0=5, num_decomps=5)),
    ("thin_1xN", _cfg(1, 40, x0=1, y0=0, num_decomps=3)),
    ("thin_Nx1", _cfg(40, 1, x0=0, y0=1, num_decomps=3)),
    ("thin_3x6", _cfg(3, 6, x0=1, y0=1, num_decomps=3)),
    ("tiled_odd", _cfg(150, 90, nc=3, bd=10, x0=5, y0=3, color_transform=True, tile=(64, 64), tile_offset=(3, 2))),
    ("sub420", _cfg(130, 34, nc=3, bd=8, x0=1, y0=1, st=ob.U8, subsampling=[(1, 1), (2, 2), (2, 2)])),
    ("fine_qstep_kmax16", _cfg(125, 20, bd=12, x0=1, qstep=0.0002)),
    ("q90_split", _cfg(128, 64, nc=3, bd=12, st=ob.U16, color_transform=True, qfactor=90, num_decomps=4)),
]
# GPU tier: large enough for 32-row forward and 64-row inverse chunks at level 1
BIG_CASES = [
    ("cfg5_3840x2160_10bit", _cfg(3840, 2160, nc=3, bd=10, st=ob.U16, color_transform=True, num_decomps=5)),
    ("cfg3_4096x4096_12bit_q90", _cfg(4096, 4096, nc=3, bd=12, st=ob.U16, color_transform=True, qfactor=90, num_decomps=6)),
    ("headline_8192x1024_12bit_q90", _cfg(8192, 1024, nc=3, bd=12, st=ob.U16, color_transform=True, qfactor=90, num_decomps=5)),
]
ALL = dict(CPU_CASES + BIG_CASES)
# the variant runs (switches read once per process) take this subset
VARIANT_CASES = ["w121_x1", "w241_x1", "ict_u16_12bit", "levels5_deep", "thin_3x6", "fine_qstep_kmax16", "q90_split"]
# no_stream_dwt: every level through the general shared-memory kernels (dwt_fwd.cu / dwt_inv.cu), which otherwise only
# take dyadic 9/7 levels of frames whose coefficients pass 2^30 words; on the GPU with a 4K frame as well
VARIANTS = {"no_fast_blocks": {"OJB_NO_FAST_BLOCKS": "1"}, "no_stream_dwt": {"OJB_NO_STREAM_DWT": "1"}}
VARIANT_GPU_EXTRA = {"no_stream_dwt": ["cfg5_3840x2160_10bit"]}


# ---- the streaming DWT's tiling (dwt_stream_tiling, dwt_stream.cu), restated to choose and audit the sizes -------
def stream_tiling(x0, y0, w, h, forward):
    """(strips, chunk_rows) of the 9/7 streaming kernels for a resolution: 120 output columns per strip; 32 forward
    or 64 inverse rows per chunk, halved (down to 8) until there are at least 8 chunks per SM of a 132-SM H100"""
    ue, ye = x0 & ~1, y0 & ~1
    strips = (x0 + w - ue + 119) // 120
    rows = 32 if forward else 64
    while rows > 8 and strips * ((y0 + h - ye + rows - 1) // rows) < 132 * 8:
        rows >>= 1
    return strips, rows


def _level1(kw):
    c = cases.make(_strip(kw))
    from openjph_b200.codestream import comp_dims
    w, h = comp_dims(c)[0]
    x0, y0 = kw["offset"]
    return stream_tiling(x0, y0, w, h, True), stream_tiling(x0, y0, w, h, False)


def _strip(kw):
    return {k: v for k, v in kw.items() if k != "st"}


# ---- geometry ---------------------------------------------------------------------------------------------------------
def _tile_comp_rects(p):
    """[(tile index, [(comp, x0, y0, x1, y1) in component coordinates])] for every tile"""
    def dc(a, b):
        return -(-a // b)
    W, H = p.width, p.height
    tw, th = (p.tile_w or W), (p.tile_h or H)
    tx0, ty0 = p.tile_off_x, p.tile_off_y
    nx, ny = dc(W - tx0, tw), dc(H - ty0, th)
    out = []
    for j in range(ny):
        for i in range(nx):
            ax0, ay0 = max(tx0 + i * tw, p.off_x), max(ty0 + j * th, p.off_y)
            ax1, ay1 = min(tx0 + (i + 1) * tw, W), min(ty0 + (j + 1) * th, H)
            out.append((j * nx + i, [(c, dc(ax0, p.dx[c]), dc(ay0, p.dy[c]), dc(ax1, p.dx[c]), dc(ay1, p.dy[c]))
                                     for c in range(p.num_comps)]))
    return out


def _bands(D):
    return [(0, 0)] + [(r, b) for r in range(1, D + 1) for b in (1, 2, 3)]


# ---- one configuration --------------------------------------------------------------------------------------------
def run_case(lib, name, ref):
    kw = ALL[name]
    st = kw["st"]
    p = cases.make(_strip(kw))
    frame = cases.frame_for(p)
    B = p.bit_depth[0]
    signed = bool(p.is_signed[0])
    half = 0 if signed else 1 << (B - 1)
    D = p.num_decomps
    planes = frame if st == ob.I32 else [f.astype(np.uint8 if st == ob.U8 else np.uint16) for f in frame]
    enc = ob.Encoder(p, st, lib=lib)
    cs = enc.encode(planes)
    dec = ob.Decoder(lib=lib)
    out = [a.astype(np.int64) for a in dec.decode(cs, st)]
    refout = [a.astype(np.int64) for a in ref.decode(cs)[0]]
    comp_org = [(-(-p.off_x // p.dx[c]), -(-p.off_y // p.dy[c])) for c in range(p.num_comps)]
    s = {}
    for key in ("fwd_n", "fwd_tie", "inv_n", "inv_tie", "cross_n", "cross_diff", "kmax"):
        s.setdefault(key, 0)
    s.setdefault("fwd_ratio", 0.0)
    s.setdefault("inv_ratio", 0.0)
    ct = bool(p.color_transform)
    for tile, rects in _tile_comp_rects(p):
        synth = []
        for c, x0, y0, x1, y1 in rects:
            info = {rb: enc.band_info(tile, c, *rb) for rb in _bands(D)}
            assert (info[(D, 1)]["res_x0"], info[(D, 1)]["res_y0"]) == (x0, y0), (name, tile, c)
            ox, oy = comp_org[c]
            sl = (slice(y0 - oy, y1 - oy), slice(x0 - ox, x1 - ox))
            # forward model
            xs = M.to_float(frame[c][sl], B, signed)
            if ct and c < 3:
                xs = M.ict_fwd(*[M.to_float(frame[k][sl], B, signed) for k in range(3)], c)
            bands, mags = M.analyse(xs, x0, y0, D)
            del xs
            words = {}
            for (r, b), a in bands.items():
                bi = info[(r, b)]
                g = enc.read_band(tile, c, r, b)
                assert g.shape == a.shape, (name, tile, c, r, b)
                words[(r, b)] = g
                if not g.size:
                    continue
                kmax, dinv = int(bi["K_max"]), float(bi["delta_inv"])
                s["kmax"] = max(s["kmax"], kmax)
                t = a * dinv
                d = D - r + 1 if r else D
                e_v = C_FWD * d * M.U32 * max(mags[:d]) * dinv + M.U32 * np.abs(t) + 0.5
                gs = np.where(g & 0x80000000, -1.0, 1.0) * (g & 0x7FFFFFFF).astype(np.float64)
                err = np.abs(gs - t)
                s["fwd_ratio"] = max(s["fwd_ratio"], float(((err - 0.5) / (d * M.U32 * max(mags[:d]) * dinv)).max()))
                assert (err <= e_v).all(), ("quantiser input off the model", name, tile, c, r, b,
                                            np.unravel_index(int(np.argmax(err - e_v)), err.shape), float(err.max()))
                # the coded magnitude: floor(|v| / 2^s) -> the rule on |t| / 2^s - 1/2
                sh = 2.0 ** (31 - kmax)
                q = (g & 0x7FFFFFFF) >> np.uint32(31 - kmax)
                nbad, ntie, first = M.check_rounding(q, np.abs(t) / sh - 0.5, e_v / sh)
                assert nbad == 0, ("coded magnitude differs from the model's", name, tile, c, r, b, first)
                sig = (q != 0) & (np.abs(t) > e_v)
                assert np.array_equal(np.signbit(t[sig]), (g[sig] >> 31).astype(bool)), ("sign", name, tile, c, r, b)
                s["fwd_n"] += g.size; s["fwd_tie"] += ntie
                # the decoder's band plane: the float32 de-quantisation of these words, bit for bit
                db = dec.read_band(tile, c, r, b)
                assert np.array_equal(db, M.dequantise_f32(g, kmax, bi["delta"])), ("decoder band plane", name, tile, c, r, b)
            # inverse model from the encoder's words
            deq = {rb: M.dequantise(words[rb], int(info[rb]["K_max"]), float(info[rb]["delta"])) for rb in words}
            origins = [None] + [(info[(r, 1)]["res_x0"], info[(r, 1)]["res_y0"]) for r in range(1, D + 1)]
            synth.append(M.synthesise(deq, origins) if D else deq[(0, 0)])
            del bands, deq
        if ct:
            synth[:3] = M.ict_inv(*synth[:3])
        lo, hi = -(1 << (B - 1)), (1 << (B - 1)) - 1
        for (c, x0, y0, x1, y1), f in zip(rects, synth):
            ox, oy = comp_org[c]
            sl = (slice(y0 - oy, y1 - oy), slice(x0 - ox, x1 - ox))
            t = f * float(1 << B)
            m_syn = float(np.abs(f).max()) if f.size else 0.0
            tau = C_INV * max(D, 1) * M.U32 * max(m_syn, 0.5) * (1 << B)
            r_lib = out[c][sl] - half
            clip = None if st == ob.I32 else (-half, (1 << B) - 1 - half)
            nbad, ntie, first = M.check_rounding(r_lib, t, tau, lo, hi, clip)
            off = (r_lib != M.expected_rounding(t, lo, hi, clip)) & (np.abs(t + half) < 2 ** B - 1)
            if off.any():      # how far inside the band the rounding decisions that differ lie, in units of tau / C_INV
                s["inv_ratio"] = max(s["inv_ratio"], float(np.abs(t - np.floor(t) - 0.5)[off].max()) * C_INV / tau)
            assert nbad == 0, ("decoded sample differs from the model's", name, tile, c, first,
                               None if first is None else (int(r_lib[first]), float(t[first])))
            s["inv_n"] += t.size; s["inv_tie"] += ntie
            # the reference's decode of the same stream: the model's rule holds for it too, it is within one of ours,
            # and it differs from ours only inside the model's tie band
            nbad_ref, _, first = M.check_rounding(refout[c][sl] - half, t, tau, lo, hi, clip)
            assert nbad_ref == 0, ("the reference's decode differs from the model's", name, tile, c, first)
            dr = refout[c][sl] - out[c][sl]
            assert np.abs(dr).max(initial=0) <= 1, (name, tile, c)
            fl = np.floor(t)
            in_band = np.abs(t - fl - 0.5) <= tau
            assert not (dr != 0)[~in_band].any(), ("reference differs outside the tie band", name, tile, c)
            s["cross_n"] += t.size; s["cross_diff"] += int((dr != 0).sum())
    for k in ("fwd", "inv"):
        assert s[k + "_tie"] <= TIE_FRACTION * max(s[k + "_n"], 1) + 2, (name, k, s)
    return s, p


def _report(name, s):
    print("%s: forward %d/%d in the tie band, inverse %d/%d, reference differs on %d/%d, K_max %d, error ratios %.1f / %.1f"
          % (name, s["fwd_tie"], s["fwd_n"], s["inv_tie"], s["inv_n"], s["cross_diff"], s["cross_n"], s["kmax"],
             s["fwd_ratio"], s["inv_ratio"]))


def _port_exact(lib, name):
    """the quantised planes equal the float32 restatement's (the reference's order: __fmul_rn / __fadd_rn, no FMA,
    round-to-nearest-even quantiser) bit for bit, on one tile"""
    import oracleport as O
    kw = ALL[name]
    p = cases.make(_strip(kw))
    if p.tile_w or any(p.dx[c] != 1 or p.dy[c] != 1 for c in range(p.num_comps)):
        return
    frame = cases.frame_for(p)
    st = kw["st"]
    planes = frame if st == ob.I32 else [f.astype(np.uint8 if st == ob.U8 else np.uint16) for f in frame]
    enc = ob.Encoder(p, st, lib=lib)
    enc.encode(planes)
    D = p.num_decomps
    info = {(c, r, b): enc.band_info(0, c, r, b) for c in range(p.num_comps) for r, b in _bands(D)}
    layout = {"origin": lambda c: (info[(c, D, 1)]["res_x0"], info[(c, D, 1)]["res_y0"]),
              "quant": lambda c, r, b: (info[(c, r, b)]["K_max"], info[(c, r, b)]["delta_inv"])}
    want = O.forward_bands(p, frame, layout)
    for key, w in want.items():
        assert np.array_equal(enc.read_band(0, *key), w), (name, key)


# ---- CPU tier -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n, _ in CPU_CASES])
def test_irv_against_model_emulated(name, emu_lib, ref):
    s, p = run_case(emu_lib, name, ref)
    _report(name, s)
    _port_exact(emu_lib, name)
    if name == "fine_qstep_kmax16":
        assert s["kmax"] > 15
    if name == "levels5_deep":       # the deepest resolutions are 1 to 3 samples across
        enc = ob.Encoder(p, ob.I32, lib=emu_lib)
        assert enc.band_info(0, 0, 1, 1)["w"] <= 3 and enc.band_info(0, 0, 1, 2)["h"] <= 3


def test_model_matches_float32_restatement(emu_lib):
    """the float32 restatement of the reference's forward path (oracleport) against the model under the rule, on the
    configurations whose quantised planes the library must match bit for bit (the encoder is only configured here, for
    its band table)"""
    import oracleport as O
    for name in ("w243_x5", "ict_u16_12bit", "signed12_i32", "levels5_deep", "thin_1xN", "q90_split"):
        kw = ALL[name]
        p = cases.make(_strip(kw))
        frame = cases.frame_for(p)
        enc = ob.Encoder(p, ob.I32, lib=emu_lib)
        D, B, signed = p.num_decomps, p.bit_depth[0], bool(p.is_signed[0])
        info = {(c, r, b): enc.band_info(0, c, r, b) for c in range(p.num_comps) for r, b in _bands(D)}
        layout = {"origin": lambda c: (info[(c, D, 1)]["res_x0"], info[(c, D, 1)]["res_y0"]),
                  "quant": lambda c, r, b: (info[(c, r, b)]["K_max"], info[(c, r, b)]["delta_inv"])}
        port = O.forward_bands(p, frame, layout)
        n = ties = 0
        for c in range(p.num_comps):
            xs = [M.to_float(f, B, signed) for f in frame]
            x = M.ict_fwd(*xs, c) if p.color_transform else xs[c]
            bands, mags = M.analyse(x, *layout["origin"](c), D)
            for (r, b), a in bands.items():
                kmax, dinv = info[(c, r, b)]["K_max"], float(info[(c, r, b)]["delta_inv"])
                g = port[(c, r, b)]
                t = a * dinv
                d = D - r + 1 if r else D
                e_v = C_FWD * d * M.U32 * max(mags[:d]) * dinv + M.U32 * np.abs(t) + 0.5
                gs = np.where(g & 0x80000000, -1.0, 1.0) * (g & 0x7FFFFFFF).astype(np.float64)
                assert (np.abs(gs - t) <= e_v).all(), (name, c, r, b)
                sh = 2.0 ** (31 - kmax)
                nbad, ntie, first = M.check_rounding((g & 0x7FFFFFFF) >> np.uint32(31 - kmax), np.abs(t) / sh - 0.5, e_v / sh)
                assert nbad == 0, (name, c, r, b, first)
                n += g.size; ties += ntie
        assert ties <= TIE_FRACTION * n, (name, ties, n)


def test_reference_block_decoder_dequantises_as_the_model(ref):
    """cleanup-only blocks through the reference's block decoder and its gen_irv_tx_from_cb32: the half-LSB
    reconstruction bit and the float32 product are what ref97.dequantise_f32 computes, and within one float32
    rounding of ref97.dequantise"""
    import ctypes as C
    L = ref.lib()
    rng = np.random.default_rng(97)
    for it in range(60):
        w = int(rng.integers(1, 65)); h = int(rng.integers(1, min(64, 4096 // w) + 1))
        kmax = int(rng.integers(2, 25))
        mag = np.minimum(np.abs(rng.laplace(0, 2 ** (kmax / 2.5), (h, w))).astype(np.uint64), (1 << kmax) - 1)
        if not mag.any():
            continue
        sign = rng.integers(0, 2, (h, w), dtype=np.uint64)
        # a quantiser word: coded bits at 30 .. 31-kmax and arbitrary bits below them, which the coder drops
        low = rng.integers(0, 1 << (31 - kmax), (h, w), dtype=np.uint64)
        words = ((sign << 31) | (mag << (31 - kmax)) | low).astype(np.uint32)
        data = ref.encode_block(words & np.uint32(~((1 << (31 - kmax)) - 1) & 0xFFFFFFFF), kmax - 1)
        dec, ok = ref.decode_block(data, w, h, kmax - 1, 1, len(data), 0)
        assert ok
        delta = np.float32(rng.uniform(0.5, 2.0) * 2.0 ** -(31 - kmax))
        got = np.zeros(dec.size, np.float32)
        src = np.ascontiguousarray(dec.ravel(), np.uint32)
        L.ojr_irv_tx_from_cb32(src.ctypes.data_as(C.c_void_p), got.ctypes.data_as(C.c_void_p), C.c_float(delta),
                               C.c_uint32(src.size))
        want = M.dequantise_f32(words.ravel(), kmax, delta)
        nz = mag.ravel() != 0
        assert np.array_equal(got.view(np.uint32)[nz], want[nz]), (it, w, h, kmax)
        assert (got[~nz] == 0).all(), (it, w, h, kmax)
        f64 = M.dequantise(words.ravel(), kmax, float(delta))
        assert (np.abs(got.astype(np.float64) - f64) <= M.U32 * np.abs(f64)).all(), (it, w, h, kmax)


# ---- GPU tier -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n, _ in CPU_CASES + BIG_CASES])
def test_irv_against_model_gpu(name, gpu_lib, ref):
    s, _ = run_case(None, name, ref)
    _report(name, s)
    _port_exact(None, name)


def test_gpu_tier_covers_the_large_chunks():
    """the GPU tier's frames reach 32-row forward and 64-row inverse chunks at level 1, several strips wide; a later
    retuning of the tiling that drops one of these seams from the tier fails here"""
    fwd = {_level1(kw)[0] for _, kw in BIG_CASES}
    inv = {_level1(kw)[1] for _, kw in BIG_CASES}
    assert {r for _, r in fwd} == {32}, fwd
    assert {r for _, r in inv} == {64}, inv
    assert min(s for s, _ in fwd | inv) >= 32
    small = {_level1(kw) for _, kw in CPU_CASES if min(kw["width"], kw["height"]) > 8}
    assert {r for f, i in small for r in (f[1], i[1])} == {8}     # the CPU tier crosses the 8-row seams
    assert max(f[0] for f, _ in small) >= 3                       # and more than two strips


def _variant_child(variant, gpu):
    if os.environ.get("OJB_IRV_VARIANT_CHILD"):
        pytest.skip("already inside the child run")
    env = dict(os.environ, OJB_IRV_VARIANT_CHILD="1", **VARIANTS[variant])
    args = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-p", "no:cacheprovider",
            "-k", ("gpu and (%s)" if gpu else "emulated and (%s)") % " or ".join(
                VARIANT_CASES + (VARIANT_GPU_EXTRA.get(variant, []) if gpu else []))]
    if gpu:
        args += ["-m", "gpu"]
    r = subprocess.run(args, env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_irv_variants_emulated(variant, emu_lib, ref):
    _variant_child(variant, False)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_irv_variants_gpu(variant, gpu_lib, ref):
    _variant_child(variant, True)
