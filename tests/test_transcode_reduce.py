"""Transcoding a codestream to a lower resolution: Encoder.from_codestream(j2c, skipped_res=r) /
ojb_enc_transcode_headers_reduced drops the input's top r resolution levels and re-codes the kept code-blocks.

  * Exact resolution oracle: the reference's decode of the output equals its decode of the input restricted to (r, r),
    sample for sample, 5/3 and 9/7 alike, and so does this library's; `dims` / info are the reference's reduced sizes.
  * Blocks carried over: the output lists the input's kept blocks with their missing MSBs, passes, lengths and bytes,
    and the transcoder's band planes hold the words the full-geometry transcoder holds for those bands.
  * reduce(r1) then reduce(r2) is reduce(r1 + r2); skipped_res = 0 is the plain transcode; frames and reconfigures.
  * Targets: a reduced transcode to a size or quality target is the transcode of the reduced stream to that target.
  * Coverage: per-component level counts down to zero, progressions with precincts, tile-part divisions with TLM,
    sub-sampling, offsets, 16-bit / signed components, NLT, ATK, the SigProp / MagRef golden stream, seeded random
    configurations.
  * Refusals: one code per cause, each leaving the encoder usable.
"""
import ctypes as C
import os

import numpy as np
import pytest

import cases
from openjph_b200 import _lib
from openjph_b200 import codestream as cs
from test_random_configs import random_case
from test_rate_control import CPU_CONFIGS, GPU_CONFIGS

_HERE = os.path.dirname(os.path.abspath(__file__))
NON_DFS = [c for c in CPU_CONFIGS if "decomp" not in c[1]]
# configurations whose reduced tile grid cannot keep every tile: code per r
GRID_REFUSED = {("tiles_tp_tlm_off", 3): "0x000B0055"}


def _levels(kw):
    return min([kw.get("num_decomps", 5)] + [st.get("num_decomps", 5) for st in kw.get("coc", {}).values()])


def _headers(L, j2c, r, on_device=False):
    """(return code, message, info) of ojb_enc_transcode_headers_reduced on a fresh encoder"""
    t = cs.Encoder.__new__(cs.Encoder)
    cs._Base.__init__(t, L)
    t.h = L.ojb_enc_create()
    buf = np.frombuffer(bytes(j2c), np.uint8)
    info = _lib.FrameInfo()
    rc = L.ojb_enc_transcode_headers_reduced(t.h, buf.ctypes.data, buf.size, 0, cs.I32, r, C.byref(info))
    msg = L.ojb_last_error().decode()
    t.close()
    return rc, msg, info


def _ours_restricted(L, j2c, r):
    d = cs.Decoder(lib=L)
    try:
        return d.decode(j2c, skip=(r, r))
    finally:
        d.close()


def _ours(L, j2c):
    d = cs.Decoder(lib=L)
    try:
        return d.decode(j2c), d.list_blocks()
    finally:
        d.close()


def _equal(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def _exact(L, ref, j2c, r):
    """item 1 of the feature: the output of a reduced transcode decodes as the input restricted to (r, r)"""
    t = cs.Encoder.from_codestream(j2c, lib=L, skipped_res=r)
    out = t.transcode(j2c)
    theirs, _ = ref.decode(out)
    want, info = ref.decode_restricted(j2c, r, r)
    assert _equal(theirs, want), r
    assert _equal(_ours(L, out)[0], _ours_restricted(L, j2c, r)), r
    assert t.dims == [(int(info.comp_w[c]), int(info.comp_h[c])) for c in range(info.num_comps)]
    return t, out


def _groups(enc):
    """per (tile, component): the (resolution, band, number of blocks) in the order the encoder numbers blocks"""
    out, t = [], 0
    while True:
        try:
            enc.band_info(t, 0, 0, 0)
        except cs.OjphError:
            return out
        for c in range(len(enc.dims)):
            res, k = [], 0
            while True:
                try:
                    enc.band_info(t, c, k, 0 if k == 0 else 1)
                except cs.OjphError:
                    break
                res.append([(k, b, enc.band_info(t, c, k, b)["nblocks"]) for b in ([0] if k == 0 else [1, 2, 3])])
                k += 1
            out.append((t, c, [g for level in reversed(res) for g in level]))
        t += 1


def _kept_blocks(full, reduced):
    """the input's block indices (numbered as `full` numbers them) of the blocks `reduced` keeps, in its order"""
    kept, base = [], 0
    g_red = {(t, c): groups for t, c, groups in _groups(reduced)}
    for t, c, groups in _groups(full):
        top = max(k for k, _, _ in g_red[(t, c)])
        for k, b, n in groups:
            if k <= top:
                kept.extend(range(base, base + n))
            base += n
    return kept


def _blocks_carried(L, j2c, out, r):
    """item 2: the kept blocks come through unchanged, in bytes and in the transcoder's band planes"""
    full = cs.Encoder.from_codestream(j2c, lib=L)
    full.transcode(j2c)
    red = cs.Encoder.from_codestream(j2c, lib=L, skipped_res=r)
    assert red.transcode(j2c) == out
    _, ib = _ours(L, j2c)
    _, ob = _ours(L, out)
    kept = _kept_blocks(full, red)
    assert len(kept) == len(ob)
    for o, i in zip(ob, (ib[k] for k in kept)):
        assert (o.w, o.h, o.missing_msbs, o.num_passes, o.len1, o.len2) == (i.w, i.h, i.missing_msbs, i.num_passes, i.len1, i.len2)
        assert out[o.byte_off:o.byte_off + o.len1 + o.len2] == j2c[i.byte_off:i.byte_off + i.len1 + i.len2]
    # read_band: the reduced transcoder's planes hold the full-geometry transcoder's words of every kept band.  The
    # restricted decoder lays its arena out for the input's geometry, so this is what plan_block_map's offsets give
    for t, c, groups in _groups(red):
        for k, b, _ in groups:
            assert np.array_equal(red.read_band(t, c, k, b), full.read_band(t, c, k, b)), (t, c, k, b)


def _encoded(L, ref, kw, who):
    p = cases.make(kw)
    frame = cases.frame_for(p)
    return ref.encode(p, frame) if who == "ref" else cs.Encoder(p, lib=L).encode(frame)


def _claim_broadcast(j2c):
    """the stream with Rsiz naming the broadcast profile (single tile, level 1) in its Part 1 field"""
    b = bytearray(j2c)
    rsiz = int.from_bytes(b[6:8], "big") | 0x0101
    b[6:8] = rsiz.to_bytes(2, "big")
    return bytes(b)


def _config(L, ref, name, kw, blocks=True):
    for who in ("ref", "ours"):
        j = _encoded(L, ref, kw, who)
        for r in range(1, _levels(kw) + 1):
            code = GRID_REFUSED.get((name, r))
            if code:
                rc, msg, _ = _headers(L, j, r)
                assert rc != 0 and code in msg, (name, r, msg)
                continue
            _, out = _exact(L, ref, j, r)
            if blocks and who == "ours":
                _blocks_carried(L, j, out, r)
        if name == "irv_broadcast":
            # an unmarked stream claims no profile (neither writer records one in Rsiz); one that names the broadcast
            # profile keeps 1 to 5 levels
            claimed = _claim_broadcast(j)
            _exact(L, ref, claimed, 4)
            rc, msg, _ = _headers(L, claimed, 5)
            assert rc != 0 and "0x000B0056" in msg, msg


@pytest.mark.parametrize("name,kw", NON_DFS, ids=[c[0] for c in NON_DFS])
def test_exact_emulator(emu_lib, ref, name, kw):
    _config(emu_lib, ref, name, kw)


# ---- composition, identity, frames ------------------------------------------------------------------------------------
def _reduce(L, j2c, r):
    return cs.Encoder.from_codestream(j2c, lib=L, skipped_res=r).transcode(j2c) if r else j2c


def _composition(L):
    for idx, pairs in ((0, [(1, 1), (1, 2), (2, 1)]), (5, [(2, 3), (1, 1)]), (10, [(1, 1)]), (15, [(1, 2)])):
        name, kw = CPU_CONFIGS[idx]
        j = _encoded(L, None, kw, "ours")
        for r1, r2 in pairs:
            assert _reduce(L, _reduce(L, j, r1), r2) == _reduce(L, j, r1 + r2), (name, r1, r2)
    # skipped_res = 0 through the new call is the plain transcode, and info is the input's geometry
    name, kw = CPU_CONFIGS[10]
    j = _encoded(L, None, kw, "ours")
    t = cs.Encoder.from_codestream(j, lib=L)
    buf = np.frombuffer(j, np.uint8)
    info = _lib.FrameInfo()
    assert L.ojb_enc_transcode_headers_reduced(t.h, buf.ctypes.data, buf.size, 0, cs.I32, 0, C.byref(info)) == 0
    assert t.transcode(j) == j
    assert [(info.comp_w[c], info.comp_h[c]) for c in range(info.num_comps)] == cs._siz_of(j)[0]
    # a second frame of the same headers, then a stream with other headers, on one encoder
    p = cases.make(kw)
    j2 = cs.Encoder(p, lib=L).encode(cases.frame_for(p, seed=9))
    t = cs.Encoder.from_codestream(j, lib=L, skipped_res=1)
    a = t.transcode(j)
    assert t.transcode(j2) == _reduce(L, j2, 1)
    assert t.transcode(j) == a
    other = _encoded(L, None, CPU_CONFIGS[0][1], "ours")
    assert t.transcode(other) == _reduce(L, other, 1)
    assert t.transcode(j) == a


def test_composition_emulator(emu_lib):
    _composition(emu_lib)


# ---- targets ---------------------------------------------------------------------------------------------------------
def _sse(a, b):
    return sum(int(np.sum((x.astype(np.int64) - y.astype(np.int64)) ** 2)) for x, y in zip(a, b))


def _targets(L, j2c, r, fractions=(1 / 4, 1 / 16), mse_fracs=(0.05, 0.3), psnr=None, tensors=False):
    """item 4: a reduced transcode to a target is the transcode of the reduced stream to that target"""
    red = _reduce(L, j2c, r)
    src = j2c
    if tensors:
        import torch
        src = torch.from_numpy(np.frombuffer(j2c, np.uint8).copy()).cuda()
        host = lambda x: x.cpu().numpy().tobytes()
    else:
        host = lambda x: x
    a = cs.Encoder.from_codestream(src, lib=L, skipped_res=r)
    b = cs.Encoder.from_codestream(red, lib=L)
    assert a.min_size == b.min_size and a.dims == b.dims
    for f in fractions:
        T = max(a.min_size, int(len(red) * f))
        a.set_target_size(T)
        b.set_target_size(T)
        got = host(a.transcode(src))
        assert got == b.transcode(red) and len(got) <= T, (r, f)
        ia, ib = a.rate_info(), b.rate_info()
        for key in ("kmax", "k", "R"):
            assert np.array_equal(ia[key], ib[key]), (r, f, key)
        assert ia["rounds"] == ib["rounds"] and ia["budget"] == ib["budget"]
    a.set_target_size(0)
    srcdec = _ours_restricted(L, j2c, r)
    empty = cs.Encoder.from_codestream(red, lib=L, target_bytes=b.min_size).transcode(red)
    worst = _sse(_ours(L, empty)[0], srcdec)
    n = sum(x.size for x in srcdec)
    targets = [dict(target_mse=worst / n * fr) for fr in mse_fracs] + ([dict(target_psnr=psnr)] if psnr else [])
    for tg in targets:
        qa = cs.Encoder.from_codestream(src, lib=L, skipped_res=r, **tg)
        qb = cs.Encoder.from_codestream(red, lib=L, **tg)
        got = host(qa.transcode(src))
        assert got == qb.transcode(red), (r, tg)
        ia, ib = qa.quality_info(), qb.quality_info()
        assert ia["rounds"] == ib["rounds"] and ia["sse"] == ib["sse"] and ia["limit"] == ib["limit"]
        # the source is the input's restricted decode
        assert _sse(_ours(L, got)[0], srcdec) == ia["sse"], (r, tg)
        assert ia["sse"] <= ia["limit"] or not ia["reached"]


def test_targets_emulator(emu_lib):
    for idx, r in ((0, 1), (5, 2), (10, 1)):
        _targets(emu_lib, _encoded(emu_lib, None, CPU_CONFIGS[idx][1], "ours"), r)


# ---- coverage --------------------------------------------------------------------------------------------------------
COVERAGE = [
    # component 1 has one level of its own: r = 1 leaves it without levels
    ("coc_levels", dict(width=150, height=110, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, planar=1,
                        coc={1: dict(reversible=True, num_decomps=1, block=(32, 32)),
                             2: dict(reversible=False, num_decomps=2, block=(16, 64))})),
    ("coc_precincts", dict(width=160, height=120, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, planar=1,
                           precincts=[(64, 64), (128, 128)], coc={0: dict(reversible=True, num_decomps=2, block=(32, 32))})),
    ("tp_both_tlm", dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=3, reversible=True,
                         prog_order="LRCP", tilepart_div=3, tlm=True, tile=(64, 64))),
    ("tp_comp_cprl", dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=2, reversible=True,
                          prog_order="CPRL", tilepart_div=2, tlm=True)),
    ("sub420_offsets", dict(width=203, height=151, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, planar=1,
                            subsampling=[(1, 1), (2, 2), (2, 2)], offset=(5, 3), tile=(128, 64), tile_offset=(2, 1))),
    ("signed16", dict(width=90, height=70, num_comps=2, bit_depth=16, is_signed=True, num_decomps=3, reversible=True)),
    ("nlt3", dict(width=96, height=64, num_comps=1, bit_depth=12, is_signed=True, num_decomps=3, reversible=True,
                  nlt={"all": 3})),
    ("atk_irv", dict(width=120, height=90, num_comps=1, bit_depth=8, num_decomps=3, reversible=False,
                     atk=dict(K=1.0, A=[0.25, -0.5]))),
]


def _coverage(L, ref, kw):
    j = _encoded(L, ref, kw, "ours")
    for r in range(1, _levels(kw) + 1):
        _, out = _exact(L, ref, j, r)
        _blocks_carried(L, j, out, r)


@pytest.mark.parametrize("name,kw", COVERAGE, ids=[c[0] for c in COVERAGE])
def test_coverage_emulator(emu_lib, ref, name, kw):
    _coverage(emu_lib, ref, kw)


def _foreign(L, ref):
    """the SigProp / MagRef stream: its reduced transcodes decode as its r = 0 transcode restricted"""
    src = np.load(os.path.join(_HERE, "golden", "test_j2c.npz"))["cs"].tobytes()
    base = cs.Encoder.from_codestream(src, lib=L).transcode(src)
    r = 1
    while True:
        rc, msg, _ = _headers(L, src, r)
        if rc != 0:
            assert "0x000300A2" in msg or "0x000B0007" in msg, msg
            break
        out = _reduce(L, src, r)
        assert _equal(ref.decode(out)[0], ref.decode_restricted(base, r, r)[0]), r
        r += 1
    assert r > 1


def test_foreign_emulator(emu_lib, ref):
    _foreign(emu_lib, ref)


def _random(L, ref, seed):
    kw = random_case(seed)
    r = int(np.random.default_rng(90000 + seed).integers(1, max(1, kw["num_decomps"]) + 1))
    j = _encoded(L, ref, kw, "ours")
    try:
        want, _ = ref.decode_restricted(j, r, r)
    except RuntimeError:
        want = None
    rc, msg, _ = _headers(L, j, r)
    if rc != 0:
        # the documented refusals: levels, tile grid; and an input no decoder reads back (tile-part divisions with
        # components of different level counts, as in test_random_configs), refused as undecodable
        codes = ("0x000300A2", "0x000B0007", "0x000B0055") + (("0x000B0051",) if want is None else ())
        assert any(code in msg for code in codes), (kw, r, msg)
        return
    if want is None:
        # the reference cannot read the input back at all (tile-part divisions with components of different level
        # counts, as in test_random_configs): this library's restricted decode is the yardstick
        out = _reduce(L, j, r)
        assert _equal(_ours(L, out)[0], _ours_restricted(L, j, r)), (kw, r)
        return
    _exact(L, ref, j, r)


@pytest.mark.parametrize("seed", range(60))
def test_random_emulator(emu_lib, ref, seed):
    _random(emu_lib, ref, seed)


# ---- refusals --------------------------------------------------------------------------------------------------------
def _refusals(L):
    good_kw = dict(CPU_CONFIGS[10][1])                       # tiles of 128 x 100, tile-parts by resolution, TLM
    good = _encoded(L, None, good_kw, "ours")
    want = _reduce(L, good, 1)
    t = cs.Encoder.from_codestream(good, lib=L, skipped_res=1)
    coc = _encoded(L, None, COVERAGE[0][1], "ours")          # component 1 has one level
    dfs = _encoded(L, None, [c for c in CPU_CONFIGS if c[0] == "dfs_atk_irv"][0][1], "ours")
    bcast = _claim_broadcast(_encoded(L, None, [c for c in CPU_CONFIGS if c[0] == "irv_broadcast"][0][1], "ours"))
    sop = bytearray(good)
    cod = good.index(b"\xff\x52")
    sop[cod + 4] |= 2
    pw = cs.make_params(64, 64, 3, 32, num_decomps=5, reversible=True, color_transform=True)
    cases_ = [(good, 4, "0x000300A2"), (coc, 2, "0x000B0007"), (dfs, 1, "0x000B0054"), (good, 3, "0x000B0055"),
              (bcast, 5, "0x000B0056"), (bytes(sop), 1, "0x000B004C"),
              (cs.Encoder(pw, lib=L).encode(cases.frame_for(pw)), 1, "0x000B0050"),
              (good[:len(good) * 2 // 3], 1, "0x000B0051")]
    buf_keep = []
    for s, r, code in cases_:
        buf = np.frombuffer(s, np.uint8)
        buf_keep.append(buf)
        rc = L.ojb_enc_transcode_headers_reduced(t.h, buf.ctypes.data, buf.size, 0, cs.I32, r, None)
        assert rc != 0 and code in L.ojb_last_error().decode(), (code, L.ojb_last_error().decode())
        # the encoder takes the next configuration
        g = np.frombuffer(good, np.uint8)
        assert L.ojb_enc_transcode_headers_reduced(t.h, g.ctypes.data, g.size, 0, cs.I32, 1, None) == 0
        assert t.transcode(good) == want, code
    with pytest.raises(cs.OjphError, match="0x000B0053"):
        t.encode([np.zeros((h, w), np.int32) for w, h in t.dims])
    assert t.transcode(good) == want


def test_refusals_emulator(emu_lib):
    _refusals(emu_lib)


# ---- on the H100 -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", NON_DFS, ids=[c[0] for c in NON_DFS])
def test_exact_gpu(gpu_lib, ref, name, kw):
    _config(gpu_lib, ref, name, kw)


@pytest.mark.gpu
def test_composition_gpu(gpu_lib):
    _composition(gpu_lib)


@pytest.mark.gpu
def test_targets_gpu(gpu_lib):
    for idx, r in ((0, 1), (5, 2), (10, 1)):
        _targets(gpu_lib, _encoded(gpu_lib, None, CPU_CONFIGS[idx][1], "ours"), r)


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", COVERAGE, ids=[c[0] for c in COVERAGE])
def test_coverage_gpu(gpu_lib, ref, name, kw):
    _coverage(gpu_lib, ref, kw)


@pytest.mark.gpu
def test_foreign_gpu(gpu_lib, ref):
    _foreign(gpu_lib, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(40))
def test_random_gpu(gpu_lib, ref, seed):
    _random(gpu_lib, ref, seed)


@pytest.mark.gpu
def test_refusals_gpu(gpu_lib):
    _refusals(gpu_lib)


def _large(L, ref, kw, rs, psnr=None):
    """a large frame through CUDA tensors: items 1, 2 and 4"""
    import torch
    j = _encoded(L, ref, kw, "ours")
    src = torch.from_numpy(np.frombuffer(j, np.uint8).copy()).cuda()
    for r in rs:
        t = cs.Encoder.from_codestream(src, lib=L, skipped_res=r)
        out = t.transcode(src)
        assert out.is_cuda
        host = out.cpu().numpy().tobytes()
        assert host == _reduce(L, j, r)
        want, info = ref.decode_restricted(j, r, r)
        assert _equal(ref.decode(host)[0], want), r
        assert _equal(_ours(L, host)[0], _ours_restricted(L, j, r)), r
        assert t.dims == [(int(info.comp_w[c]), int(info.comp_h[c])) for c in range(info.num_comps)]
        _blocks_carried(L, j, host, r)
        _targets(L, j, r, fractions=(1 / 4, 1 / 16), mse_fracs=(0.2,), psnr=psnr if r == 1 else None, tensors=True)


@pytest.mark.gpu
def test_hd_gpu(gpu_lib, ref):
    _large(gpu_lib, ref, dict(GPU_CONFIGS[0][1]), (1, 2))


@pytest.mark.gpu
def test_4k_irv_gpu(gpu_lib, ref):
    _large(gpu_lib, ref, dict(GPU_CONFIGS[1][1]), (1,))


@pytest.mark.gpu
def test_8k_gpu(gpu_lib, ref):
    _large(gpu_lib, ref, dict(GPU_CONFIGS[2][1]), (1, 2), psnr=40.0)
