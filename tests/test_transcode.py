"""Transcoding a codestream from its code-blocks (Encoder.from_codestream / transcode; ojb_enc_transcode_headers /
ojb_enc_transcode).

  * Identity without a target: for every configuration of the rate tests, transcode(encode(img)) == encode(img) byte
    for byte, and the coefficient arena the transcode fills (read_band) equals the pixel encoder's.
  * Identity with a target for lossless inputs: a transcode of the lossless stream to a size or quality target is the
    pixel encoder's stream at that target, with the same selection tables / search rounds; once more under the
    general block coders and the warp-per-block encoder.
  * Lossy inputs (a 9/7 q90 stream, a 5/3 stream already cut by a size target): every output holds its target and
    decodes with the reference, every included block's missing-MSB count is 30 - q_b - k and its bytes are the reference
    block encoder's on the input block's reference decode with the bits below q_b cleared; quality targets report the
    SSE numpy measures between the output's and the input's decode.
  * A foreign stream whose blocks carry SigProp / MagRef passes (tests/golden/test_j2c.npz) comes back cleanup-only:
    1- and 3-pass blocks decode to the input's words, 2-pass blocks differ by exactly a quarter of the cleanup step on
    the samples that became significant in the cleanup pass.
  * Refusals: one code per cause, each leaving the encoder usable.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import cases
from openjph_b200 import codestream as cs
from test_rate_control import CPU_CONFIGS, GPU_CONFIGS, _decode_ours

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
REV_CONFIGS = [c for c in CPU_CONFIGS if c[1].get("reversible")]


def _bands(enc, p):
    out = []
    ntiles = 1 if not p.tile_w else -(-(p.width - p.tile_off_x) // p.tile_w) * -(-(p.height - p.tile_off_y) // p.tile_h)
    for t in range(ntiles):
        for c in range(p.num_comps):
            for r in range(p.num_decomps + 1):
                for b in ([0] if r == 0 else [1, 2, 3]):
                    out.append((enc.read_band(t, c, r, b), enc.band_info(t, c, r, b)["K_max"]))
    return out


def _identity(L, kw):
    p = cases.make(kw)
    frame = cases.frame_for(p)
    e = cs.Encoder(p, lib=L)
    want = e.encode(frame)
    planes = _bands(e, p)
    t = cs.Encoder.from_codestream(want, lib=L)
    assert t.transcode(want) == want
    # the coded part of the pixel encoder's words: the 9/7 quantiser's words also hold bits below the band's least
    # significant plane (31 - K_max) and the signs of magnitudes quantised to 0, neither of which a codestream carries
    for (a, _), (b, K) in zip(_bands(t, p), planes):
        b = b & np.uint32((0xFFFFFFFF << (31 - K)) & 0xFFFFFFFF)
        assert np.array_equal(a, np.where(b & np.uint32(0x7FFFFFFF), b, np.uint32(0)))
    # a second frame call on the same configuration, and a reconfigure by a stream of another frame
    assert t.transcode(want) == want
    other = cs.Encoder(p, lib=L).encode(cases.frame_for(p, seed=9))
    assert t.transcode(other) == other
    return p, frame, want


@pytest.mark.parametrize("name,kw", CPU_CONFIGS, ids=[c[0] for c in CPU_CONFIGS])
def test_identity_emulator(emu_lib, name, kw):
    _identity(emu_lib, kw)


def _lossless_targets(L, kw, fractions=(0.005, 0.10, 0.30), mse_fracs=(0.02, 0.2), rate_tables=True):
    p = cases.make(kw)
    frame = cases.frame_for(p)
    full = cs.Encoder(p, lib=L).encode(frame)
    t = cs.Encoder.from_codestream(full, lib=L)
    e = cs.Encoder(p, lib=L)
    assert t.min_size == e.min_size
    for T in [max(e.min_size, int(len(full) * f)) for f in fractions] + [e.min_size]:
        e.set_target_size(T)
        t.set_target_size(T)
        want, got = e.encode(frame), t.transcode(full)
        assert got == want and len(got) <= T, T
        if rate_tables:
            a, b = e.rate_info(), t.rate_info()
            for key in ("kmax", "k", "R"):
                assert np.array_equal(a[key], b[key]), (T, key)
            assert a["rounds"] == b["rounds"] and a["budget"] == b["budget"]
    # a target at or above the unconstrained size changes nothing
    t.set_target_size(2 * len(full))
    assert t.transcode(full) == full
    t.set_target_size(0)
    # quality targets: the source is the decoded input, here the original image
    empty = cs.Encoder(p, lib=L, target_bytes=e.min_size).encode(frame)
    dec, _ = _decode_ours(L, empty)
    worst = sum(float(np.sum((a.astype(np.float64) - f.astype(np.float64)) ** 2)) for a, f in zip(dec, frame))
    n = sum(f.size for f in frame)
    for fr in mse_fracs:
        m = worst / n * fr
        a = cs.Encoder(p, lib=L, target_mse=m)
        b = cs.Encoder.from_codestream(full, lib=L, target_mse=m)
        assert b.transcode(full) == a.encode(frame), fr
        qa, qb = a.quality_info(), b.quality_info()
        assert qa["rounds"] == qb["rounds"] and qa["sse"] == qb["sse"] and qa["limit"] == qb["limit"]
    return p, frame, full


@pytest.mark.parametrize("name,kw", REV_CONFIGS, ids=[c[0] for c in REV_CONFIGS])
def test_lossless_targets_emulator(emu_lib, name, kw):
    _lossless_targets(emu_lib, kw)


def _variant_sha(lib_kind, env, kw, frac):
    code = (
        "import sys, hashlib; sys.path[:0] = [%r, %r]\n"
        "import cases\nfrom openjph_b200 import codestream as cs\n"
        "L = __import__('emu').emu_lib(build=False) if %r == 'emu' else __import__('openjph_b200._lib', fromlist=['x']).lib()\n"
        "p = cases.make(%r); f = cases.frame_for(p)\n"
        "full = cs.Encoder(p, lib=L).encode(f); T = int(len(full) * %r)\n"
        "a = cs.Encoder(p, lib=L, target_bytes=T).encode(f)\n"
        "b = cs.Encoder.from_codestream(full, lib=L, target_bytes=T).transcode(full)\n"
        "print(hashlib.sha256(a).hexdigest(), hashlib.sha256(b).hexdigest())\n") % (_ROOT, _HERE, lib_kind, kw, frac)
    full_env = dict(os.environ)
    full_env.update(env)
    return subprocess.check_output([sys.executable, "-c", code], env=full_env, cwd=_ROOT, text=True).split()


def test_variants_emulator(emu_lib):
    for env in ({"OJB_NO_FAST_BLOCKS": "1"}, {"OJB_BLOCK_ENCODER": "warp"}):
        a, b = _variant_sha("emu", env, dict(CPU_CONFIGS[0][1]), 0.1)
        assert a == b, env


# ---- lossy inputs ------------------------------------------------------------------------------------------------------
def _input_blocks(L, j2c):
    d = cs.Decoder(lib=L)
    d.decode(j2c)
    out = d.list_blocks()
    d.close()
    return out


def _q(bd):
    refined = bd.num_passes > 1 and bd.len2 and bd.missing_msbs < 29
    return (29 if refined else 30) - bd.missing_msbs


def _check_lossy_output(L, ref, src, ib, out, info, rev, bit_depths):
    """out transcoded from src (blocks ib) with the selection info"""
    ob = _input_blocks(L, out)
    assert len(ob) == len(ib)
    kmax, k = info["kmax"].astype(int), info["k"].astype(int)
    for b, (i, o) in enumerate(zip(ib, ob)):
        if not i.len1:
            assert not o.len1 and kmax[b] == 0, b
            continue
        q = _q(i)
        assert kmax[b] == 31 - q, b
        if not o.len1:
            continue
        assert o.num_passes == 1 and o.missing_msbs == 30 - q - k[b], b
        words, ok = ref.decode_block(src[i.byte_off:i.byte_off + i.len1 + i.len2], i.w, i.h, i.missing_msbs, i.num_passes,
                                     i.len1, i.len2, bool(i.causal))
        assert ok
        words &= np.uint32(~((1 << q) - 1) & 0xFFFFFFFF)
        assert out[o.byte_off:o.byte_off + o.len1] == ref.encode_block(np.ascontiguousarray(words), int(o.missing_msbs)), b
        if k[b] == 0 and i.num_passes == 1:
            assert out[o.byte_off:o.byte_off + o.len1] == src[i.byte_off:i.byte_off + i.len1], b
    ours, _ = _decode_ours(L, out)
    theirs, _ = ref.decode(out)
    if rev:
        assert all(np.array_equal(a, r) for a, r in zip(ours, theirs))
    else:
        cases.assert_irv_matches_reference(ours, theirs, "transcode", bit_depths)
    return ours


def _sse(a, b):
    return sum(int(np.sum((x.astype(np.int64) - y.astype(np.int64)) ** 2)) for x, y in zip(a, b))


def _lossy(L, ref, src, fractions, mse_fracs, rev, bit_depths):
    ib = _input_blocks(L, src)
    srcdec, _ = _decode_ours(L, src)
    t = cs.Encoder.from_codestream(src, lib=L)
    for f in fractions:
        T = max(t.min_size, int(len(src) * f))
        t.set_target_size(T)
        out = t.transcode(src)
        assert len(out) <= T
        _check_lossy_output(L, ref, src, ib, out, t.rate_info(), rev, bit_depths)
    t.set_target_size(0)
    empty = cs.Encoder.from_codestream(src, lib=L)
    empty.set_target_size(empty.min_size)
    worst = _sse(_decode_ours(L, empty.transcode(src))[0], srcdec)
    n = sum(x.size for x in srcdec)
    for fr in mse_fracs:
        q = cs.Encoder.from_codestream(src, lib=L, target_mse=worst / n * fr)
        out = q.transcode(src)
        info = q.quality_info()
        got = _sse(_decode_ours(L, out)[0], srcdec)
        assert got == info["sse"] and (got <= info["limit"] or not info["reached"]), (fr, got, info["limit"])
        if rev:
            assert info["reached"]


def _lossy_inputs(L, ref, irv_kw, rev_kw, fractions=(0.5, 0.1), mse_fracs=(0.05, 0.3)):
    p = cases.make(irv_kw)
    src = cs.Encoder(p, lib=L).encode(cases.frame_for(p))
    _lossy(L, ref, src, fractions, mse_fracs, False, list(p.bit_depth)[:p.num_comps])
    p = cases.make(rev_kw)
    f = cases.frame_for(p)
    full = cs.Encoder(p, lib=L).encode(f)
    src = cs.Encoder(p, lib=L, target_bytes=int(len(full) * 0.3)).encode(f)
    _lossy(L, ref, src, fractions, mse_fracs, True, list(p.bit_depth)[:p.num_comps])


def test_lossy_inputs_emulator(emu_lib, ref):
    _lossy_inputs(emu_lib, ref, dict(CPU_CONFIGS[5][1]), dict(CPU_CONFIGS[0][1]))


# ---- a stream with SigProp / MagRef passes -----------------------------------------------------------------------------
def _foreign(L, ref):
    src = np.load(os.path.join(_HERE, "golden", "test_j2c.npz"))["cs"].tobytes()
    ib = _input_blocks(L, src)
    t = cs.Encoder.from_codestream(src, lib=L)
    out = t.transcode(src)
    ob = _input_blocks(L, out)
    counts = {}
    quarter = 0
    for i, o in zip(ib, ob):
        np_eff = i.num_passes if i.len1 else 0
        counts[np_eff] = counts.get(np_eff, 0) + 1
        if not i.len1:
            assert not o.len1
            continue
        q = _q(i)
        assert o.num_passes == 1 and o.missing_msbs == 30 - q
        a, ok = ref.decode_block(src[i.byte_off:i.byte_off + i.len1 + i.len2], i.w, i.h, i.missing_msbs, i.num_passes,
                                 i.len1, i.len2, bool(i.causal))
        b, ok2 = ref.decode_block(out[o.byte_off:o.byte_off + o.len1], o.w, o.h, o.missing_msbs, 1, o.len1, 0, bool(o.causal))
        assert ok and ok2
        if i.num_passes == 2 and i.len2:
            # cleanup-significant samples (a bit at q or above in the input's word, none below): their bin centre at q
            # became a coded bit, so they gain half of it again, 2^(q-1)
            mag_a, mag_b = a & np.uint32(0x7FFFFFFF), b & np.uint32(0x7FFFFFFF)
            cup = (mag_a >> np.uint32(q)) != 0
            cup &= (mag_a & np.uint32((1 << q) - 1)) == 0
            assert np.array_equal(mag_b[cup], mag_a[cup] + np.uint32(1 << (q - 1)))
            assert np.array_equal(b[~cup], a[~cup])
            assert np.array_equal(b >> np.uint32(31), a >> np.uint32(31))
            quarter += int(cup.sum())
        else:
            assert np.array_equal(a, b)
    print("foreign input: blocks per pass count", dict(sorted(counts.items())), "quarter-step samples", quarter)
    assert counts.get(2, 0) + counts.get(3, 0) > 0
    ref.decode(out)
    for T in (len(src) // 4, len(src) // 16):
        t.set_target_size(T)
        j = t.transcode(src)
        assert len(j) <= T
        ref.decode(j)
    t.set_target_size(0)
    q = cs.Encoder.from_codestream(src, lib=L, target_psnr=35.0)
    j = q.transcode(src)
    info = q.quality_info()
    srcdec, _ = _decode_ours(L, src)
    assert _sse(_decode_ours(L, j)[0], srcdec) == info["sse"]
    assert info["sse"] <= info["limit"] or not info["reached"]
    ref.decode(j)


def test_foreign_input_emulator(emu_lib, ref):
    _foreign(emu_lib, ref)


# ---- refusals ---------------------------------------------------------------------------------------------------------
def _segments(j2c):
    """(marker, offset, length incl. marker) of the main header's segments, and the first SOT's offset"""
    out, q = [], 2
    while True:
        m = int.from_bytes(j2c[q:q + 2], "big")
        if m == 0xFF90:
            return out, q
        L = int.from_bytes(j2c[q + 2:q + 4], "big")
        out.append((m, q, L + 2))
        q += L + 2


def _sots(j2c):
    _, q = _segments(j2c)
    out = []
    while int.from_bytes(j2c[q:q + 2], "big") == 0xFF90:
        psot = int.from_bytes(j2c[q + 6:q + 10], "big")
        out.append((q, psot))
        q += psot
    return out


def _headers(t, j2c):
    buf = np.frombuffer(bytes(j2c), np.uint8)
    return t.L.ojb_enc_transcode_headers(t.h, buf.ctypes.data, buf.size, 0, cs.I32), t.L.ojb_last_error().decode()


def _refusals(L):
    p = cases.make(dict(CPU_CONFIGS[10][1]))                # tiles, tile-parts by resolution, TLM
    good = cs.Encoder(p, lib=L).encode(cases.frame_for(p))
    t = cs.Encoder.from_codestream(good, lib=L)
    segs, sot = _segments(good)
    bad = {}
    cod = [s for s in segs if s[0] == 0xFF52][0]
    for bit in (2, 4):                                       # SOP, EPH
        b = bytearray(good)
        b[cod[1] + 4] |= bit
        bad.setdefault("0x000B004C", []).append(bytes(b))
    poc = b"\xff\x5f" + (2 + 7).to_bytes(2, "big") + bytes([0, 0, 0, 1, 4, 3, 0])
    bad["0x000B004D"] = [good[:sot] + poc + good[sot:]]
    q, psot = _sots(good)[0]
    com = b"\xff\x64\x00\x06\x00\x01AB"
    b = bytearray(good[:q + 12] + com + good[q + 12:])
    b[q + 6:q + 10] = (psot + len(com)).to_bytes(4, "big")
    bad["0x000B004E"] = [bytes(b)]
    # tile-parts 1 and 2 of the first tile merged: a division that matches none of the four
    (q0, _), (q1, p1), (q2, p2) = _sots(good)[:3]
    b = bytearray(good[:q2] + good[q2 + 14:])
    b[q1 + 6:q1 + 10] = (p1 + p2 - 14).to_bytes(4, "big")
    for q, _ in _sots(bytes(b)):
        if int.from_bytes(b[q + 4:q + 6], "big") == 0 and b[q + 10] > 2:
            b[q + 10] -= 1
    for q, _ in _sots(bytes(b)):
        if int.from_bytes(b[q + 4:q + 6], "big") == 0:
            b[q + 11] -= 1
    bad["0x000B004F"] = [bytes(b)]
    pw = cs.make_params(64, 64, 3, 32, num_decomps=5, reversible=True, color_transform=True)
    bad["0x000B0050"] = [cs.Encoder(pw, lib=L).encode(cases.frame_for(pw))]
    bad["0x000B0051"] = [good[:len(good) * 2 // 3], good[:_sots(good)[1][0] + 40]]
    for code, streams in bad.items():
        for s in streams:
            rc, msg = _headers(t, s)
            assert rc != 0 and code in msg, (code, msg)
            assert _headers(t, good)[0] == 0 and t.transcode(good) == good, code
            # refused by the frame call as well, which leaves the configuration as it was
            with pytest.raises(cs.OjphError, match=code):
                t.transcode(s)
            assert t.transcode(good) == good, code
    # the call order: a transcode before the headers call, and on an encoder configured for pixels
    fresh = cs.Encoder.__new__(cs.Encoder)
    cs._Base.__init__(fresh, L)
    fresh.h = L.ojb_enc_create()
    buf = np.frombuffer(good, np.uint8)
    n = C.c_uint64()
    out = np.empty(len(good) * 2, np.uint8)
    assert L.ojb_enc_transcode(fresh.h, buf.ctypes.data, buf.size, 0, out.ctypes.data, out.size, C.byref(n), 0) != 0
    assert "0x000B0052" in L.ojb_last_error().decode()
    assert _headers(fresh, good)[0] == 0
    assert L.ojb_enc_transcode(fresh.h, buf.ctypes.data, buf.size, 0, out.ctypes.data, out.size, C.byref(n), 0) == 0
    assert out[:n.value].tobytes() == good
    fresh.close()
    e = cs.Encoder(p, lib=L)
    with pytest.raises(cs.OjphError, match="0x000B0052"):
        e.transcode(good)
    # a transcoder has no image
    with pytest.raises(cs.OjphError, match="0x000B0053"):
        t.encode(cases.frame_for(p))
    assert t.transcode(good) == good


def test_refusals_emulator(emu_lib):
    _refusals(emu_lib)


# ---- on the H100 -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", CPU_CONFIGS, ids=[c[0] for c in CPU_CONFIGS])
def test_identity_gpu_small(gpu_lib, name, kw):
    _identity(gpu_lib, kw)


def _tensor_identity(L, kw):
    import torch
    p, frame, want = _identity(L, kw)
    t = cs.Encoder.from_codestream(torch.from_numpy(np.frombuffer(want, np.uint8).copy()).cuda(), lib=L)
    src = torch.from_numpy(np.frombuffer(want, np.uint8).copy()).cuda()
    got = t.transcode(src)
    assert got.is_cuda and got.cpu().numpy().tobytes() == want
    out = torch.zeros(len(want) + 64, dtype=torch.uint8, device="cuda")
    n = t.transcode(src, out=out)
    assert out[:n].cpu().numpy().tobytes() == want
    return p, frame, want


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", GPU_CONFIGS, ids=[c[0] for c in GPU_CONFIGS])
def test_identity_gpu_large(gpu_lib, name, kw):
    _tensor_identity(gpu_lib, kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", REV_CONFIGS, ids=[c[0] for c in REV_CONFIGS])
def test_lossless_targets_gpu_small(gpu_lib, name, kw):
    _lossless_targets(gpu_lib, kw)


@pytest.mark.gpu
def test_lossless_targets_gpu_hd(gpu_lib):
    _lossless_targets(gpu_lib, dict(GPU_CONFIGS[0][1]), fractions=(0.02, 0.25), mse_fracs=(0.05,), rate_tables=False)


@pytest.mark.gpu
def test_variants_gpu(gpu_lib):
    for env in ({"OJB_NO_FAST_BLOCKS": "1"}, {"OJB_BLOCK_ENCODER": "warp"}):
        a, b = _variant_sha("gpu", env, dict(GPU_CONFIGS[0][1]), 0.1)
        assert a == b, env


@pytest.mark.gpu
def test_lossy_inputs_gpu(gpu_lib, ref):
    _lossy_inputs(gpu_lib, ref, dict(CPU_CONFIGS[5][1]), dict(CPU_CONFIGS[0][1]))


@pytest.mark.gpu
def test_lossy_inputs_gpu_large(gpu_lib, ref):
    _lossy_inputs(gpu_lib, ref, dict(GPU_CONFIGS[1][1]), dict(GPU_CONFIGS[0][1]), fractions=(0.25,), mse_fracs=(0.2,))


@pytest.mark.gpu
def test_foreign_input_gpu(gpu_lib, ref):
    _foreign(gpu_lib, ref)


@pytest.mark.gpu
def test_refusals_gpu(gpu_lib):
    _refusals(gpu_lib)


@pytest.mark.gpu
def test_8k_targets_tensors_gpu(gpu_lib):
    """the 8K 12-bit 5/3 + RCT frame: three size targets and three PSNR targets, transcoded through CUDA tensors, are the
    pixel encoder's streams byte for byte"""
    import torch
    L = gpu_lib
    p = cases.make(dict(GPU_CONFIGS[2][1]))
    frame = cases.frame_for(p)
    full = cs.Encoder(p, lib=L).encode(frame)
    src = torch.from_numpy(np.frombuffer(full, np.uint8).copy()).cuda()
    t = cs.Encoder.from_codestream(src, lib=L)
    e = cs.Encoder(p, lib=L)
    for f in (1 / 4, 1 / 16, 1 / 64):
        T = int(len(full) * f)
        t.set_target_size(T)
        e.set_target_size(T)
        assert t.transcode(src).cpu().numpy().tobytes() == e.encode(frame), f
    t.set_target_size(0)
    for db in (40.0, 45.0, 50.0):
        a = cs.Encoder(p, lib=L, target_psnr=db)
        b = cs.Encoder.from_codestream(src, lib=L, target_psnr=db)
        assert b.transcode(src).cpu().numpy().tobytes() == a.encode(frame), db
        assert a.quality_info()["sse"] == b.quality_info()["sse"]
