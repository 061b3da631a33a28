"""stage-level parity of the CUDA path against the oracle restatement (oracle/ojph_oracle.c): the
quantised sub-band planes the block coder reads, and batches of code-blocks through the C-ABI's
fine boundary.  Runs under the emulator on the CPU tier and on the real GPU with -m gpu."""
import numpy as np
import pytest
import cases
import oracleport as O
import openjph_b200 as ob

STAGE_CASES = [
    ("rev_rct", dict(width=150, height=99, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, color_transform=True)),
    ("rev_off", dict(width=131, height=70, num_comps=1, bit_depth=12, num_decomps=4, reversible=True, offset=(3, 1))),
    ("irv_ict", dict(width=150, height=99, num_comps=3, bit_depth=10, num_decomps=3, reversible=False, color_transform=True, qstep=0.002)),
]


def _bands_vs_port(lib, name):
    kw = dict(STAGE_CASES)[name]
    p = cases.make(kw)
    frame = cases.frame_for(p)
    enc = ob.Encoder(p, ob.I32, lib=lib)
    enc.encode(frame)
    D = p.num_decomps
    info = {(c, r, b): enc.band_info(0, c, r, b) for c in range(p.num_comps) for r in range(D + 1)
            for b in ((0,) if r == 0 else (1, 2, 3))}
    layout = {"origin": lambda c: (info[(c, D, 1)]["res_x0"], info[(c, D, 1)]["res_y0"]),
              "quant": lambda c, r, b: (info[(c, r, b)]["K_max"], info[(c, r, b)]["delta_inv"])}
    want = O.forward_bands(p, frame, layout)
    worst = 0
    for key, w in want.items():
        got = enc.read_band(0, *key)
        assert got.shape == w.shape, key
        if p.reversible:
            assert np.array_equal(got, w), key
        else:   # float path: quantiser inputs may differ in the last ulp -> magnitudes within 1 code
            d = np.abs((got & 0x7FFFFFFF).astype(np.int64) - (w & 0x7FFFFFFF).astype(np.int64))
            worst = max(worst, int(d.max()) if d.size else 0)
            assert d.max() <= 64 if d.size else True, key     # far below the coded LSB (bit 31-K_max)
    return worst


@pytest.mark.parametrize("name", [n for n, _ in STAGE_CASES])
def test_subband_planes_match_port_emulated(name, emu_lib):
    _bands_vs_port(emu_lib, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n, _ in STAGE_CASES])
def test_subband_planes_match_port_gpu(name, gpu_lib):
    _bands_vs_port(None, name)


def _blocks_vs_port(lib, n, seed):
    rng = np.random.default_rng(seed)
    bufs, descs, want, off = [], [], [], 0
    coded, geoms, wdec = [], [], []
    for it in range(n):
        w = int(rng.integers(1, 65)); h = int(rng.integers(1, min(64, 4096 // w) + 1))
        kmax = int(rng.integers(2, 28))
        mag = np.minimum(np.abs(rng.laplace(0, 2 ** (kmax / 2.5), (h, w))).astype(np.uint64), (1 << kmax) - 1)
        if it % 4 == 0: mag = rng.integers(0, 1 << kmax, (h, w), dtype=np.uint64)
        blk = ((rng.integers(0, 2, (h, w), dtype=np.uint64) << 31) | (mag << (31 - kmax))).astype(np.uint32)
        stride = (w + 15) & ~15
        buf = np.zeros((h, stride), np.uint32); buf[:, :w] = blk
        bufs.append(buf.ravel()); descs.append((off, stride, w, h, kmax - 1)); off += buf.size
        data = O.encode_block(blk, kmax - 1) if mag.any() else b""
        want.append(data)
        if data:
            coded.append((data, len(data), 0, kmax - 1, 1)); geoms.append((w, h))
            wdec.append(O.decode_block(data, w, h, kmax - 1, 1, len(data), 0)[0])
    got = ob.encode_blocks(np.concatenate(bufs), descs, lib=lib)
    for i, (g, w_) in enumerate(zip(got, want)):
        assert g == w_, (i, descs[i])
    dec = ob.decode_blocks(coded, geoms, lib=lib)
    for i, ((a, ok), b) in enumerate(zip(dec, wdec)):
        assert ok and np.array_equal(a, b), (i, geoms[i])


def test_blocks_match_port_emulated(emu_lib):
    _blocks_vs_port(emu_lib, 40, 21)


@pytest.mark.gpu
def test_blocks_match_port_gpu(gpu_lib):
    _blocks_vs_port(None, 500, 22)


def _multipass_golden(lib, causal=False):
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ht_multipass_blocks.npz"))
    coded, geoms, want = [], [], []
    for i in range(int(z["n"])):
        w, h, mm, npass, l1, l2, ok_ref = [int(v) for v in z["meta_%d" % i]]
        coded.append((z["data_%d" % i].tobytes(), l1, l2, mm, npass)); geoms.append((w, h))
        want.append(z["wantc_%d" % i] if causal else z["want_%d" % i])
    got = ob.decode_blocks(coded, geoms, lib=lib, causal=causal)
    ndiff = 0
    for i, ((a, ok), b) in enumerate(zip(got, want)):
        assert ok and np.array_equal(a, b), i
        ndiff += int(causal and not np.array_equal(b, z["want_%d" % i]))
    if causal:
        assert ndiff > 0, "the causal goldens do not exercise the causal rule"


def test_sigprop_magref_golden_emulated(emu_lib):
    _multipass_golden(emu_lib)


@pytest.mark.gpu
def test_sigprop_magref_golden_gpu(gpu_lib):
    _multipass_golden(None)


def test_sigprop_stripe_causal_golden_emulated(emu_lib):
    """stripe_causal = true: the bytes of test.j2c's blocks decoded as the reference decodes them when told so"""
    _multipass_golden(emu_lib, causal=True)


@pytest.mark.gpu
def test_sigprop_stripe_causal_golden_gpu(gpu_lib):
    _multipass_golden(None, causal=True)


def _whole_multipass_stream(lib):
    """the reference's in-tree subprojects/js/html/test.j2c (9/7, 77 of 89 coded blocks with SPP / MRP passes) decoded
    as a whole codestream, against what the reference's ojph::codestream (= ojph_expand) produces from it; then the
    same stream with the vertically-causal COD bit set"""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "test_j2c.npz"))
    for cs_key, dec_key in (("cs", "dec"), ("cs_causal", "decc")):
        out = ob.Decoder(lib=lib).decode(z[cs_key].tobytes())
        assert len(out) == 3
        for c in range(3):
            want = z["%s%d" % (dec_key, c)].astype(np.int32)
            assert out[c].shape == want.shape
            assert np.abs(out[c] - want).max() <= 1, (cs_key, c)          # 9/7: the reference tests' peak-error tolerance
            assert np.mean(out[c] != want) < 0.01, (cs_key, c)
    assert int(z["differs"]) == 1


def test_whole_multipass_stream_emulated(emu_lib):
    _whole_multipass_stream(emu_lib)


@pytest.mark.gpu
def test_whole_multipass_stream_gpu(gpu_lib):
    _whole_multipass_stream(None)


def _codestream_goldens(lib):
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "codestreams.npz"))
    allc = dict(cases.SMALL_REV + cases.SMALL_IRV)
    names = sorted({k.rsplit("_cs", 1)[0] for k in z.files if k.endswith("_cs")})
    for nme in names:
        p = cases.make(allc[nme])
        frame = [z["%s_in%d" % (nme, c)] for c in range(p.num_comps)]
        want = z["%s_cs" % nme].tobytes()
        out = ob.Decoder(lib=lib).decode(want)
        if p.reversible:
            assert ob.Encoder(p, ob.I32, lib=lib).encode(frame) == want, nme
            for c in range(p.num_comps):
                assert np.array_equal(out[c], z["%s_dec%d" % (nme, c)]), nme
        else:
            cases.assert_irv_matches_reference(out, [z["%s_dec%d" % (nme, c)] for c in range(p.num_comps)], nme)


def test_codestream_goldens_emulated(emu_lib):
    _codestream_goldens(emu_lib)


@pytest.mark.gpu
def test_codestream_goldens_gpu(gpu_lib):
    _codestream_goldens(None)
