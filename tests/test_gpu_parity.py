"""GPU tier (-m gpu): the product library on a real H100 against the unmodified reference
(oracle/_ref travels with the snapshot) -- bit-exact for 5/3 codestreams and samples, MSE/PAE
tolerance of the reference's own tests for 9/7 -- plus size-independent properties at
BASELINE.json's full sizes."""
import numpy as np
import pytest
import cases
import images
import openjph_b200 as ob

pytestmark = pytest.mark.gpu
REV = {n: k for n, k in cases.SMALL_REV}
IRV = {n: k for n, k in cases.SMALL_IRV}


@pytest.mark.parametrize("name", [n for n, _ in cases.SMALL_REV])
def test_rev_codestream_identical_and_decodes(name, gpu_lib, ref):
    p = cases.make(REV[name])
    frame = cases.frame_for(p, "noise" if "noise" in name else "synth")
    want = ref.encode(p, frame)
    got = ob.Encoder(p, ob.I32).encode(frame)
    assert got == want, "codestream differs from the reference's (%d vs %d bytes)" % (len(got), len(want))
    ref_planes, _ = ref.decode(want)
    out = ob.Decoder().decode(want)
    for a, b in zip(out, ref_planes):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("name", [n for n, _ in cases.SMALL_IRV])
def test_irv_within_tolerance(name, gpu_lib, ref):
    p = cases.make(IRV[name])
    frame = cases.frame_for(p)
    want = ref.encode(p, frame)
    ref_planes, _ = ref.decode(want)
    out = ob.Decoder().decode(want)
    got = ob.Encoder(p, ob.I32).encode(frame)
    cross, _ = ref.decode(got)
    cases.assert_irv_matches_reference(out, ref_planes, name)
    for c in range(p.num_comps):
        m_ref, p_ref = cases.mse_pae(ref_planes[c], frame[c])
        for planes in (out, cross):
            m, pa = cases.mse_pae(planes[c], frame[c])
            assert abs(m - m_ref) / (m_ref + 0.01) < 0.01      # TOL_DOUBLE, tests/test_executables.cpp:132
            assert abs(pa - p_ref) <= 1                        # TOL_INTEGER :133


def test_line_interface_matches_frame_interface(gpu_lib, ref):
    p = cases.make(REV["rgb_rct_L3"])
    frame = cases.frame_for(p)
    enc = ob.Encoder(p, ob.I32)
    want = ref.encode(p, frame)
    assert enc.encode_lines(frame) == want
    planes, order = ob.Decoder().pull_lines(want)             # create() + pull() loop
    for a, b in zip(planes, frame):
        assert np.array_equal(a, b)
    assert order[:6] == [0, 1, 2, 0, 1, 2]                    # colour transform => interleaved default


def _random_blocks(rng, n, kmax_lo=1):
    bufs, descs, blks, off = [], [], [], 0
    for it in range(n):
        w = int(rng.integers(1, 65)); h = int(rng.integers(1, min(64, 4096 // w) + 1))
        if it % 3 == 0: w, h = 64, 64
        kmax = int(rng.integers(kmax_lo, 28))
        mode = it % 5
        if mode == 0: mag = rng.integers(0, 1 << kmax, (h, w), dtype=np.uint64)
        elif mode == 1: mag = np.full((h, w), (1 << kmax) - 1, dtype=np.uint64)
        elif mode == 2: mag = (rng.random((h, w)) < 0.03) * rng.integers(0, 1 << kmax, (h, w), dtype=np.uint64)
        elif mode == 3: mag = np.minimum(np.abs(rng.laplace(0, 2 ** (kmax / 3), (h, w))).astype(np.uint64), (1 << kmax) - 1)
        else: mag = np.zeros((h, w), np.uint64)
        sign = rng.integers(0, 2, (h, w), dtype=np.uint64)
        blk = ((sign << 31) | (mag << (31 - kmax))).astype(np.uint32)
        stride = (w + 15) & ~15
        buf = np.zeros((h, stride), np.uint32); buf[:, :w] = blk
        bufs.append(buf.ravel()); descs.append((off, stride, w, h, kmax - 1)); off += buf.size
        blks.append((blk, kmax, bool(mag.any())))
    return np.concatenate(bufs), descs, blks


def test_block_encoder_matches_reference(gpu_lib, ref):
    samples, descs, blks = _random_blocks(np.random.default_rng(11), 600)
    got = ob.encode_blocks(samples, descs)
    for i, ((blk, kmax, any_sig), g) in enumerate(zip(blks, got)):
        want = ref.encode_block(blk, kmax - 1) if any_sig else b""
        assert g == want, "block %d %s" % (i, descs[i])
        if any_sig and i % 7 == 0:      # the dispatched SIMD encoder agrees with the scalar one
            assert ref.encode_block(blk, kmax - 1, variant=1) == want


def test_block_decoder_matches_reference(gpu_lib, ref):
    samples, descs, blks = _random_blocks(np.random.default_rng(13), 400, kmax_lo=2)
    coded, geoms, want = [], [], []
    for (blk, kmax, any_sig), d in zip(blks, descs):
        if not any_sig: continue
        data = ref.encode_block(blk, kmax - 1)
        coded.append((data, len(data), 0, kmax - 1, 1)); geoms.append((d[2], d[3]))
        want.append(ref.decode_block(data, d[2], d[3], kmax - 1, 1, len(data), 0)[0])
    got = ob.decode_blocks(coded, geoms)
    for i, ((a, ok), b) in enumerate(zip(got, want)):
        assert ok and np.array_equal(a, b), "block %d %s" % (i, geoms[i])


def test_cfg2_1080p_rgb8(gpu_lib, ref):
    p = ob.make_params(1920, 1080, 3, 8, num_decomps=5, reversible=True, color_transform=True)
    frame = images.synth_frame(1920, 1080, 3, 8, 1234)
    want = ref.encode(p, frame)
    got = ob.Encoder(p, ob.U8).encode([f.astype(np.uint8) for f in frame])
    assert got == want
    out = ob.Decoder().decode(want, ob.U8)
    for a, b in zip(out, frame):
        assert np.array_equal(a.astype(np.int32), b)


def test_cfg3_4k_12bit_irv_q90(gpu_lib, ref):
    p = ob.make_params(4096, 4096, 3, 12, num_decomps=6, reversible=False, color_transform=True, qfactor=90)
    frame = images.synth_frame(4096, 4096, 3, 12, 1234)
    want = ref.encode(p, frame)
    ref_planes, _ = ref.decode(want)
    got = ob.Encoder(p, ob.U16).encode([f.astype(np.uint16) for f in frame])
    out = ob.Decoder().decode(want, ob.U16)
    cross, _ = ref.decode(got)
    cases.assert_irv_matches_reference(out, ref_planes, "cfg3")
    assert abs(len(got) - len(want)) <= len(want) // 1000 + 16
    for c in range(3):
        m_ref, p_ref = cases.mse_pae(ref_planes[c], frame[c])
        for planes in (out, cross):
            m, pa = cases.mse_pae(planes[c].astype(np.int32), frame[c])
            assert abs(m - m_ref) / (m_ref + 0.01) < 0.01
            assert abs(pa - p_ref) <= 1


def test_cfg4_8k_16bit_four_tiles(gpu_lib, ref):
    p = ob.make_params(8192, 8192, 3, 16, num_decomps=5, reversible=True, color_transform=True, tile=(4096, 4096))
    frame = images.synth_frame(8192, 8192, 3, 16, 77)
    got = ob.Encoder(p, ob.U16).encode([f.astype(np.uint16) for f in frame])
    want = ref.encode(p, frame)
    assert got == want
    out = ob.Decoder().decode(got, ob.U16)
    for a, b in zip(out, frame):
        assert np.array_equal(a.astype(np.int32), b)


def test_headline_8k_12bit_roundtrip_and_identity(gpu_lib, ref):
    p = ob.make_params(8192, 8192, 3, 12, num_decomps=5, reversible=True, color_transform=True)
    frame = images.synth_frame(8192, 8192, 3, 12, 1234)
    enc = ob.Encoder(p, ob.U16)
    got = enc.encode([f.astype(np.uint16) for f in frame])
    out = ob.Decoder().decode(got, ob.U16)
    for a, b in zip(out, frame):
        assert np.array_equal(a.astype(np.int32), b)          # encode -> decode is the identity
    assert enc.encode([f.astype(np.uint16) for f in frame]) == got   # idempotent across calls
    want = ref.encode(p, frame)
    assert got == want


def test_cfg5_4k_10bit_irv_frame(gpu_lib, ref):
    p = ob.make_params(3840, 2160, 3, 10, num_decomps=5, reversible=False, color_transform=True)
    frame = images.synth_frame(3840, 2160, 3, 10, 1300)
    want = ref.encode(p, frame)
    ref_planes, _ = ref.decode(want)
    out = ob.Decoder().decode(want, ob.U16)
    got = ob.Encoder(p, ob.U16).encode([f.astype(np.uint16) for f in frame])
    cross, _ = ref.decode(got)
    cases.assert_irv_matches_reference(out, ref_planes, "cfg5")
    for c in range(3):
        m_ref, p_ref = cases.mse_pae(ref_planes[c], frame[c])
        for planes in (out, cross):
            m, pa = cases.mse_pae(planes[c].astype(np.int32), frame[c])
            assert abs(m - m_ref) / (m_ref + 0.01) < 0.01
            assert abs(pa - p_ref) <= 1


def test_errors_are_reported_not_swallowed(gpu_lib):
    with pytest.raises(ob.OjphError):
        ob.Encoder(ob.make_params(64, 64, 2, 8, color_transform=True, reversible=True), ob.I32)   # < 3 comps
    with pytest.raises(ob.OjphError):
        ob.Decoder().decode(b"\xff\x4f\xff\x51" + b"\0" * 64)


@pytest.mark.gpu
def test_alternate_block_coder_variants_gpu(gpu_lib, ref):
    """warp-per-block encoder (non-default) on the device"""
    import os, subprocess, sys
    if os.environ.get("OJB_VARIANT_CHILD"):
        pytest.skip("already inside the child run")
    env = dict(os.environ, OJB_BLOCK_ENCODER="warp", OJB_VARIANT_CHILD="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "-m", "gpu", "--timeout", "600",
                        "-k", "block_encoder or block_decoder or cfg2 or cfg3 or odd_rgb_L5 or offsets"],
                       env=env, capture_output=True, text=True, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.gpu
def test_frame_beyond_32bit_offsets_gpu(gpu_lib, ref):
    """20480 x 20480 x 3: the coefficient arena has more than 2^30 words, so the streaming DWT kernels (32-bit
    offsets) are not eligible and the general kernels take over; lossless round trip, and the codestream is the
    one the reference produces for the same frame (about 20 s of one host core)"""
    w = h = 20480
    rng = np.random.default_rng(3)
    small = rng.integers(0, 256, (h // 16, w // 16), dtype=np.uint8)
    planes = []
    for c in range(3):
        a = small.repeat(16, axis=0).repeat(16, axis=1)
        a[::3, ::5] += np.uint8(c + 1)
        planes.append(a)
    p = ob.make_params(w, h, 3, 8, num_decomps=5, reversible=True, color_transform=True)
    cs = ob.Encoder(p, ob.U8).encode(planes)
    out = ob.Decoder().decode(cs, ob.U8)
    for a, b in zip(out, planes):
        assert np.array_equal(a, b)
    del out
    want = ref.encode(p, planes)
    assert len(want) == len(cs) and want == cs
