"""CPU tier: the product's kernel sources compiled under the SIMT emulator (tests/emu) against the
unmodified reference (oracle/_ref).  Checks kernel LOGIC without a GPU; the same cases run on a
real H100 in test_gpu_parity.py."""
import numpy as np
import pytest
import cases
import openjph_b200 as ob

REV = {n: k for n, k in cases.SMALL_REV}
IRV = {n: k for n, k in cases.SMALL_IRV}


@pytest.mark.parametrize("name", cases.EMU_REV)
def test_rev_codestream_identical_and_decodes(name, emu_lib, ref):
    p = cases.make(REV[name])
    frame = cases.frame_for(p, "noise" if "noise" in name else "synth")
    want = ref.encode(p, frame)
    enc = ob.Encoder(p, ob.I32, lib=emu_lib)
    got = enc.encode(frame)
    assert got == want, "codestream differs from the reference's (%d vs %d bytes)" % (len(got), len(want))
    ref_planes, _ = ref.decode(want)
    out = ob.Decoder(lib=emu_lib).decode(want)
    for a, b in zip(out, ref_planes):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("name", cases.EMU_IRV)
def test_irv_within_tolerance(name, emu_lib, ref):
    p = cases.make(IRV[name])
    frame = cases.frame_for(p)
    want = ref.encode(p, frame)
    ref_planes, _ = ref.decode(want)
    out = ob.Decoder(lib=emu_lib).decode(want)
    got = ob.Encoder(p, ob.I32, lib=emu_lib).encode(frame)
    cross, _ = ref.decode(got)
    cases.assert_irv_matches_reference(out, ref_planes, name)
    for c in range(p.num_comps):
        m_ref, p_ref = cases.mse_pae(ref_planes[c], frame[c])
        for planes in (out, cross):
            m, pa = cases.mse_pae(planes[c], frame[c])
            # tolerances of the reference's own tests (tests/test_executables.cpp:132-133,215,225)
            assert abs(m - m_ref) / (m_ref + 0.01) < 0.01
            assert abs(pa - p_ref) <= 1


def test_block_encoder_random_blocks(emu_lib, ref):
    rng = np.random.default_rng(3)
    bufs, descs, want, off = [], [], [], 0
    for it in range(100):
        w = int(rng.integers(1, 65)); h = int(rng.integers(1, min(64, 4096 // w) + 1))
        kmax = int(rng.integers(1, 28))
        mode = it % 5
        if mode == 0: mag = rng.integers(0, 1 << kmax, (h, w), dtype=np.uint64)
        elif mode == 1: mag = np.full((h, w), (1 << kmax) - 1, dtype=np.uint64)       # 0xFF-heavy: exercises stuffing
        elif mode == 2: mag = (rng.random((h, w)) < 0.03) * rng.integers(0, 1 << kmax, (h, w), dtype=np.uint64)
        elif mode == 3: mag = np.minimum(np.abs(rng.laplace(0, 2 ** (kmax / 3), (h, w))).astype(np.uint64), (1 << kmax) - 1)
        else: mag = np.uint64(1) << rng.integers(0, kmax, (h, w), dtype=np.uint64)    # negative powers of two: MagSgn fields of ones
        sign = rng.integers(0, 2, (h, w), dtype=np.uint64) if mode != 4 else np.ones((h, w), np.uint64)
        blk = ((sign << 31) | (mag << (31 - kmax))).astype(np.uint32)
        stride = (w + 15) & ~15
        buf = np.zeros((h, stride), np.uint32); buf[:, :w] = blk
        bufs.append(buf.ravel()); descs.append((off, stride, w, h, kmax - 1)); off += buf.size
        want.append(ref.encode_block(blk, kmax - 1) if mag.any() else b"")
    got = ob.encode_blocks(np.concatenate(bufs), descs, lib=emu_lib)
    for i, (g, w_) in enumerate(zip(got, want)):
        assert g == w_, "block %d %s" % (i, descs[i])


def test_block_decoder_matches_reference(emu_lib, ref):
    rng = np.random.default_rng(5)
    coded, geoms, want = [], [], []
    for it in range(40):
        w = int(rng.integers(1, 65)); h = int(rng.integers(1, min(64, 4096 // w) + 1))
        kmax = int(rng.integers(2, 28))
        mag = np.minimum(np.abs(rng.laplace(0, 2 ** (kmax / 2.5), (h, w))).astype(np.uint64), (1 << kmax) - 1)
        if it % 5 == 0: mag = rng.integers(0, 1 << kmax, (h, w), dtype=np.uint64)
        sign = rng.integers(0, 2, (h, w), dtype=np.uint64)
        blk = ((sign << 31) | (mag << (31 - kmax))).astype(np.uint32)
        if not mag.any(): continue
        data = ref.encode_block(blk, kmax - 1)
        coded.append((data, len(data), 0, kmax - 1, 1)); geoms.append((w, h))
        want.append(ref.decode_block(data, w, h, kmax - 1, 1, len(data), 0)[0])
    got = ob.decode_blocks(coded, geoms, lib=emu_lib)
    for i, ((a, ok), b) in enumerate(zip(got, want)):
        assert ok and np.array_equal(a, b), "block %d %s" % (i, geoms[i])


@pytest.mark.parametrize("name,planar", [("odd_rgb_L5", None), ("odd_rgb_L5", True), ("sub420_planar", True)])
def test_line_interface_exchange_and_pull(name, planar, emu_lib, ref):
    """exchange()/flush() on the write side and create()/pull() on the read side give the frame-at-once
    results, in the reference's line order (ojph_codestream_local.cpp:1176-1224, :1227-1272)"""
    p = cases.make(REV[name])
    frame = cases.frame_for(p)
    want = ref.encode(p, frame)
    assert ob.Encoder(p, ob.I32, lib=emu_lib).encode_lines(frame) == want
    planes, order = ob.Decoder(lib=emu_lib).pull_lines(want, planar=planar)
    for a, b in zip(planes, frame):
        assert np.array_equal(a, b)
    nc = p.num_comps
    if planar or (planar is None and not p.color_transform):
        assert order == sorted(order)                     # component by component
    else:
        assert order[:2 * nc] == list(range(nc)) * 2      # row by row, component by component


def test_alternate_block_coder_variants(emu_lib, ref):
    """the non-default warp-per-block encoder is selected by an environment variable read once per process:
    run a subset of this file in a child process"""
    import os, subprocess, sys
    if os.environ.get("OJB_VARIANT_CHILD"):
        pytest.skip("already inside the child run")
    env = dict(os.environ, OJB_BLOCK_ENCODER="warp", OJB_VARIANT_CHILD="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-x", "-q", "--timeout", "600",
                        "-k", "cfg1_256 or odd_rgb_L5 or rgb16_noise or offsets or irv_tiles or block_"],
                       env=env, capture_output=True, text=True, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.parametrize("bd,ct", [(20, True), (24, False), (26, True), (27, True), (28, False)])
def test_high_bit_depths_on_the_32bit_path(bd, ct, emu_lib, ref):
    """the 32-bit coefficient path reaches 27-bit RGB with RCT (28-bit without): byte-identical and lossless"""
    rng = np.random.default_rng(bd)
    p = ob.make_params(96, 64, 3, bd, num_decomps=3, reversible=True, color_transform=ct, planar=0 if ct else 1)
    fr = [rng.integers(0, 1 << bd, (64, 96)).astype(np.int32) for _ in range(3)]
    want = ref.encode(p, fr)
    assert ob.Encoder(p, ob.I32, lib=emu_lib).encode(fr) == want
    for a, b in zip(ob.Decoder(lib=emu_lib).decode(want), fr):
        assert np.array_equal(a, b)


def test_beyond_the_32bit_path_runs_on_64bit_coefficients(emu_lib, ref):
    """28-bit RGB with RCT needs 33-bit coefficients: the reference switches to its 64-bit line buffers and block
    coders, and so does this build (byte-identical, lossless)"""
    rng = np.random.default_rng(1)
    p = ob.make_params(64, 48, 3, 28, num_decomps=3, reversible=True, color_transform=True)
    fr = [rng.integers(0, 1 << 28, (48, 64)).astype(np.int32) for _ in range(3)]
    cs = ref.encode(p, fr)
    assert ob.Encoder(p, ob.I32, lib=emu_lib).encode(fr) == cs
    for a, b in zip(ob.Decoder(lib=emu_lib).decode(cs), fr):
        assert np.array_equal(a, b)
