"""Seeded random parameter combinations against the reference (CPU tier, kernels under the emulator):
image size / offset, tile size / offset, component count, bit depth, signedness, sub-sampling,
decompositions, code-block size, precincts, progression order, tile-part divisions, TLM, colour
transform, per-component coding styles.  Reversible streams must be byte-identical and decode exactly;
irreversible ones must have the reference's length and decode to what the reference decodes."""
import numpy as np
import pytest
import cases
import openjph_b200 as ob

import os
# seeds of the default run; OJB_RANDOM_CASES="a:b" widens the hunt (1000 cases take ~40 s with -n 8)
_lo, _hi = (int(x) for x in os.environ.get("OJB_RANDOM_CASES", "0:120").split(":"))


def random_case(seed):
    rng = np.random.default_rng(1000 + seed)
    nc = int(rng.choice([1, 1, 3, 3, 4]))
    w, h = int(rng.integers(1, 150)), int(rng.integers(1, 120))
    ox, oy = (int(rng.integers(0, 9)), int(rng.integers(0, 9))) if rng.random() < 0.4 else (0, 0)
    kw = dict(width=w + ox, height=h + oy, num_comps=nc, offset=(ox, oy))
    kw["bit_depth"] = int(rng.choice([1, 4, 8, 10, 12, 16]))
    kw["is_signed"] = bool(rng.random() < 0.25)
    kw["num_decomps"] = int(rng.integers(0, 6))
    bw = int(rng.choice([4, 8, 16, 32, 64, 128]))
    bh = int(rng.choice([b for b in (4, 8, 16, 32, 64) if b * bw <= 4096]))
    kw["block"] = (bw, bh)
    kw["reversible"] = bool(rng.random() < 0.7)
    if not kw["reversible"]:
        kw["bit_depth"] = max(kw["bit_depth"], 4)
        kw["qstep"] = float(rng.choice([0.005, 0.02, 0.1]))
    kw["prog_order"] = str(rng.choice(["LRCP", "RLCP", "RPCL", "PCRL", "CPRL"]))
    if rng.random() < 0.4:
        tw, th = int(rng.integers(16, 100)), int(rng.integers(16, 100))
        tox, toy = (int(rng.integers(0, ox + 1)), int(rng.integers(0, oy + 1)))
        kw["tile"], kw["tile_offset"] = (tw, th), (tox, toy)
    if rng.random() < 0.3:
        kw["precincts"] = [(int(2 ** rng.integers(5, 9)), int(2 ** rng.integers(5, 9))) for _ in range(int(rng.integers(1, 4)))]
    sub = nc == 3 and rng.random() < 0.3
    if sub:
        kw["subsampling"] = [(1, 1), (2, int(rng.choice([1, 2]))), (2, int(rng.choice([1, 2])))]
        kw["planar"] = 1
    elif nc >= 3 and rng.random() < 0.6:
        kw["color_transform"] = True
    kw["tlm"] = bool(rng.random() < 0.3)
    kw["tilepart_div"] = int(rng.choice([0, 0, 1, 2, 3]))
    if nc >= 3 and not kw.get("color_transform") and rng.random() < 0.5:
        c = int(rng.integers(0, nc))
        kw["coc"] = {c: dict(reversible=bool(rng.random() < 0.5), num_decomps=int(rng.integers(0, 5)),
                             block=(int(rng.choice([16, 32, 64])), int(rng.choice([16, 32, 64]))))}
        kw["planar"] = 1
    # a separate stream for the later additions, so that the cases above stay what they were
    rng2 = np.random.default_rng(50000 + seed)
    if rng2.random() < 0.25:
        kw["nlt"] = {"all": 3} if rng2.random() < 0.5 else {int(rng2.integers(0, nc)): 3}
        if rng2.random() < 0.7:
            kw["is_signed"] = True
    if "coc" in kw and rng2.random() < 0.4:          # the component's own precinct sizes
        for st in kw["coc"].values():
            st["precincts"] = [(int(2 ** rng2.integers(5, 9)), int(2 ** rng2.integers(5, 9))) for _ in range(int(rng2.integers(1, 3)))]
    if not kw["reversible"] and rng2.random() < 0.25:  # per-component quantisation calls
        c = int(rng2.integers(0, nc))
        kw["qcc"] = [("qfactor", c, int(rng2.integers(0, 3)), int(rng2.integers(20, 100)))] if rng2.random() < 0.5 else [("qstep", c, float(rng2.choice([0.004, 0.03])))]
    return kw


def random_skip(seed, kw):
    """a (read, recon) pair for restrict_input_resolution, or None"""
    rng2 = np.random.default_rng(70000 + seed)
    dmin = min([kw["num_decomps"]] + [st.get("num_decomps", 5) for st in kw.get("coc", {}).values()])
    if dmin == 0 or rng2.random() < 0.5:
        return None
    read = int(rng2.integers(1, dmin + 1))
    return read, int(rng2.integers(0, read + 1))


@pytest.mark.parametrize("seed", range(_lo, _hi))
def test_random_configuration(seed, emu_lib, ref):
    _run_case(seed, emu_lib, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(0, 80))
def test_random_configuration_gpu(seed, gpu_lib, ref):
    _run_case(seed, None, ref)


def _run_case(seed, emu_lib, ref):
    kw = random_case(seed)
    p = cases.make(kw)
    frame = cases.frame_for(p, "noise" if seed % 3 == 0 else "synth", seed=seed)
    want = ref.encode(p, frame)
    got = ob.Encoder(p, ob.I32, lib=emu_lib).encode(frame)
    all_rev = kw["reversible"] and all(st.get("reversible", False) for st in kw.get("coc", {}).values())
    try:
        ref_planes, _ = ref.decode(want)
    except RuntimeError:
        # the reference cannot read back what it wrote (seen with tile-part divisions and components of
        # different decomposition counts): the drop-in must produce the same bytes and refuse them as well
        assert got == want or not all_rev, kw
        with pytest.raises(ob.OjphError):
            ob.Decoder(lib=emu_lib).decode(want)
        return
    dec = ob.Decoder(lib=emu_lib)
    skip = random_skip(seed, kw)
    if skip is not None:
        small, _ = ref.decode_restricted(want, *skip)
        ours = dec.decode(want, skip=skip)
        assert [a.shape for a in ours] == [b.shape for b in small], (kw, skip)
        for c, (a, b) in enumerate(zip(ours, small)):
            d = np.abs(a.astype(np.int64) - b)
            # reversible components are exact; 9/7 ones may differ by rounding ties (float associativity)
            rev_c = kw.get("coc", {}).get(c, kw).get("reversible", False)
            assert d.size == 0 or (d.max() <= (0 if rev_c else 1) and (rev_c or (d != 0).mean() < 0.02)), (kw, skip, c)
    out = dec.decode(want, skip=(0, 0))
    if all_rev:
        assert got == want, kw
        # (the reference itself is not lossless for every corner, e.g. full-range 16-bit data with zero
        # decompositions: the oracle's own decode is the yardstick, the frame only when the oracle returns it)
        for a, b in zip(out, ref_planes):
            assert np.array_equal(a, b), kw
    else:
        # 9/7 is float arithmetic: the reference's own ISA variants differ in the last bit (SURVEY fact 2), a
        # coefficient on a rounding boundary may flip one quantised value -> the stream length may differ by bytes
        assert abs(len(got) - len(want)) <= max(4, len(want) // 1000), kw
        cross, _ = ref.decode(got)
        cases.assert_irv_matches_reference(out, ref_planes, kw, list(p.bit_depth))
        for c in range(p.num_comps):
            m_ref, p_ref = cases.mse_pae(ref_planes[c], frame[c])
            for planes in (out, cross):
                # tolerances of the reference's own tests (tests/test_executables.cpp:132-133)
                m, pa = cases.mse_pae(planes[c], frame[c])
                # (plus an absolute floor: with very fine steps the MSE is ~0.08 and made of rounding ties, so a
                # handful of ties going the other way -- as between the reference's own ISA variants -- is
                # already more than 1 % of it; 0.01 means one sample in a hundred off by one level)
                slack = max(0.01 * m_ref, 0.01, 4.0 / planes[c].size)
                # (PAE: +-1, or 1 % when the quantisation step itself is hundreds of levels -- 16-bit data, coarse steps)
                assert abs(m - m_ref) <= slack and abs(pa - p_ref) <= max(1, 0.01 * p_ref), (kw, c, m, m_ref, pa, p_ref)
