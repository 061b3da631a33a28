"""shared parity cases: (name, kwargs for make_params, image kind)"""
# BASELINE.json configs: cfg1, cfg2 (1080p), cfg3 (4K 9/7 q90), cfg4 (8K 16-bit 4 tiles), cfg5 (4K 10-bit 9/7)
SMALL_REV = [
    ("cfg1_256_gray_L1", dict(width=256, height=256, num_comps=1, bit_depth=8, num_decomps=1, reversible=True)),
    ("gray_L0", dict(width=64, height=64, num_comps=1, bit_depth=8, num_decomps=0, reversible=True)),
    ("rgb_rct_L3", dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, color_transform=True)),
    ("odd_rgb_L5", dict(width=123, height=77, num_comps=3, bit_depth=8, num_decomps=5, reversible=True, color_transform=True)),
    ("tiles_128", dict(width=300, height=200, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, color_transform=True, tile=(128, 128))),
    ("offsets", dict(width=300, height=200, num_comps=1, bit_depth=8, num_decomps=3, reversible=True, tile=(128, 100), offset=(7, 5), tile_offset=(3, 2))),
    ("rgb16_noise", dict(width=160, height=120, num_comps=3, bit_depth=16, num_decomps=4, reversible=True, color_transform=True)),
    ("rgb12", dict(width=256, height=128, num_comps=3, bit_depth=12, num_decomps=5, reversible=True, color_transform=True)),
    ("block_32x32", dict(width=200, height=150, num_comps=1, bit_depth=8, num_decomps=2, reversible=True, block=(32, 32))),
    ("block_64x16", dict(width=200, height=150, num_comps=1, bit_depth=8, num_decomps=2, reversible=True, block=(64, 16))),
    ("block_4x4", dict(width=40, height=30, num_comps=1, bit_depth=8, num_decomps=1, reversible=True, block=(4, 4))),
    # wider than 64 samples: handled by the thread-per-block kernels
    ("block_128x32", dict(width=700, height=300, num_comps=3, bit_depth=10, num_decomps=3, reversible=True, color_transform=True, block=(128, 32))),
    ("block_1024x4", dict(width=1500, height=64, num_comps=1, bit_depth=8, num_decomps=2, reversible=True, block=(1024, 4))),
    ("block_256x16", dict(width=600, height=200, num_comps=1, bit_depth=12, num_decomps=2, reversible=True, block=(256, 16))),
    ("tlm_tiles", dict(width=300, height=200, num_comps=3, bit_depth=8, num_decomps=2, reversible=True, color_transform=True, tile=(128, 128), tlm=True)),
    ("sub420_planar", dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, subsampling=[(1, 1), (2, 2), (2, 2)], planar=1)),
    ("tilepart_R", dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, color_transform=True, tilepart_div=1, tlm=True)),
    ("tilepart_C_cprl", dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=3, reversible=True, prog_order="CPRL", tilepart_div=2, tlm=True)),
    ("tilepart_RC_lrcp", dict(width=200, height=150, num_comps=3, bit_depth=8, num_decomps=2, reversible=True, prog_order="LRCP", tilepart_div=3)),
    ("tiny_1x1", dict(width=1, height=1, num_comps=1, bit_depth=8, num_decomps=2, reversible=True)),
    ("thin_300x1", dict(width=300, height=1, num_comps=1, bit_depth=8, num_decomps=2, reversible=True)),
    ("thin_1x300", dict(width=1, height=300, num_comps=1, bit_depth=8, num_decomps=2, reversible=True)),
    ("thin_off", dict(width=3, height=6, num_comps=1, bit_depth=8, num_decomps=3, reversible=True, offset=(1, 1))),
    ("signed10", dict(width=100, height=80, num_comps=1, bit_depth=10, is_signed=True, num_decomps=3, reversible=True)),
    ("rgba_rct", dict(width=100, height=80, num_comps=4, bit_depth=8, num_decomps=3, reversible=True, color_transform=True)),
]
for _po in ("LRCP", "RLCP", "RPCL", "PCRL", "CPRL"):
    SMALL_REV.append(("po_%s_precincts" % _po, dict(width=300, height=260, num_comps=3, bit_depth=8, num_decomps=3,
                                                   reversible=True, color_transform=True, prog_order=_po,
                                                   precincts=[(128, 128), (64, 64)])))
SMALL_IRV = [
    ("irv_gray", dict(width=200, height=150, num_comps=1, bit_depth=8, num_decomps=3, reversible=False)),
    ("irv_rgb_q90", dict(width=256, height=200, num_comps=3, bit_depth=12, num_decomps=5, reversible=False, color_transform=True, qfactor=90)),
    ("irv_rgb_qstep", dict(width=123, height=77, num_comps=3, bit_depth=8, num_decomps=4, reversible=False, color_transform=True, qstep=0.01)),
    ("irv_tiles", dict(width=300, height=200, num_comps=3, bit_depth=10, num_decomps=3, reversible=False, color_transform=True, tile=(128, 128), qfactor=75)),
]
# a quick subset for the CPU (emulator) tier
EMU_REV = ["cfg1_256_gray_L1", "gray_L0", "odd_rgb_L5", "offsets", "rgb16_noise", "block_4x4", "block_128x32", "block_1024x4", "tilepart_RC_lrcp",
           "tiny_1x1", "thin_off", "signed10", "po_PCRL_precincts", "sub420_planar"]
EMU_IRV = ["irv_rgb_qstep", "irv_tiles"]


def make(case_kwargs):
    import openjph_b200 as ob
    kw = dict(case_kwargs)
    w, h, nc, bd = kw.pop("width"), kw.pop("height"), kw.pop("num_comps"), kw.pop("bit_depth")
    return ob.make_params(w, h, nc, bd, **kw)


def frame_for(p, kind="synth", seed=1234):
    import images
    from openjph_b200.codestream import comp_dims
    dims = comp_dims(p)
    bd = p.bit_depth[0]
    if kind == "noise":
        fr = [images.noise_frame(dw, dh, 1, bd, seed + c)[0] for c, (dw, dh) in enumerate(dims)]
    else:
        fr = images.synth_frame(p.width, p.height, p.num_comps, bd, seed, dims)
    if p.is_signed[0]:
        fr = [f - (1 << (bd - 1)) for f in fr]
    return fr


# 9/7: largest share of samples on which our decode of a codestream may differ (by one) from the reference's decode of
# the same codestream, for components of up to 12 bits.  The two differ only where a float32 result lies within
# rounding noise of a half (a tie, see tests/test_irv_precision.py); that noise is a fixed fraction of the normalised
# sample, so the tie band, in output levels, doubles with every bit of depth.  Up to 12 bits the CPU tier shows at most
# 0.03 % of samples, so 0.2 % leaves a margin of six; 16-bit components show up to 0.4 % against a bound of 3.2 %.
IRV_DIFF_FRACTION = 0.002


def assert_irv_matches_reference(ours, ref_planes, what="", bit_depths=None):
    """our decode against the reference's decode of the same codestream, sample by sample"""
    import numpy as np
    for c, (a, b) in enumerate(zip(ours, ref_planes)):
        d = np.abs(a.astype(np.int64) - b.astype(np.int64))
        assert a.shape == b.shape and (d.size == 0 or d.max() <= 1), (what, c)
        bound = IRV_DIFF_FRACTION * 2.0 ** max(0, (bit_depths[c] if bit_depths else 12) - 12)
        assert (d != 0).mean() <= bound if d.size else True, (what, c, float((d != 0).mean()))


def mse_pae(a, b):
    """per-component MSE (float) and peak absolute error (tests/mse_pae.cpp:522-567)"""
    import numpy as np
    d = a.astype(np.int64) - b.astype(np.int64)
    return float((d * d).mean()), int(np.abs(d).max())
