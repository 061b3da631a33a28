"""float64 model of the irreversible (9/7) path: sample conversion, ICT, 9/7 lifting with whole-sample symmetric
extension, de-interleave by absolute parity and quantiser input (forward); de-quantisation of cleanup-only block
output, synthesis and inverse ICT (inverse).  numpy only.  The operations are restated from the standard
(ITU-T T.800 Annex F and G.2-G.3) with the reference's float32 constants promoted to float64, so the model is what
the float32 kernels approximate; tests compare the kernels with it under `check_rounding`.

Test infrastructure only."""
import numpy as np

F32 = np.float32
# 9/7 lifting steps and K, as float32 values promoted to float64 (T.800 Table F.4; the reference's param_atk::init_irv97,
# src/core/codestream/ojph_params.cpp:2870-2881, and dwt_common.cuh hold the same float32 constants)
ALPHA = float(F32(-1.586134342059924))
BETA = float(F32(-0.052980118572961))
GAMMA = float(F32(0.882911075530934))
DELTA = float(F32(0.443506852043971))
STEPS = (ALPHA, BETA, GAMMA, DELTA)          # analysis order; step s updates odd positions for s = 0, 2, even for 1, 3
K = float(F32(1.230174104914001))
KINV = float(F32(1.0) / F32(1.230174104914001))   # the reference scales by 1.0f / K, a float32 quotient
# ICT (T.800 G.2; the reference's ojph_colour.cpp:220-230 float32 constants)
A_R, A_G, A_B = float(F32(0.299)), float(F32(0.587)), float(F32(0.114))
BETA_CB = float(F32(0.5 / (1.0 - A_B)))
BETA_CR = float(F32(0.5 / (1.0 - A_R)))
G_CB2G = float(F32(2.0 * A_B * (1.0 - A_B) / A_G))
G_CR2G = float(F32(2.0 * A_R * (1.0 - A_R) / A_G))
G_CB2B = float(F32(2.0 * (1.0 - A_B)))
G_CR2R = float(F32(2.0 * (1.0 - A_R)))
U32 = 2.0 ** -24          # unit round-off of float32 round-to-nearest


def _nbrs(n, start, parity):
    """indices of the positions of absolute parity `parity` on a line of n samples starting at absolute `start`,
    and of their left / right neighbours under whole-sample symmetric extension (x[-1] = x[1], x[n] = x[n-2])"""
    i = np.arange((parity - start) & 1, n)[::2]
    lft = np.abs(i - 1)
    rgt = i + 1
    rgt = np.where(rgt >= n, 2 * (n - 1) - rgt, rgt)
    return i, lft, rgt


def lift(x, start, forward):
    """one-dimensional 9/7 analysis (forward) or synthesis along axis 0 of x (float64, modified in place).  A line of
    one sample is not lifted: an odd-positioned sample is doubled (forward) or halved (inverse), as T.800 F.3.7 / F.4.8
    and the reference (irv_horz_ana / irv_vert: ojph_transform.cpp, ojph_resolution.cpp) do."""
    n = x.shape[0]
    if n == 0:
        return x
    if n == 1:
        if start & 1:
            x *= 2.0 if forward else 0.5
        return x
    odd = _nbrs(n, start, 1)
    even = _nbrs(n, start, 0)
    if forward:
        for s in range(4):
            i, l, r = odd if s % 2 == 0 else even
            x[i] += STEPS[s] * (x[l] + x[r])
        x[even[0]] *= KINV
        x[odd[0]] *= K
    else:
        x[even[0]] *= K
        x[odd[0]] *= KINV
        for s in (3, 2, 1, 0):
            i, l, r = odd if s % 2 == 0 else even
            x[i] -= STEPS[s] * (x[l] + x[r])
    return x


def to_float(a, bit_depth, signed):
    """sample -> normalised float: (v - 2^(B-1)) * 2^-B for unsigned samples, v * 2^-B for signed (exact in float64)"""
    half = 0 if signed else 1 << (bit_depth - 1)
    return (np.asarray(a, np.float64) - half) * 2.0 ** -bit_depth


def ict_fwd(r, g, b, comp):
    y = A_R * r + A_G * g + A_B * b
    return (y, BETA_CB * (b - y), BETA_CR * (r - y))[comp]


def ict_inv(y, cb, cr):
    return y + G_CR2R * cr, y - G_CR2G * cr - G_CB2G * cb, y + G_CB2B * cb


def _split(n, start):
    """(low, high) index arrays of a line of n samples starting at absolute `start`"""
    i = np.arange(n)
    return i[((start + i) & 1) == 0], i[((start + i) & 1) == 1]


def analyse(x, x0, y0, levels):
    """2-D analysis of a float64 plane at origin (x0, y0): per level vertical then horizontal lifting; returns
    ({(res, band): float64 coefficient plane}, [max |x| of each level's input]).  res counts as the codec does:
    levels is the finest resolution, 0 holds the final LL."""
    out, mags = {}, []
    cur = np.array(x, np.float64)
    for r in range(levels, 0, -1):
        mags.append(float(np.abs(cur).max()) if cur.size else 0.0)
        lift(cur, y0, True)
        lift(cur.T, x0, True)
        rows, cols = _split(cur.shape[0], y0), _split(cur.shape[1], x0)
        for b in (1, 2, 3):
            out[(r, b)] = cur[np.ix_(rows[b >> 1], cols[b & 1])]
        cur = cur[np.ix_(rows[0], cols[0])]
        x0, y0 = (x0 + 1) >> 1, (y0 + 1) >> 1
    out[(0, 0)] = cur
    return out, mags


def synthesise(bands, origins):
    """inverse of `analyse`: bands = {(res, band): float64 plane}, origins[r] = (x0, y0) of resolution r (r = 1..D);
    per level horizontal then vertical synthesis.  Returns the float64 plane of the finest resolution."""
    D = len(origins) - 1
    cur = bands[(0, 0)]
    for r in range(1, D + 1):
        x0, y0 = origins[r]
        hl, lh, hh = bands[(r, 1)], bands[(r, 2)], bands[(r, 3)]
        h = cur.shape[0] + lh.shape[0]
        w = cur.shape[1] + hl.shape[1]
        rows, cols = _split(h, y0), _split(w, x0)
        full = np.empty((h, w), np.float64)
        for b, a in ((0, cur), (1, hl), (2, lh), (3, hh)):
            full[np.ix_(rows[b >> 1], cols[b & 1])] = a
        lift(full.T, x0, False)
        lift(full, y0, False)
        cur = full
    return cur


def dequantise(words, K_max, delta):
    """what the block decoder hands the synthesis for a cleanup-only block, in float64: the coded magnitude bits
    (bits 30 .. 31-K_max of the quantiser's sign-magnitude word) with the half-LSB reconstruction bit below them set
    for every non-zero magnitude, times delta (the float32 value of band_info, 2^-(31-K_max) folded in)"""
    s = 31 - K_max
    mag = (words & np.uint32(0x7FFFFFFF)) >> np.uint32(s)
    rec = np.where(mag != 0, (mag.astype(np.uint64) << np.uint64(s)) | np.uint64(1 << (s - 1)), 0)
    f = rec.astype(np.float64) * float(delta)
    return np.where(words & np.uint32(0x80000000), -f, f)


def dequantise_f32(words, K_max, delta):
    """the same de-quantisation as the library computes it (float32 product), as uint32 float bits with the sign bit
    of the word: what Decoder.read_band returns for a band decoded with the 9/7 transform"""
    s = 31 - K_max
    mag = (words & np.uint32(0x7FFFFFFF)) >> np.uint32(s)
    rec = np.where(mag != 0, (mag << np.uint32(s)) | np.uint32(1 << (s - 1)), np.uint32(0)).astype(np.uint32)
    f = (rec.astype(np.float32) * np.float32(delta)).view(np.uint32)
    return np.where(mag != 0, f | (words & np.uint32(0x80000000)), np.uint32(0)).astype(np.uint32)


def check_rounding(r, t, tau, lo=None, hi=None, clip=None):
    """the comparison rule.  t = the model's float64 value just before rounding, r = the library's integer.  Where
    |frac(t) - 0.5| > tau, r must equal round(t); inside that band r must be floor(t) or ceil(t).  tau may be a scalar
    or an array.  With lo / hi, the output conversion's clamp is applied as the reference applies it, on t before the
    rounding: t < lo gives lo, t >= -lo gives hi (so t in [hi + 1/2, -lo) rounds to -lo = hi + 1; both sides of that
    threshold are allowed within tau of it).  clip = (a, b) then clips the result, as the 8 / 16-bit containers do.
    Returns (number of samples that break the rule, number of samples in the band, index of the first offending
    sample or None)."""
    t = np.asarray(t, np.float64)
    r = np.asarray(r, np.int64)
    fl = np.floor(t)
    band = np.abs(t - fl - 0.5) <= tau
    want = np.where(t - fl > 0.5, fl + 1, fl)
    alt = np.where(band, np.where(want == fl, fl + 1, fl), want)
    if lo is not None:
        top = float(-lo)
        near = np.abs(t - top) <= tau
        alt = np.where(near, np.where(t >= top, top, hi), np.where(t >= top, hi, np.where(t < lo, lo, alt)))
        want = np.where(t >= top, hi, np.where(t < lo, lo, want))
        band = band | near
    if clip is not None:
        want, alt = np.clip(want, *clip), np.clip(alt, *clip)
    bad = (r != want) & (r != alt)
    nbad = int(bad.sum())
    first = tuple(int(v) for v in np.argwhere(bad)[0]) if nbad else None
    return nbad, int(band.sum()), first


def expected_rounding(t, lo, hi, clip=None):
    """round(t) with the output conversion's clamp and the container's clip: the rule outside its tie band"""
    t = np.asarray(t, np.float64)
    want = np.where(t >= -lo, hi, np.where(t < lo, lo, np.floor(t + 0.5)))
    return want if clip is None else np.clip(want, *clip)
