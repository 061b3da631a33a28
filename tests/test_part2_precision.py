"""The Part 2 irreversible transforms held to a float64 model (below), sample by sample: arbitrary
irreversible ATK kernels of 2 to 8 lifting steps on DFS structures (levels that split both ways, one way or not at
all), run by the general shared-memory DWT kernels (dwt_fwd.cu / dwt_inv.cu), and the step sizes the encoder derives
for them.  Runs under the emulator build on the CPU tier and on the H100 with -m gpu.

For every configuration:
  forward   every band's quantiser output (Encoder.read_band) against the model's unrounded quantiser input, and on
            one tile bit for bit against the float32 restatement in the kernels' operation order;
  inverse   the decoder's band planes (float bits) against the float32 de-quantisation of the encoder's words, and its
            samples against the model's synthesis of those words;
  cross     the reference's decode of the same codestream differs from ours only inside the model's tie band.

Tolerances.  u = 2^-24 is the unit round-off of float32.  A lifting step x += A (l + r) is three float32 operations
(a sum, a product, a sum), each off by at most u times its result; on values no larger than M, the largest |sample|
entering the level, those results are at most 2M, 2|A|M and (1 + 2|A|)M, so the step adds at most
(3 + 4|A|) u M.  With the K scaling (one more rounding of a value near M) a direction of a level adds
R = sum_s (3 + 4|A_s|) + 1 roundings of size u M, and a level both ways 2R: ROUNDINGS(kernel).  The steps of a
kernel that passes DC unchanged (every kernel here) carry earlier errors on with a gain near one (C_GAIN), so after d
levels the coefficient is within C_GAIN * d * 2R * u * M of the model.  The
quantiser input v = x * delta_inv then lies within that times delta_inv, plus u |v| for the product and 1/2 for its
rounding: e_v.  The rule compares what reaches the codestream, the coded magnitude floor(|v| / 2^(31-K_max)), with
tie band e_v / 2^(31-K_max) around each quantisation threshold.
The inverse output is t = f * 2^B for a synthesised value f; the same count over D levels, plus the de-quantisation
and the inverse ICT, gives |f - model| <= C_GAIN * D * (2R + 4) * u * M_syn, M_syn the largest |value| of the
synthesised planes, so tau = that * 2^B.  The reference is held to the same band: every sample where its decode
differs from ours lies inside it.  Each check counts the samples inside its band and asserts that they stay a small
fraction, so a tolerance cannot pass by declaring every sample a tie: the band covers 2 tau of every unit interval,
which the bound above takes to about 5 % at 12 bits and eight levels, so TIE_FRACTION = 6 %.  The report prints the
largest error reached as a ratio of the bound (1.0 = at the bound)."""
import os
import struct
import subprocess
import sys
import numpy as np
import pytest
import cases
import ref97 as M
import test_irv_precision as IP
import openjph_b200 as ob

# ---- the float64 model of the general irreversible transform ------------------------------------------------------
# any irreversible ATK kernel (lifting steps A[s] in synthesis order and K) on any DFS structure (per level B both
# ways, H horizontal only, V vertical only, X unsplit; levels past the list repeat its last entry), whole-sample
# symmetric extension, de-interleave by absolute parity; the impulse-norm step sizes of every band; and a float32
# restatement of the forward path in the general DWT kernels' operation order.  The operations are restated from
# the standard (ITU-T T.801 Annex F / H, T.800 Annex F) with the kernel's float32 values promoted to float64, so the
# model is what the float32 kernels approximate.
F32 = np.float32
BAND_WEIGHT = (1.0, 2.0, 2.0, 4.0)        # the nominal range gain of LL / HL / LH / HH folded into the QCD steps


class Kernel:
    """an irreversible lifting kernel as the codestream carries it: A[s] in synthesis order, K, all float32"""

    def __init__(self, A, K):
        self.A = [float(F32(a)) for a in A]
        self.K = float(F32(K))
        self.Kinv = float(F32(1.0) / F32(K))      # the kernels scale by 1.0f / K, a float32 quotient
        self.A32 = [F32(a) for a in A]
        self.K32, self.Kinv32 = F32(K), F32(1.0) / F32(K)


def dfs_type(decomp, level):
    """DFS type of decomposition level `level` (1 = finest); None / "" is the dyadic structure"""
    if not decomp:
        return "B"
    return decomp[min(level, len(decomp)) - 1]


def splits(decomp, level):
    """(horizontal, vertical) split of a level"""
    t = dfs_type(decomp, level)
    return t in "BH", t in "BV"


def lift(x, start, forward, ker):
    """one-dimensional analysis (forward) or synthesis along axis 0 of x (float64, modified in place).  Analysis runs
    the steps s = N-1 .. 0, step s updating absolute parity s & 1 with x += A[s] (left + right), then low * 1/K and
    high * K; synthesis is the reverse.  Neighbours outside the line are mirrored (x[-1] = x[1], x[n] = x[n-2]) at
    every step, which equals the repeated whole-sample reflection of the input the kernels load for lines shorter than
    their support.  A line of one sample is not lifted: an odd-positioned sample is doubled (analysis) or halved."""
    n = x.shape[0]
    if n == 0:
        return x
    if n == 1:
        if start & 1:
            x *= 2.0 if forward else 0.5
        return x
    par = [M._nbrs(n, start, p) for p in (0, 1)]
    N = len(ker.A)
    if forward:
        for s in range(N - 1, -1, -1):
            i, l, r = par[s & 1]
            x[i] += ker.A[s] * (x[l] + x[r])
        x[par[0][0]] *= ker.Kinv
        x[par[1][0]] *= ker.K
    else:
        x[par[0][0]] *= ker.K
        x[par[1][0]] *= ker.Kinv
        for s in range(N):
            i, l, r = par[s & 1]
            x[i] -= ker.A[s] * (x[l] + x[r])
    return x


def _split(n, start, split):
    if not split:
        return np.arange(n), np.arange(0)
    return M._split(n, start)


def origins(x0, y0, levels, decomp):
    """origins[r] = (x0, y0) of resolution r (r = 1..levels; origins[0] is the final LL's): the next origin halves only
    in the directions a level splits"""
    out = [None] * (levels + 1)
    for r in range(levels, 0, -1):
        out[r] = (x0, y0)
        hs, vs = splits(decomp, levels - r + 1)
        x0, y0 = ((x0 + 1) >> 1) if hs else x0, ((y0 + 1) >> 1) if vs else y0
    out[0] = (x0, y0)
    return out


def analyse(x, x0, y0, levels, ker, decomp=None):
    """2-D analysis of a float64 plane at origin (x0, y0): per level vertical then horizontal lifting, in the directions
    the level splits; returns ({(res, band): float64 plane}, [max |x| of each level's input]).  A one-way level has
    only LL and HL (H) or LL and LH (V), an unsplit level (X) no band of its own."""
    out, mags = {}, []
    cur = np.array(x, np.float64)
    for r in range(levels, 0, -1):
        hs, vs = splits(decomp, levels - r + 1)
        mags.append(float(np.abs(cur).max()) if cur.size else 0.0)
        if vs:
            lift(cur, y0, True, ker)
        if hs:
            lift(cur.T, x0, True, ker)
        rows, cols = _split(cur.shape[0], y0, vs), _split(cur.shape[1], x0, hs)
        for b in (1, 2, 3):
            if (b & 1 and not hs) or (b & 2 and not vs):
                continue
            out[(r, b)] = cur[np.ix_(rows[b >> 1], cols[b & 1])]
        cur = cur[np.ix_(rows[0], cols[0])]
        x0, y0 = ((x0 + 1) >> 1) if hs else x0, ((y0 + 1) >> 1) if vs else y0
    out[(0, 0)] = cur
    return out, mags


def synthesise(bands, orgs, ker, decomp=None):
    """inverse of `analyse`: bands = {(res, band): float64 plane}, orgs = origins(...); per level horizontal then
    vertical synthesis.  Returns the float64 plane of the finest resolution."""
    D = len(orgs) - 1
    cur = bands[(0, 0)]
    for r in range(1, D + 1):
        hs, vs = splits(decomp, D - r + 1)
        x0, y0 = orgs[r]
        h = cur.shape[0] + (bands[(r, 2)].shape[0] if vs else 0)
        w = cur.shape[1] + (bands[(r, 1)].shape[1] if hs else 0)
        rows, cols = _split(h, y0, vs), _split(w, x0, hs)
        full = np.empty((h, w), np.float64)
        for b in (0, 1, 2, 3):
            if (b & 1 and not hs) or (b & 2 and not vs):
                continue
            full[np.ix_(rows[b >> 1], cols[b & 1])] = cur if b == 0 else bands[(r, b)]
        if hs:
            lift(full.T, x0, False, ker)
        if vs:
            lift(full, y0, False, ker)
        cur = full
    return cur


# ---- step sizes -------------------------------------------------------------------------------------------------------
def _line(ker):
    """length of the coarsest band of a line on which no waveform of the kernel reaches an edge: an n-stage waveform
    spans less than (N + 1) 2^n samples either side of its coefficient, N the kernel's step count"""
    return 4 * len(ker.A) + 8


def norm_1d(ker, n, high):
    """L2 norm of the synthesis waveform of one coefficient of the low band after n stages (high = False) or of the
    high band of stage n (n - 1 low stages first): a unit impulse synthesised through the model, on a line long enough
    that the waveform never meets its ends"""
    if n == 0:
        return 1.0
    m = _line(ker)
    low, hi = np.zeros(m), np.zeros(m)
    (hi if high else low)[m // 2] = 1.0
    for j in range(n, 0, -1):
        full = np.empty(2 * low.size)
        full[0::2], full[1::2] = low, hi
        low = lift(full, 0, False, ker)
        hi = np.zeros(low.size)
    return float(np.sqrt(np.sum(low * low)))


def bibo_1d(ker, n, high):
    """worst-case amplification of the same band: the largest L1 norm of a row of the analysis, from the analysis of
    every unit impulse of such a line (columns of an identity matrix; small n only)"""
    if n == 0:
        return 1.0
    m = _line(ker)
    L = m << n
    x = np.eye(L)
    ln = L
    for j in range(n):
        lift(x[:ln], 0, True, ker)
        x[:ln] = np.concatenate([x[0:ln:2], x[1:ln:2]])
        ln //= 2
    rows = x[ln:2 * ln] if high else x[:ln]
    return float(np.abs(rows).sum(axis=1).max())


def band_counts(decomp, D, r, b):
    """(stages in x, stages in y) between band (r, b) and the image, and whether the band is high in x / in y: a band
    of level l passes through every level 1..l that splits in a direction"""
    l = D - r + 1 if r else D
    nx = sum(splits(decomp, k)[0] for k in range(1, l + 1))
    ny = sum(splits(decomp, k)[1] for k in range(1, l + 1))
    return nx, ny, bool(b & 1), bool(b & 2)


def band_norm(ker, decomp, D, r, b, cache=None):
    """L2 norm of one coefficient's synthesis waveform of band (r, b): separable, so a product of 1-D norms"""
    cache = {} if cache is None else cache
    nx, ny, hx, hy = band_counts(decomp, D, r, b)
    for key in ((nx, hx), (ny, hy)):
        if key not in cache:
            cache[key] = norm_1d(ker, *key)
    return cache[(nx, hx)] * cache[(ny, hy)]


def step(base_delta, ker, decomp, D, r, b, cache=None):
    """the band's quantisation step, as band_info reports it times 2^(31 - K_max): base_delta / norm_b (the QCD stores
    base_delta / (norm_b * BAND_WEIGHT[b]) and the decoder multiplies the weight back in)"""
    return base_delta / band_norm(ker, decomp, D, r, b, cache)


def guard_bits(ker, decomp, D):
    """guard bits of the QCD: enough for the largest BIBO gain over the nominal range gain of any band, at least one"""
    cache = {}
    worst = 1.0
    for r, b in bands_of(decomp, D):
        nx, ny, hx, hy = band_counts(decomp, D, r, b)
        for key in ((nx, hx), (ny, hy)):
            if key not in cache:
                cache[key] = bibo_1d(ker, *key)
        worst = max(worst, cache[(nx, hx)] * cache[(ny, hy)] / BAND_WEIGHT[b])
    return max(1, int(np.ceil(np.log2(worst) - 1e-9)))


def bands_of(decomp, D):
    """(res, band) keys of every band, in marker order"""
    out = [(0, 0)]
    for r in range(1, D + 1):
        hs, vs = splits(decomp, D - r + 1)
        out += [(r, b) for b in (1, 2, 3) if not ((b & 1 and not hs) or (b & 2 and not vs))]
    return out


# ---- float32 restatement of the general kernels' forward path ---------------------------------------------------------
def _lift32(x, start, ker):
    """dwt_fwd.cu's lifting along axis 0 of a float32 array: x = x + A * (l + r), three correctly rounded float32
    operations in that order (no FMA), then low * (1/K) and high * K"""
    n = x.shape[0]
    if n == 1:
        if start & 1:
            x *= F32(2.0)
        return x
    par = [M._nbrs(n, start, p) for p in (0, 1)]
    for s in range(len(ker.A) - 1, -1, -1):
        i, l, r = par[s & 1]
        x[i] = x[i] + ker.A32[s] * (x[l] + x[r])
    x[par[0][0]] *= ker.Kinv32
    x[par[1][0]] *= ker.K32
    return x


def forward32(x, x0, y0, levels, ker, decomp, quant):
    """the quantised planes of one component, in the kernels' order: per level vertical steps, vertical K, horizontal
    steps, horizontal K, then rint(v * delta_inv) into sign-magnitude words.  x = the float32 input plane (after the
    sample conversion and the ICT), quant(res, band) -> float32 delta_inv.  Returns {(res, band): uint32 plane}."""
    def q(a, dinv):
        v = np.rint(a * F32(dinv)).astype(np.int64)
        return (np.where(v < 0, np.uint32(0x80000000), np.uint32(0)) | np.abs(v).astype(np.uint32)).astype(np.uint32)
    out = {}
    cur = np.array(x, F32)
    for r in range(levels, 0, -1):
        hs, vs = splits(decomp, levels - r + 1)
        if vs:
            _lift32(cur, y0, ker)
        if hs:
            _lift32(cur.T, x0, ker)
        rows, cols = _split(cur.shape[0], y0, vs), _split(cur.shape[1], x0, hs)
        for b in (1, 2, 3):
            if (b & 1 and not hs) or (b & 2 and not vs):
                continue
            out[(r, b)] = q(cur[np.ix_(rows[b >> 1], cols[b & 1])], quant(r, b))
        cur = np.ascontiguousarray(cur[np.ix_(rows[0], cols[0])])
        x0, y0 = ((x0 + 1) >> 1) if hs else x0, ((y0 + 1) >> 1) if vs else y0
    out[(0, 0)] = q(cur, quant(0, 0))
    return out


def to_float32(a, bit_depth, signed):
    """the kernels' sample conversion: (v - 2^(B-1)) * 2^-B in float32 (exact)"""
    half = 0 if signed else 1 << (bit_depth - 1)
    return ((np.asarray(a, np.int64) - half).astype(F32) * F32(2.0 ** -bit_depth)).astype(F32)


def ict_fwd32(r, g, b, comp):
    """dwt_fwd.cu's ICT: y = (a_r r + a_g g) + a_b b, cb = beta_cb (b - y), cr = beta_cr (r - y), all float32"""
    y = (F32(0.299) * r + F32(0.587) * g) + F32(0.114) * b
    return (y, F32(M.BETA_CB) * (b - y), F32(M.BETA_CR) * (r - y))[comp]


C_GAIN = 1.0
TIE_FRACTION = 0.06
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

IRV97 = dict(K=1.230174104914001, A=[0.443506852043971, 0.882911075530934, -0.052980118572961, -1.586134342059924])
REV53 = dict(reversible=True, steps=[(1, 2, 2), (-1, 1, 1)])


def _balanced(A):
    """an irreversible kernel from steps A (synthesis order) with A[1] and K chosen so that the high-pass removes DC
    and the low-pass passes it with gain one, as a wavelet kernel must (analysis: steps N-1 .. 0 on a constant line)"""
    A = list(A)
    e = o = 1.0
    for s in range(len(A) - 1, -1, -1):
        if s == 1:
            A[1] = -o / (2 * e)
        if s & 1:
            o += 2 * A[s] * e
        else:
            e += 2 * A[s] * o
    return dict(K=e, A=A)


K2 = dict(K=1.0, A=[0.25, -0.5])                                    # the 5/3 taps, irreversible
K6 = _balanced([0.05, 0, 0.1, -0.2, 0.15, -0.3])
K8 = _balanced([0.06, 0, -0.05, 0.1, 0.12, -0.25, 0.08, -0.35])


def ROUNDINGS(A):
    """float32 roundings of size u M in one level, both directions (see the module docstring)"""
    return 2 * (sum(3 + 4 * abs(a) for a in A) + 1)


def _cfg(w, h, nc=1, bd=10, x0=0, y0=0, st=ob.I32, **kw):
    d = dict(width=w + x0, height=h + y0, num_comps=nc, bit_depth=bd, reversible=False, offset=(x0, y0), st=st)
    d.setdefault("num_decomps", 3)
    d.update(kw)
    return d


CPU_CASES = [
    ("dfs_BHXV_97_even", _cfg(131, 67, decomp="BHXV", num_decomps=5, atk=IRV97)),     # level 5 repeats V
    ("dfs_BHXV_97_odd", _cfg(131, 67, x0=3, y0=1, decomp="BHXV", num_decomps=5, atk=IRV97)),
    ("dfs_VHB_builtin_odd", _cfg(97, 53, x0=1, y0=2, decomp="VHB", num_decomps=4)),
    ("k2_VHB_even", _cfg(90, 70, decomp="VHB", num_decomps=4, atk=K2)),
    ("k2_VHB_odd", _cfg(90, 70, x0=5, y0=3, decomp="VHB", num_decomps=4, atk=K2)),
    ("k6_BHH_even", _cfg(150, 40, decomp="BHH", num_decomps=4, atk=K6)),
    ("k6_BHH_odd", _cfg(150, 40, x0=1, y0=1, decomp="BHH", num_decomps=4, atk=K6)),
    ("k8_B_odd", _cfg(77, 45, x0=3, y0=5, num_decomps=4, atk=K8)),
    ("k8_XB_even", _cfg(77, 45, decomp="XB", num_decomps=3, atk=K8)),
    ("tile_w127_h31", _cfg(127, 31, x0=1, decomp="BV", atk=K8)),
    ("tile_w128_h32", _cfg(128, 32, decomp="BH", atk=K8, num_decomps=2)),
    ("tile_w129_h33", _cfg(129, 33, x0=1, y0=1, decomp="B", atk=K8, num_decomps=2)),
    ("tile_w257_h65", _cfg(257, 65, x0=2, y0=1, decomp="BHV", atk=IRV97, num_decomps=3)),
    ("tiles_offsets", _cfg(150, 90, nc=3, x0=5, y0=3, color_transform=True, tile=(64, 48), tile_offset=(3, 2),
                           decomp="BHV", atk=IRV97)),
    ("ict_k6_u8", _cfg(70, 41, nc=3, bd=8, x0=1, y0=1, st=ob.U8, color_transform=True, decomp="HB", atk=K6)),
    ("u16_12bit_k8", _cfg(66, 37, bd=12, x0=2, st=ob.U16, decomp="VB", atk=K8)),
    ("signed12_k2", _cfg(61, 29, bd=12, x0=3, y0=1, is_signed=True, decomp="BX", atk=K2)),
    ("H8_builtin", _cfg(600, 20, x0=1, decomp="H", num_decomps=8)),                  # eight horizontal levels
    ("V7H_k6", _cfg(24, 400, y0=1, decomp="VVVVVVVH", num_decomps=8, atk=K6)),
]
# lines of 1 to 9 samples under the 8-step kernel: the kernels reflect a line shorter than their 8-sample halo over and
# over, and a line of one sample is not lifted
for _w, _h in ((1, 9), (9, 1), (2, 5), (3, 7), (5, 3), (7, 8), (4, 4), (6, 2), (9, 9)):
    for _o in (0, 1):
        CPU_CASES.append(("k8_short_%dx%d_o%d" % (_w, _h, _o), _cfg(_w, _h, x0=_o, y0=_o, decomp="BHV", atk=K8, num_decomps=3)))
BIG_CASES = [
    ("big_3840x2160_BHVHB_97", _cfg(3840, 2160, nc=3, bd=10, st=ob.U16, color_transform=True, decomp="BHVHB",
                                    num_decomps=5, atk=IRV97)),
    ("big_4600x300_k8_level1_36_tiles", _cfg(4600, 300, x0=1, decomp="BH", num_decomps=3, atk=K8)),
]
ALL = dict(CPU_CASES + BIG_CASES)


def _kernel(kw):
    a = kw.get("atk") or IRV97
    return Kernel(a["A"], a["K"])


def _strip(kw):
    return {k: v for k, v in kw.items() if k != "st"}


# ---- one configuration --------------------------------------------------------------------------------------------
def run_case(lib, name, ref):
    kw = ALL[name]
    st = kw["st"]
    p = cases.make(_strip(kw))
    frame = cases.frame_for(p)
    ker, decomp = _kernel(kw), kw.get("decomp")
    B = p.bit_depth[0]
    signed = bool(p.is_signed[0])
    half = 0 if signed else 1 << (B - 1)
    D = p.num_decomps
    R = ROUNDINGS(ker.A)
    planes = frame if st == ob.I32 else [f.astype(np.uint8 if st == ob.U8 else np.uint16) for f in frame]
    enc = ob.Encoder(p, st, lib=lib)
    cs = enc.encode(planes)
    dec = ob.Decoder(lib=lib)
    out = [a.astype(np.int64) for a in dec.decode(cs, st)]
    refout = [a.astype(np.int64) for a in ref.decode(cs)[0]]
    comp_org = [(-(-p.off_x // p.dx[c]), -(-p.off_y // p.dy[c])) for c in range(p.num_comps)]
    s = dict(fwd_n=0, fwd_tie=0, inv_n=0, inv_tie=0, cross_n=0, cross_diff=0, fwd_ratio=0.0, inv_ratio=0.0)
    ct = bool(p.color_transform)
    keys = bands_of(decomp, D)
    for tile, rects in IP._tile_comp_rects(p):
        synth = []
        for c, x0, y0, x1, y1 in rects:
            info = {rb: enc.band_info(tile, c, *rb) for rb in keys}
            orgs = origins(x0, y0, D, decomp)
            for (r, b) in keys:
                if r:
                    assert (info[(r, b)]["res_x0"], info[(r, b)]["res_y0"]) == orgs[r], (name, tile, c, r, b)
            ox, oy = comp_org[c]
            sl = (slice(y0 - oy, y1 - oy), slice(x0 - ox, x1 - ox))
            xs = M.to_float(frame[c][sl], B, signed)
            if ct and c < 3:
                xs = M.ict_fwd(*[M.to_float(frame[k][sl], B, signed) for k in range(3)], c)
            bands, mags = analyse(xs, x0, y0, D, ker, decomp)
            assert sorted(bands) == sorted(keys), (name, sorted(bands))
            words = {}
            for (r, b), a in bands.items():
                bi = info[(r, b)]
                g = enc.read_band(tile, c, r, b)
                if not a.size:
                    assert not g.size, (name, tile, c, r, b)
                    words[(r, b)] = np.zeros(a.shape, np.uint32)
                    continue
                assert g.shape == a.shape, (name, tile, c, r, b, g.shape, a.shape)
                words[(r, b)] = g
                kmax, dinv = int(bi["K_max"]), float(bi["delta_inv"])
                t = a * dinv
                d = D - r + 1 if r else D
                e_x = C_GAIN * d * R * M.U32 * max(mags[:d]) * dinv
                e_v = e_x + M.U32 * np.abs(t) + 0.5
                gs = np.where(g & 0x80000000, -1.0, 1.0) * (g & 0x7FFFFFFF).astype(np.float64)
                err = np.abs(gs - t)
                s["fwd_ratio"] = max(s["fwd_ratio"], float(((err - 0.5 - M.U32 * np.abs(t)) / e_x).max()))
                assert (err <= e_v).all(), ("quantiser input off the model", name, tile, c, r, b,
                                            np.unravel_index(int(np.argmax(err - e_v)), err.shape), float(err.max()))
                sh = 2.0 ** (31 - kmax)
                q = (g & 0x7FFFFFFF) >> np.uint32(31 - kmax)
                nbad, ntie, first = M.check_rounding(q, np.abs(t) / sh - 0.5, e_v / sh)
                assert nbad == 0, ("coded magnitude differs from the model's", name, tile, c, r, b, first)
                sig = (q != 0) & (np.abs(t) > e_v)
                assert np.array_equal(np.signbit(t[sig]), (g[sig] >> 31).astype(bool)), ("sign", name, tile, c, r, b)
                s["fwd_n"] += g.size; s["fwd_tie"] += ntie
                db = dec.read_band(tile, c, r, b)
                assert np.array_equal(db, M.dequantise_f32(g, kmax, bi["delta"])), ("decoder band plane", name, tile, c, r, b)
            deq = {rb: M.dequantise(words[rb], int(info[rb]["K_max"]), float(info[rb]["delta"])) for rb in words}
            synth.append(synthesise(deq, orgs, ker, decomp) if D else deq[(0, 0)])
            del bands, deq
        if ct:
            synth[:3] = M.ict_inv(*synth[:3])
        lo, hi = -(1 << (B - 1)), (1 << (B - 1)) - 1
        for (c, x0, y0, x1, y1), f in zip(rects, synth):
            ox, oy = comp_org[c]
            sl = (slice(y0 - oy, y1 - oy), slice(x0 - ox, x1 - ox))
            t = f * float(1 << B)
            m_syn = float(np.abs(f).max()) if f.size else 0.0
            tau = C_GAIN * max(D, 1) * (R + 4) * M.U32 * max(m_syn, 0.5) * (1 << B)
            r_lib = out[c][sl] - half
            clip = None if st == ob.I32 else (-half, (1 << B) - 1 - half)
            nbad, ntie, first = M.check_rounding(r_lib, t, tau, lo, hi, clip)
            off = (r_lib != M.expected_rounding(t, lo, hi, clip)) & (np.abs(t + half) < 2 ** B - 1)
            if off.any():      # how far inside the band the rounding decisions that differ lie, as a share of tau
                s["inv_ratio"] = max(s["inv_ratio"], float(np.abs(t - np.floor(t) - 0.5)[off].max()) / tau)
            assert nbad == 0, ("decoded sample differs from the model's", name, tile, c, first,
                               None if first is None else (int(r_lib[first]), float(t[first])))
            s["inv_n"] += t.size; s["inv_tie"] += ntie
            nbad_ref, _, first = M.check_rounding(refout[c][sl] - half, t, tau, lo, hi, clip)
            assert nbad_ref == 0, ("the reference's decode differs from the model's", name, tile, c, first)
            dr = refout[c][sl] - out[c][sl]
            fl = np.floor(t)
            in_band = (np.abs(t - fl - 0.5) <= tau) | (np.abs(t + lo) <= tau)
            assert not (dr != 0)[~in_band].any(), ("reference differs outside the tie band", name, tile, c)
            s["cross_n"] += t.size; s["cross_diff"] += int((dr != 0).sum())
    for k in ("fwd", "inv"):
        assert s[k + "_tie"] <= TIE_FRACTION * max(s[k + "_n"], 1) + 2, (name, k, s)
    return s, p, enc


def _report(name, s):
    print("%s: forward %d/%d in the tie band, inverse %d/%d, reference differs on %d/%d, error ratios %.3f / %.3f"
          % (name, s["fwd_tie"], s["fwd_n"], s["inv_tie"], s["inv_n"], s["cross_diff"], s["cross_n"],
             s["fwd_ratio"], s["inv_ratio"]))


def _exact(name, p, enc):
    """the quantised planes equal the float32 restatement in the kernels' order bit for bit, on the first tile"""
    kw = ALL[name]
    ker, decomp, D = _kernel(kw), kw.get("decomp"), p.num_decomps
    frame = cases.frame_for(p)
    B, signed = p.bit_depth[0], bool(p.is_signed[0])
    _, rects = IP._tile_comp_rects(p)[0]
    xs = []
    for c, x0, y0, x1, y1 in rects:
        ox, oy = -(-p.off_x // p.dx[c]), -(-p.off_y // p.dy[c])
        xs.append(to_float32(frame[c][y0 - oy:y1 - oy, x0 - ox:x1 - ox], B, signed))
    for c, x0, y0, x1, y1 in rects:
        x = ict_fwd32(*xs[:3], c) if p.color_transform and c < 3 else xs[c]
        want = forward32(x, x0, y0, D, ker, decomp, lambda r, b: enc.band_info(0, c, r, b)["delta_inv"])
        for (r, b), w in want.items():
            g = enc.read_band(0, c, r, b)
            assert (g.size == 0 and w.size == 0) or np.array_equal(g, w), (name, c, r, b)


# ---- CPU tier -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n, _ in CPU_CASES])
def test_part2_against_model_emulated(name, emu_lib, ref):
    s, p, enc = run_case(emu_lib, name, ref)
    _report(name, s)
    _exact(name, p, enc)


# ---- step sizes -----------------------------------------------------------------------------------------------------
def _qcd(cs):
    i = cs.index(b"\xff\x5c"); n = struct.unpack(">H", cs[i + 2:i + 4])[0]
    return cs[i + 4], cs[i + 5:i + 2 + n]


def _steps(q):
    u = struct.unpack(">%dH" % (len(q) // 2), q)
    return [(1 + (x & 0x7FF) / 2048.0) / 2.0 ** (x >> 11) for x in u]


def _encode_zeros(lib, nd, rev, **kw):
    p = ob.make_params(64, 64, 1, 8, num_decomps=nd, reversible=rev, **kw)
    return ob.Encoder(p, ob.I32, lib=lib).encode([np.zeros((64, 64), np.int32)])


def test_atk_97_steps_match_the_builtin_at_every_depth(emu_lib):
    """the 9/7 taps given as an ATK get the built-in 9/7's step sizes (the reference's tables) at every level count the
    library accepts; the six-level gains used to be reused for deeper levels, which gave the deepest bands steps 2 to
    2^14 times too large"""
    worst = []
    for nd in range(1, 33):
        try:
            sa, qa = _qcd(_encode_zeros(emu_lib, nd, False))
        except ob.OjphError as e:           # the built-in's deepest steps need more than 32-bit coefficients: so do the ATK's
            with pytest.raises(ob.OjphError) as e2:
                _encode_zeros(emu_lib, nd, False, atk=IRV97)
            assert str(e2.value) == str(e), nd
            worst.append(None)
            continue
        sb, qb = _qcd(_encode_zeros(emu_lib, nd, False, atk=IRV97))
        assert sa == sb and len(qa) == len(qb), nd
        da, db = _steps(qa), _steps(qb)
        ratio = max(max(x / y, y / x) for x, y in zip(da, db))
        worst.append(ratio)
        assert ratio - 1 <= 2e-3, (nd, ratio)
    print("largest step ratio per level count", [r and round(r, 5) for r in worst])
    assert sum(r is not None for r in worst) >= 12, worst


def test_atk_53_qcd_is_the_builtin_at_every_depth(emu_lib):
    """the 5/3 taps given as a reversible ATK: the QCD is byte for byte the built-in 5/3's (its guard bits and
    exponents come from the BIBO gains)"""
    for nd in range(1, 33):
        assert _qcd(_encode_zeros(emu_lib, nd, True)) == _qcd(_encode_zeros(emu_lib, nd, True, atk=REV53)), nd


STEP_CASES = [
    ("H8", None, "H", 8, 12),
    ("V9", None, "V", 9, 8),
    ("HHHHHHHV", None, "HHHHHHHV", 9, 10),
    ("BHVX", None, "BHVX", 6, 8),
    ("X_first", None, "XXB", 4, 8),
    ("k6_H7", K6, "H", 7, 8),
    ("k8_BVH", K8, "BVH", 5, 12),
    ("k2_VVVVVVVB", K2, "VVVVVVVB", 8, 8),
    ("97_B8", IRV97, "B", 8, 8),
]


@pytest.mark.parametrize("name", [c[0] for c in STEP_CASES])
def test_dfs_steps_are_the_impulse_norm_steps(name, emu_lib):
    """every band's step (band_info) is base_delta / the L2 norm of its synthesis waveform, the model's impulse
    response, within the QCD's 11-bit mantissa; up to six levels in each direction the guard bits are the model's
    BIBO ones"""
    _, atk, decomp, nd, bd = [c for c in STEP_CASES if c[0] == name][0]
    kw = dict(decomp=decomp)
    if atk:
        kw["atk"] = atk
    p = ob.make_params(300, 300, 1, bd, num_decomps=nd, reversible=False, **kw)
    enc = ob.Encoder(p, ob.I32, lib=emu_lib)
    cs = enc.encode([np.zeros((300, 300), np.int32)])
    ker = Kernel((atk or IRV97)["A"], (atk or IRV97)["K"])
    base = 1.0 / (1 << bd)
    cache = {}
    for r, b in bands_of(decomp, nd):
        bi = enc.band_info(0, 0, r, b)
        got = float(bi["delta"]) * 2.0 ** (31 - int(bi["K_max"]))
        want = step(base, ker, decomp, nd, r, b, cache)
        assert abs(got / want - 1) <= 2.0 ** -11, (name, r, b, got, want)
    nx, ny, _, _ = band_counts(decomp, nd, 0, 0)
    if max(nx, ny) <= 6:
        assert _qcd(cs)[0] >> 5 == guard_bits(ker, decomp, nd), name


# QCD bodies (Sqcd, then the steps) the encoder wrote before the gains reached past six levels: every structure with at
# most six levels in each direction keeps them
_IRV6 = dict(K=1.1, A=[0.1, -0.2, 0.05, 0.3, -0.1, 0.2])
_IRV8 = dict(K=0.9, A=[0.05, -0.1, 0.2, -0.3, 0.15, -0.25, 0.1, -0.45])
_REV8 = dict(reversible=True, steps=[(1, 4, 3), (-1, 1, 1), (1, 2, 2), (-1, 2, 2), (1, 8, 4), (-1, 4, 3), (1, 2, 2), (-1, 1, 1)])
PINNED_QCD = [
    (dict(decomp="BHVHB", atk=IRV97), 5, 8, "2262b962a362c962b45aee5003539a57d257d25761"),
    (dict(decomp="HVHVHV"), 6, 12, "228735874c7aee7003739a77d26b17"),
    (dict(decomp="BBBBBB", atk=_REV8), 6, 8, "2068686870606068606060585860585858505058"),
    (dict(decomp="BHVHB", atk=_REV8), 5, 12, "2078808080787870707078"),
    (dict(decomp="XBH", atk=_IRV6), 4, 8, "224994533954a3566c566c5083"),
    (dict(decomp="HHHHHH", atk=_IRV8), 6, 12, "627ad478027acf7e9c71f775cd68e9"),
    (dict(decomp="VVVVVV", atk=REV53), 6, 8, "2040484848484840"),
]


def test_qcd_up_to_six_levels_unchanged(emu_lib):
    """up to six levels in each direction the gains are measured as they always were: the QCD bytes stay put"""
    for kw, nd, bd, want in PINNED_QCD:
        rev = bool(kw.get("atk", {}).get("reversible"))
        p = ob.make_params(64, 64, 1, bd, num_decomps=nd, reversible=rev, **kw)
        cs = ob.Encoder(p, ob.I32, lib=emu_lib).encode([np.zeros((64, 64), np.int32)])
        i = cs.index(b"\xff\x5c"); n = struct.unpack(">H", cs[i + 2:i + 4])[0]
        assert cs[i + 4:i + 2 + n].hex() == want, (kw, nd, bd, cs[i + 4:i + 2 + n].hex())


# ---- the general kernels on dyadic frames -------------------------------------------------------------------------
def _child(gpu, env):
    """(encoder launches, decoder launches) of a four-component 9/7 ICT frame, and whether a 5/3 frame's codestream is
    the reference's, in a process of its own (the switch is read when a codec is created)"""
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import numpy as np, openjph_b200 as ob, cases, refharness as R\n"
            "lib = None\n" % (ROOT, os.path.join(ROOT, "tests")) +
            ("" if gpu else "import emu; lib = emu.emu_lib()\n") +
            "p = ob.make_params(96, 64, 4, 8, num_decomps=3, reversible=False, color_transform=True)\n"
            "f = [np.full((64, 96), 100 + 20 * c, np.int32) for c in range(4)]\n"
            "e = ob.Encoder(p, ob.I32, lib=lib); cs = e.encode(f); d = ob.Decoder(lib=lib); d.decode(cs)\n"
            "same = 1\n"
            "for kw in (dict(width=123, height=77, num_comps=3, bit_depth=8, num_decomps=5, reversible=True, color_transform=True),\n"
            "           dict(width=300, height=200, num_comps=1, bit_depth=12, num_decomps=4, reversible=True, offset=(7, 5), tile=(128, 100), tile_offset=(3, 2))):\n"
            "    q = cases.make(kw); fr = cases.frame_for(q)\n"
            "    same &= int(ob.Encoder(q, ob.I32, lib=lib).encode(fr) == R.encode(q, fr))\n"
            "print(e.kernel_launches, d.kernel_launches, same)\n")
    env = dict({k: v for k, v in os.environ.items() if k != "OJB_NO_STREAM_DWT"}, **env)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    return tuple(int(v) for v in r.stdout.split()[-3:])


def _switch_takes_effect(gpu):
    """OJB_NO_STREAM_DWT sends every level to the general kernels: a four-component ICT frame's first level then runs
    its colour triple and its fourth component in one launch each way instead of two; 5/3 codestreams stay the
    reference's byte for byte"""
    plain = _child(gpu, {})
    forced = _child(gpu, {"OJB_NO_STREAM_DWT": "1"})
    assert forced[:2] == (plain[0] - 1, plain[1] - 1), (plain, forced)
    assert plain[2] == forced[2] == 1, (plain, forced)


def test_no_stream_dwt_switch_emulated(emu_lib, ref):
    _switch_takes_effect(False)


# ---- GPU tier -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n, _ in CPU_CASES + BIG_CASES])
def test_part2_against_model_gpu(name, gpu_lib, ref):
    s, p, enc = run_case(None, name, ref)
    _report(name, s)
    _exact(name, p, enc)


@pytest.mark.gpu
def test_no_stream_dwt_switch_gpu(gpu_lib, ref):
    _switch_takes_effect(True)
