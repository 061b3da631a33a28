// ojb_params.cpp -- see ojb_params.h for the reference file:line each piece mirrors.
#include "ojb_params.h"
#include <cmath>
#include <cstring>
#include <algorithm>
#include <algorithm>

namespace ojb {

#include "ojb_gain_tables.inc"

namespace {

inline float energy_gain_l(uint32_t d, bool rev) { return rev ? kEnergy_5x3_l[d] : kEnergy_9x7_l[d]; }
inline float energy_gain_h(uint32_t d, bool rev) { return rev ? kEnergy_5x3_h[d] : kEnergy_9x7_h[d]; }
inline float bibo_gain_l(uint32_t d, bool rev) { return rev ? kBibo_5x3_l[d] : kBibo_9x7_l[d]; }
inline float bibo_gain_h(uint32_t d, bool rev) { return rev ? kBibo_5x3_h[d] : kBibo_9x7_h[d]; }

// Qfactor model (ojph_params.cpp:604-726): visual weight tables by chroma format and
// component type, reference step from the quality factor.
const float* visual_weights(uint32_t sx, uint32_t sy, int ctype, bool& ok) {
  ok = true;
  int fmt;  // 1: 420, 2: 422, 3: 444
  if (sx == 2 && sy == 2) fmt = 1;
  else if (sx == 2 && sy == 1) fmt = 2;
  else if (sx == 1 && sy == 1) fmt = 3;
  else { ok = false; return kVw_y; }
  if (ctype == 0) return kVw_y;
  if (ctype == 1) return fmt == 1 ? kVw_cb420 : (fmt == 2 ? kVw_cb422 : kVw_cb444);
  return fmt == 1 ? kVw_cr420 : (fmt == 2 ? kVw_cr422 : kVw_cr444);
}
inline float vw_weight(const float* v, uint32_t level, uint32_t band) {
  if (band == 0) return v[18];
  level = std::min(level, 6u);
  return v[(level - 1) * 3 + (3 - band)];
}
inline float vw_gain(int ctype) {
  if (ctype == 0) return 1.0f;
  if (ctype == 1) return 1.8051f / 1.7321f;
  return 1.5734f / 1.7321f;
}
// Reference step size of the Qfactor model (param_qcd::get_delta_ref, ojph_params.cpp:690-725): a JPEG-style quality
// scale `slope(Q)` -- 50/Q below 50, 2 (1 - Q/100) above -- weighted by a colour / level factor that is 0.04 up to the
// knee Q = 65, 0.10 from Q = 97 and geometrically interpolated in log-slope between them; `blend` (1 at the knee, 0 at
// the top) is also the exponent the visual weights are raised to.  Every operation is in float in this order: the
// packed QCD values must come out identical to the reference's.
float vw_delta_ref(uint32_t qfactor, uint32_t bit_depth, float& blend) {
  constexpr uint8_t knee = 65, top = 97;
  constexpr float w_knee = 0.04f, w_top = 0.10f;
  constexpr float slope_knee = 2.0f * (1.0f - knee / 100.0f);
  constexpr float slope_top = 2.0f * (1.0f - top / 100.0f);
  const float slope = qfactor < 50 ? 50.0f / (float)qfactor : 2.0f * (1.0f - (float)qfactor / 100.0f);
  float weight;
  if (qfactor <= knee) { blend = 1.0f; weight = w_knee; }
  else if (qfactor < top) {
    blend = std::log(slope) - std::log(slope_top);
    blend /= std::log(slope_knee) - std::log(slope_top);
    weight = w_top * std::pow(w_knee / w_top, blend);
  } else { blend = 0.0f; weight = w_top; }
  const float floor_step = std::sqrt(0.5f) * std::ldexp(1.0f, -(int)bit_depth);      // never below ~0.7 LSB
  return weight * slope + floor_step;
}

// exponent/mantissa packing of an irreversible step (encode_SPqcd, ojph_params.cpp:1602)
uint16_t pack_step(float delta) {
  int exp = 0;
  while (delta < 1.0f) { exp++; delta *= 2.0f; }
  int mantissa = (int)round(delta * (float)(1 << 11)) - (1 << 11);
  mantissa = mantissa < (1 << 11) ? mantissa : 0x7FF;
  return (uint16_t)((exp << 11) | mantissa);
}

} // namespace

//------------------------------------------------------------------------------------------
// QuantSet
//------------------------------------------------------------------------------------------
void QuantSet::set_rev_quant(uint32_t nd, uint32_t bd, bool color) {
  uint32_t B = bd + (color ? 1u : 0u);          // one extra bit after the RCT
  int s = 0;
  double bl = bibo_gain_l(nd, true);
  uint32_t X = (uint32_t)ceil(log(bl * bl) / M_LN2);
  uint8_t tmp[97];
  tmp[s++] = (uint8_t)(B + X);
  uint32_t max_BX = B + X;
  for (uint32_t d = nd; d > 0; --d) {
    double l = bibo_gain_l(d, true), h = bibo_gain_h(d - 1, true);
    X = (uint32_t)ceil(log(h * l) / M_LN2);
    tmp[s++] = (uint8_t)(B + X); max_BX = std::max(max_BX, B + X);
    tmp[s++] = (uint8_t)(B + X);
    X = (uint32_t)ceil(log(h * h) / M_LN2);
    tmp[s++] = (uint8_t)(B + X); max_BX = std::max(max_BX, B + X);
  }
  if (max_BX > 38)
    fail(0x00050151, "The specified combination of bit_depth, colour transform, and type of "
         "wavelet transform requires more than 38 bits; it requires %d bits.", max_BX);
  int guard = std::max(1, (int)max_BX - 31);
  Sqcd = (uint8_t)(guard << 5);
  for (int i = 0; i < s; ++i) SP[i] = (uint16_t)(uint8_t)((uint8_t)(tmp[i] - guard) << 3);
}

void QuantSet::set_irrev_quant(uint32_t nd) {
  Sqcd = (uint8_t)((1 << 5) | 0x2);             // one guard bit, scalar expounded
  float g_c = 1.0f, delta_ref = base_delta, power = 1.0f;
  const float* weights = kVw_no_weights;
  if (qfactor != 0) {
    bool ok;
    weights = visual_weights(sx, sy, ctype, ok);
    if (!ok)
      fail(0x00050161, "Qfactor can only be used on components with 4:4:4, 4:2:2 or 4:2:0 sampling");
    if (ctype == 0 && sx != 1 && sy != 1)
      fail(0x00050162, "Qfactor can only be used for a Y or luminance component when it is "
           "not downsampled.");
    g_c = vw_gain(ctype);
    delta_ref = vw_delta_ref(qfactor, bit_depth, power);
  }
  uint32_t b = 0;
  float gl = energy_gain_l(nd, false);
  float w_b = std::pow(vw_weight(weights, nd, 0), power);
  SP[b++] = pack_step(delta_ref / (gl * gl * g_c * w_b));
  for (uint32_t d = nd; d > 0; --d) {
    float l = energy_gain_l(d, false), h = energy_gain_h(d - 1, false);
    w_b = std::pow(vw_weight(weights, d, 1), power);
    SP[b++] = pack_step(delta_ref / (h * l * g_c * w_b));
    w_b = std::pow(vw_weight(weights, d, 2), power);
    SP[b++] = pack_step(delta_ref / (l * h * g_c * w_b));
    w_b = std::pow(vw_weight(weights, d, 3), power);
    SP[b++] = pack_step(delta_ref / (h * h * g_c * w_b));
  }
}

uint32_t QuantSet::kmax_at(uint32_t idx) const {
  if (idx >= num_subbands) idx = num_subbands - 1;
  uint32_t bits = 0;
  if ((Sqcd & 0x1F) == 0) { bits = (uint32_t)(SP[idx] & 0xFF) >> 3; bits = bits ? bits - 1 : 0; }
  else bits = (uint32_t)(SP[idx] >> 11) - 1;
  return bits + guard_bits();
}

uint32_t QuantSet::largest_kmax() const {
  uint32_t bits = 0;
  for (uint32_t i = 0; i < num_subbands; ++i) {
    uint32_t t;
    if ((Sqcd & 0x1F) == 0) { t = (uint32_t)(SP[i] & 0xFF) >> 3; t = t ? t - 1 : 0; }
    else t = (uint32_t)(SP[i] >> 11) - 1;
    bits = std::max(bits, t);
  }
  return bits + guard_bits();
}

float QuantSet::irrev_delta_at(uint32_t idx, uint32_t band) const {
  static const float arr[4] = { 1.0f, 2.0f, 2.0f, 4.0f };
  if ((Sqcd & 0x1F) != 2)
    fail(0x00050101, "irreversible transform with reversible (no quantization) step sizes");
  if (idx >= num_subbands) idx = num_subbands - 1;
  int eps = SP[idx] >> 11;
  float mantissa = (float)((SP[idx] & 0x7FF) | 0x800) * arr[band];
  mantissa /= (float)(1 << 11);
  mantissa /= (float)(1u << eps);
  return mantissa;
}

//------------------------------------------------------------------------------------------
// DFS / ATK (Part 2 wavelet structures)
//------------------------------------------------------------------------------------------
DfsType DfsSpec::type(uint32_t decomp_level) const {
  decomp_level = std::min<uint32_t>(decomp_level, Ids);      // levels past the list repeat its last entry
  uint32_t d = decomp_level - 1;
  return (DfsType)((Ddfs[d >> 2] >> (6 - 2 * (d & 3))) & 3);
}

uint32_t DfsSpec::subband_idx(const uint32_t num_decomps, uint32_t res, uint32_t band) const {
  static const uint32_t ns[4] = { 0, 3, 1, 1 };
  if (res == 0) return 0;
  uint32_t idx = 0, i = 1;
  for (; i < res; ++i) idx += ns[type(num_decomps - i + 1)];
  idx += band;
  if (type(num_decomps - i + 1) == DFS_VERT && band == 2) --idx;
  return idx;
}

AtkSpec AtkSpec::irv97() {
  AtkSpec a; a.Satk = 0x4a00; a.K = (float)1.230174104914001; a.steps.resize(4);
  a.steps[0].A = (float)0.443506852043971; a.steps[1].A = (float)0.882911075530934;
  a.steps[2].A = (float)-0.052980118572961; a.steps[3].A = (float)-1.586134342059924;
  return a;
}
AtkSpec AtkSpec::rev53() {
  AtkSpec a; a.Satk = 0x5801; a.steps.resize(2);
  a.steps[0].a = 1; a.steps[0].b = 2; a.steps[0].e = 2;
  a.steps[1].a = -1; a.steps[1].b = 1; a.steps[1].e = 1;
  return a;
}

const AtkSpec& Params::atk_for(uint32_t w) const {
  static const AtkSpec k97 = AtkSpec::irv97(), k53 = AtkSpec::rev53();
  for (const AtkSpec& a : atk) if (a.index() == w) return a;
  if (w == 0) return k97;
  if (w == 1) return k53;
  fail(0x00050131, "A COD/COC segment employs the DWT kernel atk = %d, but a corresponding ATK segment cannot be found.", w);
}

const DfsSpec* Params::dfs_of(uint32_t c) const {
  const CodStyle* s = find_coc(c);
  if (s == nullptr || s->dfs_idx < 0) return nullptr;
  if (dfs.empty())
    fail(0x00070001, "There is a problem with codestream marker segments. COD/COC specifies the use of a DFS marker "
         "but there are no DFS markers within the main codestream headers");
  for (const DfsSpec& d : dfs) if (d.Sdfs == (uint16_t)s->dfs_idx) return &d;
  fail(0x00070002, "There is a problem with codestream marker segments. COD/COC specifies the use of a DFS marker "
       "with index %d, but there are no such marker within the main codestream headers", s->dfs_idx);
}

void Params::res_downsamp(uint32_t c, uint32_t skipped, uint32_t& fx, uint32_t& fy) const {
  fx = fy = 1;
  for (uint32_t level = 1; level <= skipped; ++level) {
    DfsType t = dwt_type(c, level);
    if (t == DFS_BIDIR || t == DFS_HORZ) fx *= 2;
    if (t == DFS_BIDIR || t == DFS_VERT) fy *= 2;
  }
}

uint32_t Params::subband_index(uint32_t c, uint32_t res, uint32_t band) const {
  const DfsSpec* d = dfs_of(c);
  if (d) return d->subband_idx(decomps(c), res, band);
  return res ? (res - 1) * 3 + band : 0;
}

namespace {
// Step sizes for a decomposition structure / kernel the reference has no tables for (it only decodes them): the
// same recipe as set_rev_quant / set_irrev_quant (ojph_params.cpp:1495-1599) with the gains measured on the
// kernel itself, 1-D and linearised (a reversible step is a / 2^e without rounding), for every level count a component
// can have (DEPTH):
//   bibo_l[n] / bibo_h[n]: worst-case amplification of n low-pass stages / of n - 1 low-pass stages and a high-pass one
//   norm_l[n] / norm_h[n]: L2 norm of the synthesis waveform of one coefficient of those bands
// Up to FINITE levels they are measured on a line of 16 << FINITE samples with symmetric extension, even origin (the
// BIBO gains from the whole analysis matrix); the codestreams of such structures keep the steps they always had.
// Deeper levels take the waveforms on an unbounded line: a unit impulse in the band carried back through n stages,
// by synthesis or by the transpose of analysis (the transpose of the step "x[i] += a (x[i-1] + x[i+1]) on parity p"
// is the same step on parity 1 - p, and the transposed stage runs the steps in synthesis order).  The work doubles
// with every level, so past EXACT levels the gains continue at the ratio they settle to: the L2 norms at their last
// measured ratio (sqrt(2) for the 9/7), the L1 norms at the DC gain of a low-pass analysis stage (one for every kernel
// whose low-pass passes DC unchanged).
struct KernelGains {
  enum { DEPTH = 32, FINITE = 6, EXACT = 12 };
  double bibo_l[DEPTH + 1], bibo_h[DEPTH + 1], norm_l[DEPTH + 1], norm_h[DEPTH + 1];
  static double coef(const AtkSpec& k, size_t s) { return k.reversible() ? (double)k.steps[s].a / (double)(1u << k.steps[s].e) : (double)k.steps[s].A; }
  // one analysis stage on the first len entries of every column of m (rows = samples), even origin
  static void analyse(std::vector<std::vector<double>>& m, size_t len, const AtkSpec& k) {
    const size_t N = k.steps.size(), W = m[0].size();
    auto row = [&](long i) -> std::vector<double>& { if (i < 0) i = -i; if (i >= (long)len) i = 2 * ((long)len - 1) - i; return m[(size_t)i]; };
    for (size_t s = N; s-- > 0; ) {
      const double a = coef(k, s);
      for (size_t i = (s & 1); i < len; i += 2) {
        const std::vector<double>& p = row((long)i - 1); const std::vector<double>& q = row((long)i + 1);
        std::vector<double>& d = m[i];
        for (size_t j = 0; j < W; ++j) d[j] += a * (p[j] + q[j]);
      }
    }
    std::vector<std::vector<double>> t(len);
    const double kl = k.reversible() ? 1.0 : 1.0 / (double)k.K, kh = k.reversible() ? 1.0 : (double)k.K;
    const size_t nl = (len + 1) / 2;
    for (size_t i = 0; i < len; ++i) {
      std::vector<double>& d = t[(i & 1) ? nl + i / 2 : i / 2];
      d.swap(m[i]);
      for (double& v : d) v *= (i & 1) ? kh : kl;
    }
    for (size_t i = 0; i < len; ++i) m[i].swap(t[i]);
  }
  static void synthesise(std::vector<double>& x, size_t len, const AtkSpec& k) {
    const size_t N = k.steps.size(), nl = (len + 1) / 2;
    std::vector<double> t(len);
    const double kl = k.reversible() ? 1.0 : (double)k.K, kh = k.reversible() ? 1.0 : 1.0 / (double)k.K;
    for (size_t i = 0; i < len; ++i) t[i] = (i & 1) ? x[nl + i / 2] * kh : x[i / 2] * kl;
    auto at = [&](long i) { if (i < 0) i = -i; if (i >= (long)len) i = 2 * ((long)len - 1) - i; return t[(size_t)i]; };
    for (size_t s = 0; s < N; ++s) {
      const double a = coef(k, s);
      for (size_t i = (s & 1); i < len; i += 2) t[i] -= a * (at((long)i - 1) + at((long)i + 1));
    }
    for (size_t i = 0; i < len; ++i) x[i] = t[i];
  }
  // the waveform of one coefficient of the low (hi = false) or high band of stage n on an unbounded line, carried back
  // to the input by synthesis or by the transposed analysis
  static std::vector<double> waveform(const AtkSpec& k, int n, bool hi, bool analysis) {
    const size_t N = k.steps.size(), P = 2 * (N / 2 + 1);      // even margin: every step widens the support by one
    const double K = k.reversible() ? 1.0 : (double)k.K;
    const double sl = analysis ? 1.0 / K : K, sh = analysis ? K : 1.0 / K;
    std::vector<double> x(1, 1.0);
    for (int j = n; j >= 1; --j) {
      const bool high = hi && j == n;
      std::vector<double> t(2 * x.size() + 2 * P, 0.0);
      for (size_t i = 0; i < x.size(); ++i) t[P + 2 * i + (high ? 1 : 0)] = x[i] * (high ? sh : sl);
      for (size_t s = 0; s < N; ++s) {
        const double a = analysis ? coef(k, s) : -coef(k, s);
        for (size_t i = 2 - ((s & 1) ^ (analysis ? 1 : 0)); i + 1 < t.size(); i += 2) t[i] += a * (t[i - 1] + t[i + 1]);
      }
      x.swap(t);
    }
    return x;
  }
  explicit KernelGains(const AtkSpec& k) {
    const size_t L = (size_t)16 << FINITE;
    bibo_l[0] = norm_l[0] = 1.0; bibo_h[0] = norm_h[0] = 1.0;
    std::vector<std::vector<double>> m(L, std::vector<double>(L, 0.0));
    for (size_t i = 0; i < L; ++i) m[i][i] = 1.0;
    size_t len = L;
    auto worst = [&](size_t a, size_t b) { double g = 0; for (size_t i = a; i < b; ++i) { double s = 0; for (double v : m[i]) s += std::fabs(v); g = std::max(g, s); } return g; };
    for (int n = 1; n <= FINITE; ++n) {
      analyse(m, len, k);
      bibo_l[n] = worst(0, len / 2); bibo_h[n] = worst(len / 2, len);
      len /= 2;
    }
    for (int n = 1; n <= FINITE; ++n) {
      for (int hi = 0; hi < 2; ++hi) {
        std::vector<double> x(L, 0.0);
        size_t l = L >> n;                         // length of the low band after n stages
        x[(hi ? l : 0) + l / 2] = 1.0;
        for (int j = n; j >= 1; --j) synthesise(x, L >> (j - 1), k);
        double e = 0; for (double v : x) e += v * v;
        (hi ? norm_h : norm_l)[n] = std::sqrt(e);
      }
    }
    for (int n = FINITE + 1; n <= EXACT; ++n) {
      for (int hi = 0; hi < 2; ++hi) {
        double l1 = 0, l2 = 0;
        for (double v : waveform(k, n, hi != 0, true)) l1 += std::fabs(v);
        for (double v : waveform(k, n, hi != 0, false)) l2 += v * v;
        (hi ? bibo_h : bibo_l)[n] = l1;
        (hi ? norm_h : norm_l)[n] = std::sqrt(l2);
      }
    }
    double dc = 0;
    for (double v : waveform(k, 1, false, true)) dc += v;
    const double rl = norm_l[EXACT] / norm_l[EXACT - 1], rh = norm_h[EXACT] / norm_h[EXACT - 1];
    for (int n = EXACT + 1; n <= DEPTH; ++n) {
      bibo_l[n] = bibo_l[n - 1] * std::fabs(dc); bibo_h[n] = bibo_h[n - 1] * std::fabs(dc);
      norm_l[n] = norm_l[n - 1] * rl; norm_h[n] = norm_h[n - 1] * rh;
    }
  }
};
} // namespace

//------------------------------------------------------------------------------------------
// Params
//------------------------------------------------------------------------------------------
const QuantSet& Params::quant_for(uint32_t c) const {
  for (const QuantSet& q : qcc) if (q.comp_idx == c) return q;
  return qcd;
}
QuantSet* Params::find_qcc(uint32_t c) {
  for (QuantSet& q : qcc) if (q.comp_idx == c) return &q;
  return nullptr;
}
QuantSet& Params::add_qcc(uint32_t c) {
  qcc.emplace_back();
  QuantSet& q = qcc.back();
  q.is_qcc = true; q.comp_idx = (uint16_t)c;
  return q;
}

uint32_t Params::precision(uint32_t c) const {
  uint32_t p = 0;
  if (color_transform() && c < 3) {
    for (uint32_t i = 0; i < 3; ++i) p = std::max(p, quant_for(i).largest_kmax());
  } else
    p = quant_for(c).largest_kmax();
  return p + 2;   // + sign bit + one spare bit (ojph_params.cpp:1700-1706)
}

bool Params::needs_wide() const {
  bool wide = false;
  for (uint32_t c = 0; c < num_comps(); ++c)
    if (precision(c) > 32) {
      wide = true;
      bool rev = reversible(c);
      if (color_transform() && c < 3) rev = reversible(0) && reversible(1) && reversible(2);
      if (!rev)
        fail(0x000B0001, "component %u needs %u-bit coefficients and is irreversible; the 64-bit path is built for "
             "reversible components only", c, precision(c));
    }
  return wide;
}

void Params::set_block_dims(uint32_t w, uint32_t h) {
  uint32_t lw = w ? ilog2(w) : 0, lh = h ? ilog2(h) : 0;
  if (w == 0 || w != (1u << lw) || h == 0 || h != (1u << lh) || lw < 2 || lh < 2 || lw + lh > 12)
    fail(0x00050011, "incorrect code block dimensions");
  cb_w_exp = (uint8_t)(lw - 2); cb_h_exp = (uint8_t)(lh - 2);
}

void Params::set_precincts(int n, const uint32_t* w, const uint32_t* h) {
  if (n == 0 || w == nullptr || h == nullptr) { Scod &= 0xFE; return; }
  Scod |= 1;
  for (int i = 0; i <= num_decomps; ++i) {
    uint32_t pw = w[i < n ? i : n - 1], ph = h[i < n ? i : n - 1];
    if (pw == 0 || ph == 0) fail(0x00050021, "precinct width or height cannot be 0");
    uint32_t PPx = ilog2(pw), PPy = ilog2(ph);
    if (pw != (1u << PPx) || ph != (1u << PPy))
      fail(0x00050022, "precinct width and height should be a power of 2");
    if (PPx > 15 || PPy > 15) fail(0x00050023, "precinct size is too large");
    if (i > 0 && (PPx == 0 || PPy == 0)) fail(0x00050024, "precinct size is too small");
    precinct_size[i] = (uint8_t)(PPx | (PPy << 4));
  }
}

// bands of a component with a DFS structure and / or an ATK kernel in marker order (LL, then for every resolution 1..D
// the bands its level produces), with their gains measured on the kernel (see KernelGains)
namespace {
struct Part2Band { double bibo, norm; uint32_t band; };
std::vector<Part2Band> part2_bands(uint32_t comp, const Params& p) {
  const AtkSpec& k = p.atk_of(comp);
  const KernelGains g(k);
  const uint32_t D = p.decomps(comp);
  typedef Part2Band B;
  std::vector<B> bands;
  auto count = [&](uint32_t upto, bool horz) {          // levels 1..upto that split in this direction
    uint32_t n = 0;
    for (uint32_t l = 1; l <= upto; ++l) { DfsType t = p.dwt_type(comp, l); if (t == DFS_BIDIR || t == (horz ? DFS_HORZ : DFS_VERT)) ++n; }
    return n;
  };
  {
    const uint32_t nx = count(D, true), ny = count(D, false);
    bands.push_back(B{ g.bibo_l[nx] * g.bibo_l[ny], g.norm_l[nx] * g.norm_l[ny], 0 });
  }
  for (uint32_t r = 1; r <= D; ++r) {
    const uint32_t level = D - r + 1;
    const DfsType t = p.dwt_type(comp, level);
    const bool hx = t == DFS_BIDIR || t == DFS_HORZ, vy = t == DFS_BIDIR || t == DFS_VERT;
    const uint32_t nx = count(level - 1, true), ny = count(level - 1, false), nx1 = nx + 1, ny1 = ny + 1;
    for (uint32_t b = 1; b < 4; ++b) {
      const bool bh = (b & 1) != 0, bv = (b & 2) != 0;
      if ((bh && !hx) || (bv && !vy)) continue;
      const double bx = hx ? (bh ? g.bibo_h[nx1] : g.bibo_l[nx1]) : g.bibo_l[nx], by = vy ? (bv ? g.bibo_h[ny1] : g.bibo_l[ny1]) : g.bibo_l[ny];
      const double ex = hx ? (bh ? g.norm_h[nx1] : g.norm_l[nx1]) : g.norm_l[nx], ey = vy ? (bv ? g.norm_h[ny1] : g.norm_l[ny1]) : g.norm_l[ny];
      bands.push_back(B{ bx * by, ex * ey, b });
    }
  }
  return bands;
}
} // namespace

// QCD / QCC of a component with a DFS structure and / or an ATK kernel
static void make_part2_steps(QuantSet& q, uint32_t comp, const Params& p) {
  const bool rev = p.atk_of(comp).reversible();
  if (q.qfactor != 0) fail(0x000B0020, "Qfactor needs the 9/7 kernel on a dyadic decomposition");
  typedef Part2Band B;
  const std::vector<B> bands = part2_bands(comp, p);
  q.num_subbands = (uint32_t)bands.size();
  if (rev) {
    const uint32_t Bd = q.bit_depth + ((comp < 3 && q.is_color_trans) ? 1u : 0u);
    uint32_t max_BX = 0; uint8_t tmp[97];
    for (size_t i = 0; i < bands.size(); ++i) {
      uint32_t X = (uint32_t)std::max(0.0, ceil(log(bands[i].bibo) / M_LN2 - 1e-9));
      // a band nothing has filtered (every level of the DFS leaves the resolution unsplit) still has to hold
      // -2^(B-1), whose magnitude needs B bits: the reference's zero-decomposition streams lose exactly that value
      // (K_max = B - 1 there, see ENC_CHECK_NEGZERO); a writer free to choose its exponents need not
      if (bands[i].bibo <= 1.0) X = 1;
      tmp[i] = (uint8_t)(Bd + X); max_BX = std::max(max_BX, Bd + X);
    }
    if (max_BX > 38)
      fail(0x00050151, "The specified combination of bit_depth, colour transform, and type of "
           "wavelet transform requires more than 38 bits; it requires %d bits.", max_BX);
    int guard = std::max(1, (int)max_BX - 31);
    q.Sqcd = (uint8_t)(guard << 5);
    for (size_t i = 0; i < bands.size(); ++i) q.SP[i] = (uint16_t)(uint8_t)((uint8_t)(tmp[i] - guard) << 3);
  } else {
    static const double arr[4] = { 1.0, 2.0, 2.0, 4.0 };
    if (q.base_delta == -1.0f) q.base_delta = 1.0f / (float)(1u << std::min(16u, q.bit_depth));
    double worst = 1.0;
    for (const B& b : bands) worst = std::max(worst, b.bibo / arr[b.band]);
    int guard = std::max(1, (int)ceil(log(worst) / M_LN2 - 1e-9));
    if (guard > 7) fail(0x000B0021, "the transformation kernel amplifies by more than 7 guard bits");
    q.Sqcd = (uint8_t)((guard << 5) | 0x2);
    for (size_t i = 0; i < bands.size(); ++i)
      q.SP[i] = pack_step((float)((double)q.base_delta / (bands[i].norm * arr[bands[i].band])));
  }
}

std::vector<double> Params::band_energy_gains(uint32_t c) const {
  std::vector<double> g;
  if (is_part2(c)) {
    for (const Part2Band& b : part2_bands(c, *this)) g.push_back(b.norm * b.norm);
    return g;
  }
  // the 1-D synthesis gains set_rev_quant / set_irrev_quant weigh the bands with
  const bool rev = wavelet_of(c) == DWT_REV53;
  const uint32_t D = decomps(c);
  const double gl = energy_gain_l(D, rev);
  g.push_back(gl * gl * gl * gl);
  for (uint32_t d = D; d > 0; --d) {
    const double l = energy_gain_l(d, rev), h = energy_gain_h(d - 1, rev);
    g.push_back(h * l * h * l); g.push_back(l * h * l * h); g.push_back(h * h * h * h);
  }
  return g;
}

static void make_quant_steps(QuantSet& q, uint32_t comp, const Params& p) {
  if (q.is_init) fail(0x00040001, "Quantization step sizes already initialized.");
  q.is_init = true;
  q.num_decomps = p.decomps(comp);              // the component's COC when it has one (:1432-1460)
  q.bit_depth = p.comps[comp].bit_depth;
  q.is_signed = p.comps[comp].is_signed;
  q.is_color_trans = p.color_transform();
  q.wavelet = p.wavelet_of(comp);
  q.sx = p.comps[comp].dx; q.sy = p.comps[comp].dy;
  q.num_subbands = 1 + 3 * q.num_decomps;
  if (p.is_part2(comp)) { make_part2_steps(q, comp, p); return; }
  if (q.wavelet == DWT_REV53)
    q.set_rev_quant(q.num_decomps, q.bit_depth, comp < 3 ? q.is_color_trans : false);
  else {
    if (q.base_delta == -1.0f) {
      uint32_t t = std::min(16u, q.bit_depth);
      q.base_delta = 1.0f / (float)(1 << t);
    }
    q.set_irrev_quant(q.num_decomps);
  }
}

uint32_t Params::cap_magb() const {
  // MAGB over QCD and every QCC (ojph_params.cpp:1615)
  uint32_t B = 0;
  const bool part2 = any_part2();
  auto magb = [&](const QuantSet& q) {
    uint32_t nd = (q.num_subbands - 1) / 3;
    for (uint32_t i = 0; i < q.num_subbands; ++i) {
      uint32_t t;
      if (part2) { B = std::max(B, q.kmax_at(i)); continue; }      // no dyadic level to take the band's gain from
      if ((q.Sqcd & 0x1F) == 0) t = ((uint32_t)(q.SP[i] & 0xFF) >> 3) + q.guard_bits() - 1u;
      else { uint32_t nb = nd - (i ? (i - 1) / 3 : 0); t = (uint32_t)(q.SP[i] >> 11) + q.guard_bits() - nb; }
      B = std::max(B, t);
    }
  };
  magb(qcd);
  for (const QuantSet& q : qcc) magb(q);
  return (B <= 8) ? 0 : (B < 28 ? B - 8 : 13 + (B >> 2));
}

void Params::finalize_for_encode() {
  // tile size 0x0 => one tile covering the image (ojph_codestream_local.cpp:562-570)
  if (XTsiz == 0 && YTsiz == 0) { XTsiz = Xsiz + XOsiz; YTsiz = Ysiz + YOsiz; }
  // SIZ validity (ojph_params_local.h:234-248)
  if (Xsiz == 0 || Ysiz == 0 || XTsiz == 0 || YTsiz == 0)
    fail(0x00040001, "Image extent and/or tile size cannot be zero");
  if (XTOsiz > XOsiz || YTOsiz > YOsiz)
    fail(0x00040002, "Tile offset has to be smaller than the image offset");
  if (XTsiz + XTOsiz <= XOsiz || YTsiz + YTOsiz <= YOsiz)
    fail(0x00040003, "The top left tile must intersect with the image");
  if (Xsiz <= XOsiz || Ysiz <= YOsiz)
    fail(0x00040004, "The image extent must be larger than the image offset");
  uint32_t nc = num_comps();
  if (nc == 0 || nc > 16384) fail(0x00040005, "wrong number of components");
  // COD validity (ojph_params_local.h:450-513)
  if (mc_trans == 1 && nc < 3)
    fail(0x00040011, "color transform can only be employed when the image has 3 or more "
         "color components");
  if (mc_trans == 1) {
    for (uint32_t i = 1; i < 3; ++i) {
      if (comps[i].dx != comps[0].dx || comps[i].dy != comps[0].dy)
        fail(0x00040012, "when color transform is used, the first 3 colour components must "
             "have the same downsampling factor.");
      if (comps[i].bit_depth != comps[0].bit_depth)
        fail(0x00040014, "when color transform is used, the first 3 colour components must "
             "have the same bit depth.");
      if (comps[i].is_signed != comps[0].is_signed)
        fail(0x00040015, "when color transform is used, the first 3 colour components must "
             "have the same signedness (signed or unsigned).");
    }
  }
  if (prog_order == PO_RPCL || prog_order == PO_PCRL)
    for (uint32_t i = 0; i < nc; ++i)
      if ((comps[i].dx & (comps[i].dx - 1)) || (comps[i].dy & (comps[i].dy - 1)))
        fail(0x00040013, "For RPCL and PCRL progression orders,component downsampling "
             "factors have to be powers of 2");

  // Part 2 structures asked of the encoder: one DFS (index 1) and / or one ATK (index 2) shared by every component
  // through its COC -- the only place a DFS index can go (param_cod::is_dfs_defined, ojph_params_local.h:613-618)
  if (!enc_dfs.empty() || enc_atk_set) {
    if (!enc_dfs.empty()) {
      if (enc_dfs.size() > 32) fail(0x000B0022, "at most 32 decomposition levels can be described");
      DfsSpec d; d.Sdfs = 1; d.Ids = (uint8_t)enc_dfs.size();
      for (size_t i = 0; i < enc_dfs.size(); ++i) {
        if (enc_dfs[i] > 3) fail(0x000B0022, "decomposition level type must be 0 (no split), 1 (both ways), 2 (horizontal) or 3 (vertical)");
        d.Ddfs[i >> 2] = (uint8_t)(d.Ddfs[i >> 2] | (enc_dfs[i] << (6 - 2 * (i & 3))));
      }
      dfs.assign(1, d);
      Rsiz |= 0x8080;
    }
    if (enc_atk_set) {
      AtkSpec a = enc_atk;
      const bool rev = a.reversible();
      if (a.steps.empty() || a.steps.size() > 255) fail(0x000B0023, "a transformation kernel needs 1..255 lifting steps");
      // whole-sample symmetric, even-indexed first step, symmetric extension; 16-bit integers or floats
      a.Satk = (uint16_t)(2u | (rev ? 0x1100u : 0x0200u) | 0x0800u | 0x4000u);
      if (rev) for (const AtkStep& t : a.steps) if (t.e > 30) fail(0x000B0023, "lifting step down-shift beyond 30 bits");
      atk.assign(1, a);
      Rsiz |= 0x8020;
    }
    for (uint32_t c = 0; c < nc; ++c) {
      CodStyle* st = const_cast<CodStyle*>(find_coc(c));
      if (st == nullptr) {
        CodStyle n; n.comp_idx = (uint16_t)c; n.Scoc = (uint8_t)(Scod & 1); n.num_decomps = num_decomps; n.cb_w_exp = cb_w_exp;
        n.cb_h_exp = cb_h_exp; n.block_style = block_style; n.wavelet = wavelet;
        memcpy(n.precinct_size, precinct_size, sizeof(n.precinct_size));
        coc.push_back(n); st = &coc.back();
      }
      if (!enc_dfs.empty()) {
        if (st->num_decomps != num_decomps) fail(0x000B0024, "a decomposition structure needs the same number of levels in every component");
        st->dfs_idx = 1;
      }
      if (enc_atk_set) st->wavelet = 2;
    }
  }

  // QCD / QCC (param_qcd::check_validity, ojph_params.cpp:1359-1431)
  for (QuantSet& q : qcc) q.enabled = q.comp_idx < nc;
  uint32_t qcd_comp = 0;
  // the first component that uses COD (no COC) and has no QCC (ojph_params.cpp:1367-1377)
  for (uint32_t c = 0; c < nc; ++c) if (find_coc(c) == nullptr && find_qcc(c) == nullptr) { qcd_comp = c; break; }
  if (qcd.qfactor != 0) {
    for (uint32_t i = 0; i < nc; ++i) {
      if (find_qcc(i) == nullptr) {
        QuantSet& q = add_qcc(i);
        q.qfactor = qcd.qfactor;
        q.ctype = (nc < 3) ? 0 : (int)(i < 3u ? i : 0u);
      }
    }
  }
  make_quant_steps(qcd, qcd_comp, *this);
  for (uint32_t c = 0; c < nc; ++c) {
    QuantSet* q = find_qcc(c);
    if (q == nullptr) {
      bool needed = qcd.num_decomps != decomps(c) || qcd.bit_depth != comps[c].bit_depth ||
                    qcd.is_signed != comps[c].is_signed ||
                    qcd.is_color_trans != color_transform() || qcd.wavelet != wavelet_of(c);
      if (!needed) continue;
      QuantSet& nq = add_qcc(c);
      nq.base_delta = qcd.base_delta;
      q = &nq;
    }
    make_quant_steps(*q, c, *this);
  }

  // CAP (ojph_params_local.h:982-998)
  if (reversible()) Ccap0 &= 0xFFDF; else Ccap0 |= 0x0020;
  Ccap0 &= 0xFFE0;
  Ccap0 = (uint16_t)(Ccap0 | (uint16_t)cap_magb());

  (void)needs_wide();        // 64-bit coefficients: reversible components only (refuses the rest)

  nlt_check_validity();
  if (profile) check_profile();

  // tile-part division rules (ojph_codestream_local.cpp:583-621)
  if ((prog_order == PO_LRCP || prog_order == PO_RLCP) && tilepart_div == TP_COMP)
    tilepart_div |= TP_RES;
  if (prog_order == PO_RPCL && (tilepart_div & TP_COMP)) tilepart_div &= ~(uint32_t)TP_COMP;
  if (prog_order == PO_PCRL && tilepart_div != 0) tilepart_div = 0;
  if (prog_order == PO_CPRL && (tilepart_div & TP_RES)) tilepart_div &= ~(uint32_t)TP_RES;
  if (planar == -1) planar = color_transform() ? 1 : 0;
  else if (planar == 1 && color_transform())
    fail(0x00030021, "the planar interface option cannot be used when colour transform is "
         "employed");
}

//------------------------------------------------------------------------------------------
// NLT: type 3 (two's complement <-> sign-magnitude mapping of signed samples) is the only
// non-linearity the reference implements (ojph_params.cpp:2176-2190)
//------------------------------------------------------------------------------------------
void Params::set_nonlinear_transform(uint32_t comp, uint32_t type) {
  if (type != 0 && type != 3)
    fail(0x00050171, "Nonliearities other than type 0 (No Nonlinearity) or type  3 (Binary Binary Complement to "
         "Sign Magnitude Conversion) are not supported yet");
  NltEntry* e = nullptr;
  if (comp == 0xFFFF) e = &nlt_all;
  else {
    for (NltEntry& x : nlt) if (x.comp_idx == comp) e = &x;
    if (e == nullptr) { nlt.push_back(NltEntry()); e = &nlt.back(); e->comp_idx = (uint16_t)comp; }
  }
  e->Tnlt = (uint8_t)type; e->enabled = true;
}

void Params::nlt_check_validity() {          // param_nlt::check_validity, ojph_params.cpp:2087-2173
  if (!nlt_any()) return;
  const uint32_t nc = num_comps();
  auto own = [&](uint32_t c) -> NltEntry* { for (NltEntry& x : nlt) if (x.comp_idx == c) return &x; return nullptr; };
  auto bd_of = [&](uint32_t c) { return (uint8_t)((comps[c].bit_depth - 1) | (comps[c].is_signed ? 0x80 : 0)); };
  if (nlt_all.enabled && nlt_all.Tnlt == 0) nlt_all.enabled = false;
  if (nlt_all.enabled && nlt_all.Tnlt == 3) {
    bool all_same = true;
    uint32_t bit_depth = 0; bool is_signed = false;
    for (uint32_t c = 0; c < nc; ++c) {
      NltEntry* e = own(c);
      if (e == nullptr || !e->enabled) {
        if (bit_depth != 0) all_same = all_same && bit_depth == comps[c].bit_depth && is_signed == comps[c].is_signed;
        else { bit_depth = comps[c].bit_depth; is_signed = comps[c].is_signed; }
      } else e->BDnlt = bd_of(c);
    }
    if (all_same && bit_depth != 0) nlt_all.BDnlt = (uint8_t)((bit_depth - 1) | (is_signed ? 0x80 : 0));
    else if (!all_same) {
      nlt_all.enabled = false;
      for (uint32_t c = 0; c < nc; ++c) {
        NltEntry* e = own(c);
        if (e == nullptr || !e->enabled) {
          if (e == nullptr) { nlt.push_back(NltEntry()); e = &nlt.back(); e->comp_idx = (uint16_t)c; }
          e->enabled = true; e->Tnlt = 3; e->BDnlt = bd_of(c);
        }
      }
    }
  } else {
    for (uint32_t c = 0; c < nc; ++c) { NltEntry* e = own(c); if (e && e->enabled) e->BDnlt = bd_of(c); }
  }
  for (NltEntry& e : nlt) if (e.enabled && e.comp_idx >= nc) e.enabled = false;   // trim_non_existing_components
  if (nlt_any()) Rsiz |= 0x8000 | 0x0200;    // RSIZ_EXT_FLAG | RSIZ_NLT_FLAG
}

uint32_t Params::nlt_type(uint32_t c) const {  // get_nonlinear_transform + the check of ojph_tile.cpp:292-300
  const NltEntry* e = nullptr;
  for (const NltEntry& x : nlt) if (x.comp_idx == c && x.enabled) e = &x;
  if (e == nullptr && nlt_all.enabled) e = &nlt_all;
  if (e == nullptr) return 0;
  uint32_t bd = (uint32_t)(e->BDnlt & 0x7F) + 1; if (bd > 38) bd = 38;
  const bool is = (e->BDnlt & 0x80) != 0;
  if (bd != comps[c].bit_depth || is != comps[c].is_signed)
    fail(0x000300A1, "Mismatch between Ssiz (bit_depth = %d, is_signed = %s) from SIZ marker segment, and BDnlt "
         "(bit_depth = %d, is_signed = %s) from NLT marker segment, for component %d", comps[c].bit_depth,
         comps[c].is_signed ? "True" : "False", bd, is ? "True" : "False", c);
  return e->Tnlt == 3 ? 3u : 0u;
}

//------------------------------------------------------------------------------------------
// IMF / BROADCAST profiles: parameter rules only -- but they also switch TLM on and force tile-part
// division by components, so they change the bytes (check_imf_validity :292-455,
// check_broadcast_validity :458-535)
//------------------------------------------------------------------------------------------
void Params::check_profile() {
  const bool imf = profile == 1;
  const char* nm = imf ? "IMF" : "broadcast";
  const uint32_t base = imf ? 0x000300C0u : 0x000300B0u;       // the reference's error code blocks
  const uint32_t nc = num_comps();
  const bool rev = reversible();
  // (the reference's frame-size tests for the 2K / 4K / 8K IMF levels are written `flag &= true` and never
  // reject anything, :302-330; the levels only differ in the decomposition ceilings below)
  bool lvl[3] = { true, true, true };
  if (XOsiz || YOsiz) fail(base + (imf ? 3 : 1), "For %s profile, image offset (XOsiz, YOsiz) has to be 0.", nm);
  if (XTOsiz || YTOsiz) fail(base + (imf ? 4 : 2), "For %s profile, tile offset (XTOsiz, YTOsiz) has to be 0.", nm);
  if (nc > (imf ? 3u : 4u))
    fail(base + (imf ? 5 : 3), "For %s profile, the number of components has to be less  or equal to %d", nm, imf ? 3 : 4);
  bool plain = true, x422 = true;                                // 4:4:4, or 4:2:2 on components 1 and 2
  for (uint32_t c = 0; c < nc; ++c) {
    if (comps[c].dy != 1) plain = x422 = false;
    if (comps[c].dx != 1) plain = false;
    if (comps[c].dx != ((c == 1 || c == 2) ? 2u : 1u)) x422 = false;
  }
  if (!plain && !x422)
    fail(base + (imf ? 6 : 4), "For %s profile, either no component downsampling is used, or the x-dimension of the 2nd "
         "and 3rd components is downsampled by 2.", nm);
  for (uint32_t c = 0; c < nc; ++c)
    if (comps[c].bit_depth < 8 || comps[c].bit_depth > (imf ? 16u : 12u) || comps[c].is_signed)
      fail(base + (imf ? 7 : 5), "For %s profile, compnent bit_depth has to be between 8 and %d bits inclusively, and the "
           "samples must be unsigned", nm, imf ? 16 : 12);
  if (imf) {
    if (log_cb_w() != 5 || log_cb_h() != 5)
      fail(0x000300C8, "For IMF profile, codeblock dimensions are restricted. Use \"-block_size {32,32}\" at the commandline");
  } else {
    if (num_decomps == 0 || num_decomps > 5)
      fail(0x000300B6, "For broadcast profile, number of decompositions has to be between1 and 5 inclusively.");
    if (log_cb_w() < 5 || log_cb_w() > 7)
      fail(0x000300B7, "For broadcast profile, codeblock dimensions are restricted such that codeblock width has to be "
           "either 32, 64, or 128.");
    if (log_cb_h() < 5 || log_cb_h() > 7)
      fail(0x000300B8, "For broadcast profile, codeblock dimensions are restricted such that codeblock height has to be "
           "either 32, 64, or 128.");
  }
  // precincts: 128x128 at the coarsest resolution, 256x256 above (the reference's loop keeps only the test of
  // the LAST resolution when there is more than one -- reproduced)
  bool pz = log_pp_w(0) == 7 && log_pp_h(0) == 7;
  for (uint32_t r = 1; r <= num_decomps; ++r) pz = log_pp_w(r) == 8 && log_pp_h(r) == 8;
  if (!pz) fail(base + 9, "For %s profile, precinct sizes are restricted. Use \"-precincts {128,128},{256,256}\" at the commandline", nm);
  if (prog_order != PO_CPRL)
    fail(base + 10, "For %s profile, the CPRL progression order must be used. Use \"-prog_order CPRL\".", nm);
  const uint32_t ntiles = div_ceil(Xsiz, XTsiz) * div_ceil(Ysiz, YTsiz);
  if (imf) {
    for (int i = 0; i < 3; ++i) lvl[i] = num_decomps <= 5u + (uint32_t)i;
    if (num_decomps == 0 || !(lvl[0] || lvl[1] || lvl[2]))
      fail(0x000300CB, "Number of decompositions does not match the IMF profile dictated by wavelet reversibility and "
           "image dimensions.");
    if (ntiles > 1) {
      if (!rev) fail(0x000300CC, "Lossy IMF profile must have one tile.");
      // square tiles of 1024 / 2048 / 4096, and enough tile width for the decomposition count
      const uint32_t tw = XTsiz, th = YTsiz;
      auto deep = [&](int top) {        // top: how many (width, levels) pairs the level allows
        static const uint32_t w[4] = { 1024, 2048, 4096, 8192 };
        for (int i = 0; i <= top; ++i) if (tw >= w[i] && num_decomps <= 4u + (uint32_t)i) return true;
        return false;
      };
      auto square = [&](int top) { for (int i = 0; i <= top; ++i) if (tw == (1024u << i) && th == (1024u << i)) return true; return false; };
      const bool ok2 = lvl[0] && square(0) && deep(1), ok4 = lvl[1] && square(1) && deep(2), ok8 = lvl[2] && square(2) && deep(3);
      if (!ok2 && !ok4 && !ok8)
        fail(0x000300CD, "Number of decompositions does not match the IMF profile dictated by wavelet reversibility and "
             "image dimensions and tiles.");
    }
  } else if (ntiles != 1 && ntiles != 4)
    fail(0x000300BB, "The broadcast profile can only have 1 or 4 tiles");
  need_tlm = true;
  tilepart_div = TP_COMP;                   // (the reference warns when it has to correct this)
}

static void write_quant(std::vector<uint8_t>& o, const QuantSet& q, uint32_t nc) {
  int irrev = q.Sqcd & 0x1F;
  uint32_t L = q.is_qcc ? (4 + (nc < 257 ? 0 : 1)) : 3;
  L += (irrev == 0 ? 1 : 2) * q.num_subbands;
  put_u16(o, q.is_qcc ? M_QCC : M_QCD);
  put_u16(o, L);
  if (q.is_qcc) { if (nc < 257) put_u8(o, q.comp_idx); else put_u16(o, q.comp_idx); }
  put_u8(o, q.Sqcd);
  for (uint32_t i = 0; i < q.num_subbands; ++i)
    if (irrev == 0) put_u8(o, q.SP[i] & 0xFF); else put_u16(o, q.SP[i]);
}

void Params::write_main_header(std::vector<uint8_t>& o, const char* const* comments,
                               const uint32_t* comment_lens, uint32_t n_comments) const {
  uint32_t nc = num_comps();
  put_u16(o, M_SOC);
  // SIZ
  put_u16(o, M_SIZ); put_u16(o, 38 + 3 * nc); put_u16(o, Rsiz);
  put_u32(o, Xsiz); put_u32(o, Ysiz); put_u32(o, XOsiz); put_u32(o, YOsiz);
  put_u32(o, XTsiz); put_u32(o, YTsiz); put_u32(o, XTOsiz); put_u32(o, YTOsiz);
  put_u16(o, nc);
  for (uint32_t c = 0; c < nc; ++c) {
    put_u8(o, (uint32_t)(comps[c].bit_depth - 1) + (comps[c].is_signed ? 0x80u : 0u));
    put_u8(o, comps[c].dx); put_u8(o, comps[c].dy);
  }
  // CAP
  put_u16(o, M_CAP); put_u16(o, 8); put_u32(o, Pcap); put_u16(o, Ccap0);
  // COD
  put_u16(o, M_COD);
  put_u16(o, 12 + ((Scod & 1) ? 1 + num_decomps : 0));
  put_u8(o, Scod); put_u8(o, prog_order); put_u16(o, num_layers); put_u8(o, mc_trans);
  put_u8(o, num_decomps); put_u8(o, cb_w_exp); put_u8(o, cb_h_exp); put_u8(o, block_style);
  put_u8(o, wavelet);
  if (Scod & 1) for (int i = 0; i <= num_decomps; ++i) put_u8(o, precinct_size[i]);
  // COC, in creation order (param_cod::write_coc / internal_write_coc, ojph_params.cpp:1081-1143)
  for (const CodStyle& c : coc) {
    if (c.comp_idx >= nc) continue;
    put_u16(o, M_COC);
    const uint32_t nd = c.dfs_idx >= 0 ? num_decomps : c.num_decomps;
    put_u16(o, (nc < 257 ? 9u : 10u) + ((c.Scoc & 1) ? 1u + nd : 0u));
    if (nc < 257) put_u8(o, c.comp_idx); else put_u16(o, c.comp_idx);
    put_u8(o, c.Scoc); put_u8(o, c.dfs_idx >= 0 ? (0x80u | (uint32_t)c.dfs_idx) : c.num_decomps); put_u8(o, c.cb_w_exp); put_u8(o, c.cb_h_exp);
    put_u8(o, c.block_style); put_u8(o, c.wavelet);
    if (c.Scoc & 1) for (uint32_t i = 0; i <= nd; ++i) put_u8(o, c.precinct_size[i]);
  }
  // QCD, QCC
  write_quant(o, qcd, nc);
  for (const QuantSet& q : qcc) if (q.enabled) write_quant(o, q, nc);
  // DFS / ATK (T.801 A.3.? layouts as param_dfs::read / param_atk::read expect them, ojph_params.cpp:2596-2645, :2770-2867)
  for (const DfsSpec& d : dfs) {
    const uint32_t nb = (d.Ids + 3u) / 4u;
    put_u16(o, M_DFS); put_u16(o, 5 + nb); put_u16(o, d.Sdfs); put_u8(o, d.Ids);
    for (uint32_t i = 0; i < nb; ++i) put_u8(o, d.Ddfs[i]);
  }
  for (const AtkSpec& a : atk) {
    const bool rev = a.reversible();
    const uint32_t cs = a.coeff_type() == 0 ? 1u : a.coeff_type() == 1 ? 2u : 4u;
    auto put_coef = [&](float f, int iv) {
      if (rev) { if (cs == 1) put_u8(o, (uint32_t)(uint8_t)(int8_t)iv); else put_u16(o, (uint32_t)(uint16_t)(int16_t)iv); }
      else { uint32_t u; memcpy(&u, &f, 4); put_u32(o, u); }
    };
    const uint32_t n = (uint32_t)a.steps.size();
    put_u16(o, M_ATK);
    put_u16(o, 5 + (rev ? n * (4 + cs) : cs + n * (1 + cs)));
    put_u16(o, a.Satk);
    if (!rev) put_coef(a.K, 0);
    put_u8(o, n);
    for (const AtkStep& t : a.steps) {
      if (rev) { put_u8(o, t.e); put_u16(o, (uint32_t)(uint16_t)t.b); put_u8(o, 1); put_coef(0.f, t.a); }
      else { put_u8(o, 1); put_coef(t.A, 0); }
    }
  }
  // NLT: the default entry, then the per-component ones in creation order (param_nlt::write, :2210-2235)
  auto put_nlt = [&](const NltEntry& e) {
    if (!e.enabled) return;
    put_u16(o, M_NLT); put_u16(o, 6); put_u16(o, e.comp_idx); put_u8(o, e.BDnlt); put_u8(o, e.Tnlt);
  };
  put_nlt(nlt_all);
  for (const NltEntry& e : nlt) put_nlt(e);
  // COM: library signature, needed for byte-identical output
  // (ojph_codestream_local.cpp:668-686)
  static const char sig[] = "OpenJPH Ver 0.31.0.";
  put_u16(o, M_COM); put_u16(o, (uint32_t)strlen(sig) + 4); put_u16(o, 1);
  o.insert(o.end(), sig, sig + strlen(sig));
  for (uint32_t i = 0; i < n_comments; ++i) {
    put_u16(o, M_COM); put_u16(o, comment_lens[i] + 4); put_u16(o, 1);
    o.insert(o.end(), comments[i], comments[i] + comment_lens[i]);
  }
  for (const Comment& c : this->comments) {  // write_headers(file, comments, num_comments), :688-706
    put_u16(o, M_COM); put_u16(o, (uint32_t)c.data.size() + 4); put_u16(o, c.Rcom);
    o.insert(o.end(), c.data.begin(), c.data.end());
  }
}

//------------------------------------------------------------------------------------------
// main-header parsing
//------------------------------------------------------------------------------------------
namespace {
struct Reader {
  const uint8_t* d; size_t n, pos;
  bool has(size_t k) const { return pos + k <= n; }
  uint32_t u8() { if (!has(1)) fail(0x00030051, "File ended before finding a tile segment"); return d[pos++]; }
  uint32_t u16() { uint32_t a = u8(); return (a << 8) | u8(); }
  uint32_t u32() { uint32_t a = u16(); return (a << 16) | u16(); }
};

void read_quant(Reader& r, QuantSet& q, bool is_qcc, uint32_t nc) {
  uint32_t L = r.u16();
  uint32_t hdr = 3;
  q.is_qcc = is_qcc;
  if (is_qcc) {
    if (nc < 257) { q.comp_idx = (uint16_t)r.u8(); hdr = 4; }
    else { q.comp_idx = (uint16_t)r.u16(); hdr = 5; }
  }
  q.Sqcd = (uint8_t)r.u8();
  int style = q.Sqcd & 0x1F;
  if (style == 0) {
    q.num_subbands = L - hdr;
    if (q.num_subbands == 0 || q.num_subbands > 97)
      fail(0x00050083, "wrong Lqcd value of %d in QCD marker", L);
    for (uint32_t i = 0; i < q.num_subbands; ++i) q.SP[i] = (uint16_t)r.u8();
  } else if (style == 2) {
    q.num_subbands = (L - hdr) / 2;
    if (q.num_subbands == 0 || q.num_subbands > 97 || L != hdr + 2 * q.num_subbands)
      fail(0x00050086, "wrong Lqcd value of %d in QCD marker", L);
    for (uint32_t i = 0; i < q.num_subbands; ++i) q.SP[i] = (uint16_t)r.u16();
  } else if (style == 1)
    fail(0x00050089, "Scalar derived quantization is not supported yet in QCD marker");
  else
    fail(0x00050088, "wrong Sqcd value in QCD marker");
  q.is_init = true;
}
} // namespace

size_t Params::read_main_header(const uint8_t* data, size_t len) {
  Reader r{ data, len, 0 };
  // find SOC then SIZ (find_marker, ojph_codestream_local.cpp:706-730: after a 0xFF the next byte is consumed
  // whether it matches or not; read_headers ignores a failed search, so a stream without SOC / SIZ ends up
  // in param_siz::read at the end of the data, :855-857)
  auto find = [&](uint16_t m) {
    while (r.pos < r.n) {
      if (r.d[r.pos++] != 0xFF) continue;
      if (r.pos >= r.n) return false;
      if (r.d[r.pos++] == (m & 0xFF)) return true;
    }
    return false;
  };
  if (!find(M_SOC) || !find(M_SIZ) || !r.has(2)) fail(0x00050041, "error reading SIZ marker");
  // SIZ
  {
    uint32_t L = r.u16();
    int nc = ((int)L - 38) / 3;
    if ((int)L != 38 + 3 * nc) fail(0x00050042, "error in SIZ marker length");
    Rsiz = (uint16_t)r.u16();
    if ((Rsiz & 0x4000) == 0) fail(0x00050044, "Rsiz bit 14 is not set (this is not a JPH file)");
    Xsiz = r.u32(); Ysiz = r.u32(); XOsiz = r.u32(); YOsiz = r.u32();
    XTsiz = r.u32(); YTsiz = r.u32(); XTOsiz = r.u32(); YTOsiz = r.u32();
    uint32_t C = r.u16();
    if ((int)C != nc) fail(0x0005004E, "Csiz does not match the SIZ marker size");
    if (C == 0) fail(0x0005004F, "Wrong Csiz value of 0 in SIZ marker segment");
    comps.resize(C);
    for (uint32_t c = 0; c < C; ++c) {
      uint32_t s = r.u8(), xr = r.u8(), yr = r.u8();
      if ((s & 0x7F) > 37) fail(0x00050054, "Wrong SIZ-SSiz value of %d", s);
      if (xr == 0) fail(0x00050055, "Wrong SIZ-XRsiz value of %d", xr);
      if (yr == 0) fail(0x00050056, "Wrong SIZ-YRsiz value of %d", yr);
      comps[c].bit_depth = (uint8_t)((s & 0x7F) + 1);
      comps[c].is_signed = (s & 0x80) != 0;
      comps[c].dx = (uint8_t)xr; comps[c].dy = (uint8_t)yr;
    }
    if (Xsiz == 0 || Ysiz == 0 || XTsiz == 0 || YTsiz == 0)
      fail(0x00040001, "Image extent and/or tile size cannot be zero");
    if (XTOsiz > XOsiz || YTOsiz > YOsiz)
      fail(0x00040002, "Tile offset has to be smaller than the image offset");
    if (XTsiz + XTOsiz <= XOsiz || YTsiz + YTOsiz <= YOsiz)
      fail(0x00040003, "The top left tile must intersect with the image");
    if (Xsiz <= XOsiz || Ysiz <= YOsiz)
      fail(0x00040004, "The image extent must be larger than the image offset");
  }
  int received = 0;
  qcc.clear(); coc.clear(); nlt.clear(); nlt_all = NltEntry(); dfs.clear(); atk.clear();
  for (;;) {
    // scan to the next 0xFF xx marker of interest (the reference skips unknown bytes too)
    if (r.pos + 1 >= r.n) fail(0x00030051, "File ended before finding a tile segment");
    if (r.d[r.pos] != 0xFF) { ++r.pos; continue; }
    uint16_t m = (uint16_t)(0xFF00 | r.d[r.pos + 1]);
    bool known = m == M_CAP || m == M_PRF || m == M_CPF || m == M_COD || m == M_COC || m == M_QCD ||
                 m == M_QCC || m == M_RGN || m == M_POC || m == M_PPM || m == M_TLM || m == M_PLM ||
                 m == M_CRG || m == M_COM || m == M_DFS || m == M_ATK || m == M_NLT || m == M_SOT;
    if (!known) { ++r.pos; continue; }
    if (m == M_SOT) break;
    r.pos += 2;
    if (m == M_CAP) {
      uint32_t L = r.u16();
      Pcap = r.u32();
      if (Pcap & 0xFFFDFFFF) fail(0x00050063, "error Pcap in CAP has options that are not supported");
      if ((Pcap & 0x00020000) == 0)
        fail(0x00050064, "error Pcap should have its 15th MSB set, Pcap^15.  This is not a JPH file");
      Ccap0 = (uint16_t)r.u16();
      if (L != 8) fail(0x00050066, "error in CAP marker length");
    } else if (m == M_COD) {
      uint32_t L = r.u16();
      Scod = (uint8_t)r.u8(); prog_order = (uint8_t)r.u8(); num_layers = (uint16_t)r.u16();
      mc_trans = (uint8_t)r.u8(); num_decomps = (uint8_t)r.u8(); cb_w_exp = (uint8_t)r.u8();
      cb_h_exp = (uint8_t)r.u8(); block_style = (uint8_t)r.u8(); wavelet = (uint8_t)r.u8();
      if (num_decomps > 32 || cb_w_exp > 8 || cb_h_exp > 8 || cb_w_exp + cb_h_exp > 8 ||
          (block_style & 0x40) != 0x40 || (block_style & 0xB7) != 0x00)
        fail(0x0005007D, "wrong settings in a COD-SPcod parameter");
      if (Scod & 1)
        for (int i = 0; i <= num_decomps; ++i) {
          precinct_size[i] = (uint8_t)r.u8();
          if (i && ((precinct_size[i] & 0xF) == 0 || (precinct_size[i] >> 4) == 0))
            fail(0x0005007F, "Precinct width or height for resolutions other than the coarsest "
                 "must be larger than 1");
        }
      if (L != 12u + ((Scod & 1) ? 1u + num_decomps : 0u)) fail(0x0005007C, "error in COD segment length");
      if (num_layers != 1)
        fail(0x00030053, "The current implementation supports 1 quality layer only.  This "
             "codestream has %d quality layers", num_layers);
      if (prog_order > 4) fail(0x0005007D, "wrong settings in a COD-SPcod parameter");
      received |= 1;
    } else if (m == M_QCD) {
      read_quant(r, qcd, false, num_comps());
      received |= 2;
    } else if (m == M_QCC) {
      QuantSet q;
      read_quant(r, q, true, num_comps());
      if (q.comp_idx >= num_comps())
        fail(0x00030054, "The codestream carries a QCC marker segment for a component indexed "
             "by %d, which is more than the allowed index number, since the codestream has %d "
             "components", q.comp_idx, num_comps());
      if (find_qcc(q.comp_idx))
        fail(0x00030055, "The codestream has two QCC marker segments for one component of "
             "index %d", q.comp_idx);
      qcc.push_back(q);
    } else if (m == M_COC) {                    // param_cod::read_coc, ojph_params.cpp:1207-1290
      uint32_t L = r.u16();
      const uint32_t nc = num_comps();
      CodStyle c;
      c.comp_idx = (uint16_t)(nc < 257 ? r.u8() : r.u16());
      c.Scoc = (uint8_t)r.u8(); c.num_decomps = (uint8_t)r.u8(); c.cb_w_exp = (uint8_t)r.u8();
      c.cb_h_exp = (uint8_t)r.u8(); c.block_style = (uint8_t)r.u8(); c.wavelet = (uint8_t)r.u8();
      if (c.comp_idx >= nc)
        fail(0x00030056, "The codestream carries a COC marker segment for a component indexed by %d, which is "
             "more than the allowed index number, since the codestream has %d components", c.comp_idx, nc);
      if (find_coc(c.comp_idx))
        fail(0x00030057, "The codestream has two COC marker segments for one component of index %d", c.comp_idx);
      // a decomposition byte with its top bit set names a DFS marker segment; the level count is then the COD's as
      // read so far (is_dfs_defined / get_num_decompositions, ojph_params_local.h:503-518, :613-618)
      if (c.num_decomps & 0x80) { c.dfs_idx = c.num_decomps & 0xF; c.num_decomps = num_decomps; }
      if (c.num_decomps > 32 || c.cb_w_exp > 8 || c.cb_h_exp > 8 || c.cb_w_exp + c.cb_h_exp > 8 ||
          (c.block_style & 0x40) != 0x40 || (c.block_style & 0xB7) != 0x00)
        fail(0x0005012D, "wrong settings in a COC-SPcoc parameter");
      if (c.Scoc & 1)
        for (int i = 0; i <= c.num_decomps; ++i) {
          c.precinct_size[i] = (uint8_t)r.u8();
          if (i && ((c.precinct_size[i] & 0xF) == 0 || (c.precinct_size[i] >> 4) == 0))
            fail(0x0005012E, "Precinct width or height for resolutions other than the coarsest must be larger than 1");
        }
      if (L != (nc < 257 ? 9u : 10u) + ((c.Scoc & 1) ? 1u + c.num_decomps : 0u))
        fail(0x0005012F, "error in COC segment length");
      coc.push_back(c);
    } else if (m == M_NLT) {                // param_nlt::read, ojph_params.cpp:2238-2266
      if (!r.has(6)) fail(0x00050141, "error reading NLT marker segment");
      uint32_t L = r.u16(), comp = r.u16(), bd = r.u8(), t = r.u8();
      if (L != 6 || (t != 3 && t != 0)) fail(0x00050145, "Unsupported NLT type %d\n", t);
      NltEntry* e = nullptr;
      if (comp == 0xFFFF) e = &nlt_all;
      else {
        for (NltEntry& x : nlt) if (x.comp_idx == comp) e = &x;
        if (e == nullptr) { nlt.push_back(NltEntry()); e = &nlt.back(); }
      }
      e->enabled = true; e->comp_idx = (uint16_t)comp; e->BDnlt = (uint8_t)bd; e->Tnlt = (uint8_t)t;
    } else if (m == M_DFS) {                // param_dfs::read, ojph_params.cpp:2596-2645
      if (!r.has(2)) fail(0x000500D1, "error reading DFS-Ldfs parameter");
      (void)r.u16();
      if (!r.has(2)) fail(0x000500D2, "error reading DFS-Sdfs parameter");
      DfsSpec d; d.Sdfs = (uint16_t)r.u16();
      if (d.Sdfs > 15) fail(0x000500D3, "The DFS-Sdfs parameter is %d, which is larger than the permissible 15", d.Sdfs);
      if (!r.has(1)) fail(0x000500D4, "error reading DFS-Ids parameter");
      const uint32_t ids = r.u8();
      if (ids == 0) fail(0x000500D8, "The value of the Ids member in the DFS marker segment cannot be 0");
      d.Ids = (uint8_t)std::min(ids, 32u);
      for (uint32_t i = 0; i < d.Ids; i += 4) { if (!r.has(1)) fail(0x000500D6, "error reading DFS-Ddfs parameters"); d.Ddfs[i / 4] = (uint8_t)r.u8(); }
      for (uint32_t i = d.Ids; i < ids; i += 4) { if (!r.has(1)) fail(0x000500D7, "error reading DFS-Ddfs parameters"); (void)r.u8(); }
      dfs.push_back(d);
    } else if (m == M_ATK) {                // param_atk::read, ojph_params.cpp:2770-2867
      if (!r.has(2)) fail(0x000500E1, "error reading ATK-Latk parameter");
      int bytes = (int)r.u16() - 2;
      if (!r.has(2)) fail(0x000500E2, "error reading ATK-Satk parameter");
      AtkSpec a; a.Satk = (uint16_t)r.u16(); bytes -= 2;
      const uint32_t idx = a.index();
      bool dup = idx == 0 || idx == 1;
      for (const AtkSpec& o2 : atk) if (o2.index() == idx) dup = true;
      if (dup) fail(0x000500F3, "ATK-Satk parameter sets ATK marker index to the illegal value of %d. ATK-Satk should be in "
                    "(2-255) and must not be repeated", idx);
      if (a.Satk & 0x2000) fail(0x000500E3, "ATK-Satk parameter sets m_init to 1, requiring odd-indexed subsequence in first "
                                "reconstruction step, which is not supported yet.");
      if (!(a.Satk & 0x800)) fail(0x000500E4, "ATK-Satk parameter specified ARB filter, which is not supported yet.");
      if (a.reversible() && a.coeff_type() >= 2) fail(0x000500E5, "ATK-Satk parameter does not make sense. It employs floats with reversible filtering.");
      if (!(a.Satk & 0x4000)) fail(0x000500E6, "ATK-Satk parameter requires constant boundary extension, which is not supported yet.");
      // coefficient readers (read_coefficient, :2687-2767); a 128-bit float keeps sign, 8 exponent bits and 23 mantissa bits
      auto read_float = [&](float& K) -> bool {
        switch (a.coeff_type()) {
          case 0: if (!r.has(1)) return false; K = (float)r.u8(); bytes -= 1; return true;
          case 1: if (!r.has(2)) return false; K = (float)r.u16(); bytes -= 2; return true;
          case 2: { if (!r.has(4)) return false; uint32_t u = r.u32(); memcpy(&K, &u, 4); bytes -= 4; return true; }
          case 3: { if (!r.has(8)) return false; uint64_t u = ((uint64_t)r.u32() << 32); u |= r.u32(); double d; memcpy(&d, &u, 8); K = (float)d; bytes -= 8; return true; }
          case 4: {
            if (!r.has(16)) return false;
            uint64_t v = ((uint64_t)r.u32() << 32); v |= r.u32(); (void)r.u32(); (void)r.u32(); bytes -= 16;
            int e = (int)((v >> 48) & 0x7FFF); e -= 16383; e += 127; e &= 0xFF; e <<= 23;
            uint32_t i = ((uint32_t)(v >> 32) & 0x80000000u) | (uint32_t)e | (uint32_t)((v >> 25) & 0x007FFFFF);
            memcpy(&K, &i, 4); return true;
          }
          default: return true;               // types 5..7: nothing is read (the reference's fall-through)
        }
      };
      auto read_int = [&](int16_t& K) -> bool {
        if (a.coeff_type() == 0) { if (!r.has(1)) return false; K = (int16_t)(int8_t)r.u8(); bytes -= 1; return true; }
        if (a.coeff_type() == 1) { if (!r.has(2)) return false; K = (int16_t)r.u16(); bytes -= 2; return true; }
        return false;
      };
      if (!a.reversible() && !read_float(a.K)) fail(0x000500E7, "error reading ATK-Katk parameter");
      if (!r.has(1)) fail(0x000500E8, "error reading ATK-Natk parameter");
      const uint32_t n = r.u8(); bytes -= 1;
      a.steps.resize(n);
      for (uint32_t i = 0; i < n; ++i) {
        AtkStep& t = a.steps[i];
        if (a.reversible()) {
          if (!r.has(1)) fail(0x000500E9, "error reading ATK-Eatk parameter");
          t.e = (uint8_t)r.u8(); bytes -= 1;
          if (!r.has(2)) fail(0x000500EA, "error reading ATK-Batk parameter");
          t.b = (int16_t)r.u16(); bytes -= 2;
          if (!r.has(1)) fail(0x000500EB, "error reading ATK-LCatk parameter");
          const uint32_t lc = r.u8(); bytes -= 1;
          if (lc == 0) fail(0x000500EC, "Encountered a ATK-LCatk value of zero; something is wrong.");
          if (lc > 1) fail(0x000500ED, "ATK-LCatk value greater than 1; that is, a multitap filter is not supported");
          if (!read_int(t.a)) fail(0x000500EE, "Error reding ATK-Aatk parameter");
        } else {
          if (!r.has(1)) fail(0x000500EF, "error reading ATK-LCatk parameter");
          const uint32_t lc = r.u8(); bytes -= 1;
          if (lc == 0) fail(0x000500F0, "Encountered a ATK-LCatk value of zero; something is wrong.");
          if (lc > 1) fail(0x000500F1, "ATK-LCatk value greater than 1; that is, a multitap filter is not supported.");
          if (!read_float(t.A)) fail(0x000500F2, "Error reding ATK-Aatk parameter");
        }
      }
      if (bytes != 0) fail(0x000500F3, "The length of an ATK marker segment (ATK-Latk) is not correct");
      atk.push_back(a);
    } else {  // PRF CPF RGN POC PPM TLM PLM CRG COM: skipped
      uint32_t L = r.u16();
      if (L < 2 || !r.has(L - 2)) fail(0x00030041, "error reading marker");
      r.pos += L - 2;
    }
  }
  // param_cod::update_atk (ojph_params.cpp:1279-1298): every kernel index must resolve
  (void)atk_for(wavelet);
  for (const CodStyle& c : coc)
    if (c.wavelet > 1) {
      bool found = false;
      for (const AtkSpec& a : atk) if (a.index() == c.wavelet) found = true;
      if (!found) fail(0x00050132, "A COC segment employs the DWT kernel atk = %d, but a corresponding ATK segment cannot be found", c.wavelet);
    }
  if (received != 3) fail(0x00030052, "markers error, COD and QCD are required");
  return r.pos;
}

//------------------------------------------------------------------------------------------
// The same codestream with its top resolution levels dropped
//------------------------------------------------------------------------------------------
// The profile a codestream's Rsiz names in its Part 1 field (bits 8-11, meaningful only without the Part 2 flag,
// bit 15): 1-3 broadcast, 4-9 IMF.  Returned as Params::profile (0 none, 1 IMF, 2 broadcast).
static uint32_t claimed_profile(uint16_t Rsiz) {
  if (Rsiz & 0x8000) return 0;
  const uint32_t f = (Rsiz >> 8) & 0xFu;
  return (f >= 1 && f <= 3) ? 2u : (f >= 4 && f <= 9) ? 1u : 0u;
}

void reduce_main_header(const std::vector<uint8_t>& hdr, const Params& in, uint32_t r, std::vector<uint8_t>& out,
                        Params& outp) {
  const uint32_t nc = in.num_comps();
  // the levels: the decoder's own refusals of restrict_input_resolution (Decoder::restrict_resolution)
  if (r > in.num_decomps)
    fail(0x000300A2, "skipped_resolution for data %d must be smaller than  the number of decomposition levels %d",
         r, in.num_decomps);
  for (uint32_t c = 0; c < nc; ++c)
    if (r > in.decomps(c))
      fail(0x000B0007, "component %u has %u decomposition levels; %u cannot be skipped", c, in.decomps(c), r);
  // a DFS level's split sets the reduction per direction and renumbers the kept bands' step-size entries
  for (uint32_t c = 0; c < nc; ++c)
    if (in.dfs_of(c) != nullptr)
      fail(0x000B0054, "component %u uses a DFS decomposition structure: its resolutions cannot be dropped", c);
  // SIZ: extent, image and tile offsets / 2^r rounded up; the tile size / 2^r along a direction with more than one
  // tile (which must divide), else rounded up, which still covers the image.  Every tile must keep samples, so that
  // tile indices -- and with them tile-parts and TLM entries -- stay the input's.
  const uint64_t s = 1ull << r;
  auto up = [&](uint32_t v) { return (uint32_t)(((uint64_t)v + s - 1) >> r); };
  uint32_t tsz[2];
  for (uint32_t d = 0; d < 2; ++d) {
    const uint32_t X = d ? in.Ysiz : in.Xsiz, XO = d ? in.YOsiz : in.XOsiz, XT = d ? in.YTsiz : in.XTsiz,
                   XTO = d ? in.YTOsiz : in.XTOsiz;
    const uint32_t nt = (uint32_t)(((uint64_t)X - XTO + XT - 1) / XT);
    if (nt > 1 && (XT & (s - 1)) != 0)
      fail(0x000B0055, "the tile %s %u is not a multiple of 2^%u, and there is more than one tile along it",
           d ? "height" : "width", XT, r);
    const uint32_t X1 = up(X), XO1 = up(XO), XTO1 = up(XTO), XT1 = nt > 1 ? XT >> r : up(XT);
    for (uint32_t k = 0; k < nt; ++k) {
      const uint64_t a = std::max<uint64_t>((uint64_t)XTO1 + (uint64_t)k * XT1, XO1);
      const uint64_t b = std::min<uint64_t>((uint64_t)XTO1 + (uint64_t)(k + 1) * XT1, X1);
      if (a >= b)
        fail(0x000B0055, "tile %s %u would be empty with %u resolution levels dropped", d ? "row" : "column", k, r);
    }
    tsz[d] = XT1;
  }
  // the step-size list a QCD serves: the components without a QCC
  uint32_t qcd_levels = in.num_decomps;
  for (uint32_t c = 0; c < nc; ++c)
    if (!std::any_of(in.qcc.begin(), in.qcc.end(), [&](const QuantSet& q) { return q.comp_idx == c; }))
      qcd_levels = std::max(qcd_levels, in.decomps(c));
  const uint32_t cs = nc < 257 ? 1u : 2u;            // component index bytes of COC / QCC
  out.assign(hdr.begin(), hdr.begin() + 2);          // SOC
  size_t cap_at = 0;
  for (size_t q = 2; q + 4 <= hdr.size(); ) {
    const uint32_t m = ((uint32_t)hdr[q] << 8) | hdr[q + 1], L = ((uint32_t)hdr[q + 2] << 8) | hdr[q + 3];
    std::vector<uint8_t> g(hdr.begin() + q, hdr.begin() + std::min(hdr.size(), q + 2 + L));
    q += 2 + L;
    auto put32 = [&](size_t o, uint32_t v) { g[o] = (uint8_t)(v >> 24); g[o + 1] = (uint8_t)(v >> 16); g[o + 2] = (uint8_t)(v >> 8); g[o + 3] = (uint8_t)v; };
    auto cut = [&](size_t keep) {                   // the segment's first `keep` bytes, its length field to match
      g.resize(keep);
      g[2] = (uint8_t)((keep - 2) >> 8); g[3] = (uint8_t)(keep - 2);
    };
    if (m == M_SIZ && g.size() >= 40) {
      put32(6, up(in.Xsiz)); put32(10, up(in.Ysiz)); put32(14, up(in.XOsiz)); put32(18, up(in.YOsiz));
      put32(22, tsz[0]); put32(26, tsz[1]); put32(30, up(in.XTOsiz)); put32(34, up(in.YTOsiz));
    } else if (m == M_CAP) {
      cap_at = out.size();
    } else if (m == M_COD && g.size() >= 14) {
      g[9] = (uint8_t)(g[9] - r);                    // SPcod: decomposition levels
      if (g[4] & 1) cut(g.size() - r);               // user precincts: entries 0 .. D - r
    } else if (m == M_COC && g.size() >= 10 + cs) {
      g[5 + cs] = (uint8_t)(g[5 + cs] - r);
      if (g[4 + cs] & 1) cut(g.size() - r);
    } else if ((m == M_QCD || m == M_QCC) && g.size() >= 5 + (m == M_QCC ? cs : 0)) {
      const size_t h = 5 + (m == M_QCC ? cs : 0);    // marker, length, [component,] Sqcd
      const uint32_t es = (g[h - 1] & 0x1F) == 0 ? 1u : 2u;
      uint32_t levels = qcd_levels;
      if (m == M_QCC) levels = in.decomps(cs == 1 ? g[4] : ((uint32_t)g[4] << 8) | g[5]);
      // the bands are listed from the LL band up (get_Kmax / get_irrev_delta index (resolution - 1) * 3 + band): the
      // kept ones are the first 1 + 3 (D - r), with the K_max and step size they had
      const size_t n = (g.size() - h) / es, keep = std::min<size_t>(n, 1 + 3 * (levels - r));
      cut(h + keep * es);
    }
    out.insert(out.end(), g.begin(), g.end());
  }
  // the reduced parameters as a decoder of the output reads them
  std::vector<uint8_t> parse(out);
  parse.push_back(0xFF); parse.push_back(0x90);
  outp = Params();
  outp.read_main_header(parse.data(), parse.size());
  // CAP: MAGB of the cut step-size lists (the input's may overstate it)
  if (cap_at) {
    outp.Ccap0 = (uint16_t)((outp.Ccap0 & 0xFFE0) | outp.cap_magb());
    out[cap_at + 8] = (uint8_t)(outp.Ccap0 >> 8); out[cap_at + 9] = (uint8_t)outp.Ccap0;
  }
  // a profile the input claims must hold for the output too (only its parameter rules: the tile-part division and
  // TLM it would impose on an encoder stay the input's)
  if (const uint32_t prof = claimed_profile(in.Rsiz)) {
    Params pc = outp;
    pc.profile = prof;
    try { pc.check_profile(); }
    catch (const Error& e) {
      fail(0x000B0056, "the codestream claims the %s profile (Rsiz 0x%04X), which it would break with %u resolution "
           "levels dropped: %s", prof == 1 ? "IMF" : "broadcast", in.Rsiz, r, e.what());
    }
  }
}

} // namespace ojb
