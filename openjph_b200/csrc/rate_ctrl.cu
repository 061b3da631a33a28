// rate_ctrl.cu -- encode to a target codestream size: each code-block's cleanup pass is placed at the bit-plane a
// post-compression rate-distortion selection chooses, on the device, inside the frame's graph.
//
// An HT code-block may start its cleanup pass at any bit-plane; the packet header's missing-MSB count tells the decoder
// where.  Coding block b with its k lowest magnitude planes dropped is coding it with p = EncBlock::p + k, and
// k = K_max_b leaves it out of the packet.  The stream stays single-layer and cleanup-only.
//
//   rc_dist     one warp per block, one read per sample: D_b(k) for every k at once, and the block's top magnitude plane
//   (lengths)   ht_encode_serial_kernel<false, true>, one thread per (block, k): R_b(k), the exact cleanup length
//   rc_hull     one thread per block: lower convex hull of (R_b(k), D_b(k)), slope keys of its segments
//   rc_init     the unconstrained selection (k = 0 everywhere) into the working block array
//   rc_select   one CTA: the smallest slope key t whose selection fits the body budget, by bisection over the 32 key bits
//   rc_apply    one thread per block: the hull point after every segment with key >= t, into the working block array
//   rc_check    one thread: the exact stream size of the selection (packet header kernels, pkt_headers.cu) against the
//               target; over it, the budget shrinks by the overshoot and the next round selects again
// Every kernel after the first check is a no-op once RcState::done is set, so a fixed number of rounds can sit in a graph.
//
// A quality target (a squared-error limit) shares rc_dist, the lengths and rc_hull; its rounds measure each selection
// instead of trusting the model sum_b D_b, which holds to a factor only:
//   rq_init     one thread: the bracket (t_pass = 0, the unconstrained selection; t_fail = 2^32, every block left out)
//   rc_select<true>  one CTA: the key to try -- in the first RQ_MODEL_ROUNDS rounds the model's proposal (the
//               largest key whose sum_b D_b is within c * limit) when it lies inside the bracket, t_pass + 1 when it
//               lies on or below it; otherwise the selection that halves the bracket's body gap; after RQ_BODY_ROUNDS
//               rounds the bracket's key midpoint
//   rc_apply<1> that selection into the working block array
//   rq_recon    one warp per block: what the decoder's store writes for each block coded at p + k, into a second
//               coefficient arena; then the inverse DWT launches of the decoder write the decoded image into a scratch
//   rq_sse      the exact squared error of the scratch against the source, per component, in 128-bit integers
//   rq_update   one thread: the bracket, the model's correction c, the stop rule
//   rc_apply<2> the final selection, at t_pass
// The round kernels are no-ops once RqState::done is set (the DWT launches in between are not, so only a few rounds
// sit in the frame's graph; the rest run eagerly).
#include "ojb_device.h"
#include "ojb_kernels.h"
#include "dwt_common.cuh"
#include "dequant.cuh"
#include <algorithm>

namespace ojb {

namespace {

__device__ __forceinline__ uint32_t rc_len(const EncResult& r) { return r.len_head == RC_LEN_INVALID ? RC_LEN_INVALID : r.len_head + r.len_tail; }

// D_b(k) = W_b sum_i (m_i - r_k(m_i))^2, m_i the magnitude in quantiser units; r_k(m) = 0 when m >> k == 0, else
// ((m >> k) << k) + h_k with h_k = 2^(k-1) (k >= 1), 1/2 (k = 0, irreversible) or 0 (k = 0, reversible): the bin centre
// the decoders reconstruct
// One read per sample: every lane keeps a partial sum per k (fp64, in registers: the k loop is unrolled over the 32
// possible planes), then one warp reduction per k
__global__ void __launch_bounds__(128)
rc_dist_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks, const uint32_t* __restrict__ coef, RcTables t)
{
  const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (b >= nblocks) return;
  const EncBlock blk = blocks[b];
  const uint32_t p = blk.p, kmax = 31u - p;
  const uint32_t* src = coef + blk.src_off;
  const double h0 = t.irv[b] ? 0.5 : 0.0;
  double acc[32];
  #pragma unroll
  for (int k = 0; k < 32; ++k) acc[k] = 0.0;
  uint32_t top = 0;
  for (uint32_t y = 0; y < blk.h; ++y)
    for (uint32_t x = lane; x < blk.w; x += 32) {
      const uint32_t m = (src[(size_t)y * blk.stride + x] & 0x7FFFFFFFu) >> p;
      top |= m;
      #pragma unroll
      for (uint32_t k = 0; k < 32; ++k) {
        const double half = k ? (double)(1u << (k - 1)) : h0;
        const double e = (m >> k) ? (double)(m & ((1u << k) - 1u)) - half : (double)m;
        acc[k] += e * e;
      }
    }
  #pragma unroll
  for (int d = 16; d; d >>= 1) top |= __shfl_xor_sync(0xFFFFFFFFu, top, d);
  #pragma unroll
  for (uint32_t k = 0; k < 32; ++k) {
    double v = acc[k];
    #pragma unroll
    for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
    if (lane == 0 && k <= kmax) t.dist[(size_t)b * t.kc + k] = t.weight[b] * v;
  }
  if (lane == 0) {
    const uint32_t planes = top ? 32u - (uint32_t)__clz((int)top) : 0u;
    t.ncand[b] = (uint8_t)((blk.flags & ENC_CHECK_NEGZERO) ? 1u : planes);    // a NEGZERO block is coded whole or not at all
  }
}

__global__ void __launch_bounds__(128)
rc_hull_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks, RcTables t)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  const uint32_t kc = t.kc, kmax = 31u - blocks[b].p, nc = t.ncand[b];
  const EncResult* cand = t.cand + (size_t)b * kc;
  const double* dist = t.dist + (size_t)b * kc;
  // gift wrapping from the excluded point (0, D_b(K_max)): the next hull point is the one of largest slope
  // (D_cur - D) / (R - R_cur) among those with R > R_cur and D < D_cur; equal slopes: the larger R
  uint32_t cur_r = 0, n = 0, last_key = 0xFFFFFFFFu;
  double cur_d = dist[kmax];
  t.hull_k[(size_t)b * (kc + 1)] = (uint8_t)kmax;
  for (;;) {
    int best = -1; double best_s = 0.0; uint32_t best_r = 0;
    for (uint32_t k = 0; k < nc; ++k) {
      const uint32_t r = rc_len(cand[k]);
      if (r == RC_LEN_INVALID || r <= cur_r || !(dist[k] < cur_d)) continue;
      const double s = (cur_d - dist[k]) / (double)(r - cur_r);
      if (best < 0 || s > best_s || (s == best_s && r > best_r)) { best = (int)k; best_s = s; best_r = r; }
    }
    if (best < 0) break;
    uint32_t key = __float_as_uint((float)best_s);       // positive floats order as their bit patterns
    key = min(key, last_key); last_key = key;
    t.hull_key[(size_t)b * kc + n] = key;
    t.hull_len[(size_t)b * kc + n] = best_r;
    t.hull_k[(size_t)b * (kc + 1) + n + 1] = (uint8_t)best;
    ++n; cur_r = best_r; cur_d = dist[best];
  }
  t.hull_n[b] = (uint8_t)n;
  const uint32_t r0 = nc ? rc_len(cand[0]) : 0u;
  if (r0 && r0 != RC_LEN_INVALID) atomicAdd(&t.state->sum0, (unsigned long long)r0);
}

// hull segments of block b with key >= key_t (a prefix: keys do not increase along the hull)
__device__ __forceinline__ uint32_t rc_taken(const RcTables& t, uint32_t b, unsigned long long key_t) {
  const uint32_t n = t.hull_n[b];
  const uint32_t* key = t.hull_key + (size_t)b * t.kc;
  uint32_t j = 0;
  while (j < n && key[j] >= key_t) ++j;
  return j;
}

// the point block b is coded at for slope key key_t: its k, and the cleanup length in len.  zero_init (quality target):
// key 0 is the unconstrained selection, every block at k = 0 as rc_init writes it (the hull's last point can be a
// k > 0 of equal distortion)
__device__ __forceinline__ uint32_t rc_point(const RcTables& t, uint32_t b, unsigned long long key_t, bool zero_init, uint32_t& len) {
  if (zero_init && key_t == 0) {
    const uint32_t r0 = t.ncand[b] ? rc_len(t.cand[(size_t)b * t.kc]) : 0u;
    len = r0 == RC_LEN_INVALID ? 0u : r0;
    return 0;
  }
  const uint32_t j = rc_taken(t, b, key_t);
  len = j ? t.hull_len[(size_t)b * t.kc + j - 1] : 0u;
  return t.hull_k[(size_t)b * (t.kc + 1) + j];
}

__global__ void __launch_bounds__(128)
rc_init_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks, EncBlock* __restrict__ work, EncResult* __restrict__ res, RcTables t)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  work[b] = blocks[b];
  t.chosen[b] = 0;
  uint32_t len; rc_point(t, b, 0, true, len);
  res[b].len_head = len; res[b].len_tail = 0;
}

#define RS_THREADS 1024u
// QUALITY = false: the smallest slope key whose selection's body fits the budget (size target).  QUALITY = true: the key
// a round of the quality target tries (see the top of the file).  Both sums run in a fixed order (a thread's blocks in
// index order, then a fixed tree), so the selection is deterministic.
template <bool QUALITY>
__global__ void __launch_bounds__(RS_THREADS)
rc_select_kernel(uint32_t nblocks, RcTables t)
{
  __shared__ unsigned long long red[RS_THREADS];
  __shared__ double redd[QUALITY ? RS_THREADS : 1];
  if (QUALITY ? t.q->done : t.state->done) return;
  const uint32_t tid = threadIdx.x;
  auto body = [&](unsigned long long key_t) -> unsigned long long {
    unsigned long long s = 0;
    for (uint32_t b = tid; b < nblocks; b += RS_THREADS) { uint32_t len; rc_point(t, b, key_t, QUALITY, len); s += len; }
    red[tid] = s;
    __syncthreads();
    for (uint32_t d = RS_THREADS / 2; d; d >>= 1) { if (tid < d) red[tid] += red[tid + d]; __syncthreads(); }
    const unsigned long long r = red[0];
    __syncthreads();
    return r;
  };
  // the smallest key t with body(t) <= budget; body(2^32) = 0 (no key reaches it)
  auto fitting = [&](unsigned long long budget) -> unsigned long long {
    unsigned long long lo = 0, hi = 1ull << 32;
    if (body(0) <= budget) return 0;
    while (hi - lo > 1) { const unsigned long long mid = (lo + hi) >> 1; if (body(mid) <= budget) hi = mid; else lo = mid; }
    return hi;
  };
  if (!QUALITY) {
    const unsigned long long hi = fitting(t.state->budget > 0 ? (unsigned long long)t.state->budget : 0ull);
    const unsigned long long fin = body(hi);
    if (tid == 0) { t.state->thresh = (uint32_t)min(hi, 0xFFFFFFFFull); t.state->body = fin; }
    return;
  }
  auto dist = [&](unsigned long long key_t) -> double {
    double s = 0.0;
    for (uint32_t b = tid; b < nblocks; b += RS_THREADS) {
      uint32_t len; const uint32_t k = rc_point(t, b, key_t, true, len);
      s += t.dist[(size_t)b * t.kc + k];
    }
    redd[tid] = s;
    __syncthreads();
    for (uint32_t d = RS_THREADS / 2; d; d >>= 1) { if (tid < d) redd[tid] += redd[tid + d]; __syncthreads(); }
    const double r = redd[0];
    __syncthreads();
    return r;
  };
  RqState& q = *t.q;
  const unsigned long long full = 1ull << 32, tp = q.t_pass, tf = q.t_fail;
  const uint32_t r = q.rounds;
  bool halve = r < RQ_BODY_ROUNDS;
  unsigned long long key = (tp + tf) >> 1;
  if (q.force_zero) { key = 0; halve = false; }
  else if (r < RQ_MODEL_ROUNDS) {
    // the largest key whose modelled error is within c * limit (dist does not fall as the key grows)
    const double lim = q.c * (double)q.limit;
    unsigned long long tm = 0;
    if (dist(full) <= lim) tm = full;
    else if (dist(0) <= lim) {
      unsigned long long lo = 0, hi = full;
      while (hi - lo > 1) { const unsigned long long mid = (lo + hi) >> 1; if (dist(mid) <= lim) lo = mid; else hi = mid; }
      tm = lo;
    }
    // inside the bracket: take it.  On or below t_pass (the model's selections change only at hull keys: it says the
    // next step overshoots): t_pass + 1, which drops only the segments of key t_pass
    if ((tm > tp && tm < tf) || (tm == full && !q.fail_measured)) { key = tm; halve = false; }
    else if (tm <= tp) { key = tp + 1; halve = false; }
  }
  // halving: the selection whose body is the nearest at or under the middle of the bracket's bodies, kept inside the
  // bracket (the stop rule is one on bodies); after RQ_BODY_ROUNDS rounds the key midpoint bounds the search
  if (halve) key = min(max(fitting((q.body_pass + q.body_fail) >> 1), tp + 1), tf - 1);
  const unsigned long long fin = body(key);
  const double model = r == 0 ? dist(key) : 0.0;
  if (tid == 0) {
    q.key = key; q.body = fin;
    if (r == 0) q.model1 = model;
  }
  if (tid < 2 * RQ_MAX_COMPS) q.comp_cur[tid >> 1][tid & 1] = 0;
}

// MODE 0: the size target's selection (RcState::thresh); 1: the key a quality round tries; 2: the quality target's
// final selection, at t_pass
template <int MODE>
__global__ void __launch_bounds__(128)
rc_apply_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks, EncBlock* __restrict__ work, EncResult* __restrict__ res, RcTables t)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  unsigned long long key_t;
  if (MODE == 0) {
    if (t.state->done) return;
    key_t = t.state->thresh == 0xFFFFFFFFu ? (1ull << 32) : t.state->thresh;
  } else if (MODE == 1) {
    if (t.q->done) return;
    key_t = t.q->key;
  } else key_t = t.q->t_pass;
  uint32_t len;
  const uint32_t k = rc_point(t, b, key_t, MODE != 0, len);
  EncBlock e = blocks[b];
  if (k >= 31u - e.p) e.flags &= (uint16_t)~ENC_CHECK_NEGZERO;     // left out: nothing may keep it coded
  e.p = (uint16_t)(e.p + k);
  work[b] = e;
  t.chosen[b] = (uint8_t)k;
  res[b].len_head = len; res[b].len_tail = 0;
}

// first: the unconstrained stream was sized; if it does not fit, B_0 = the target less the stream with every block left
// out (min_bytes).  That budget counts no header bytes for the blocks it includes, so a small target keeps room for
// bodies (the headers of the unconstrained selection can exceed the whole target).  A round whose stream is over the
// target sets B = body - overshoot, body being what its selection used (<= B): the next selection's body is strictly
// smaller, so the rounds end -- at the latest at B = 0, the stream of min_bytes <= target
__global__ void rc_check_kernel(RcState* __restrict__ s, const uint64_t* __restrict__ total, unsigned long long target,
                                unsigned long long min_bytes, uint32_t first)
{
  if (s->done) return;
  const unsigned long long tot = total[0];
  s->total = tot;
  if (first) {
    s->budget = (long long)target - (long long)min_bytes;
    s->body = s->sum0;
  } else {
    s->rounds += 1;
    if (tot > target) s->budget = (long long)min((unsigned long long)s->budget, s->body) - (long long)(tot - target);
  }
  if (s->budget < 0) s->budget = 0;
  if (tot <= target) s->done = 1;
}

// the stop rule: the bracket is closed when its keys are adjacent, or when the two selections' bodies differ by at most
// max(0.25 % of the passing body, 64 bytes).  A closed bracket whose passing side was never measured (key 0, an
// irreversible component) measures key 0 next: the quantisation sets a floor only a measurement finds
__device__ void rq_close(RqState& q) {
  const unsigned long long gap = q.body_pass - q.body_fail;
  if (q.t_fail - q.t_pass <= 1 || gap * 400 <= q.body_pass || gap <= 64) {
    if (q.pass_measured) { q.done = 1; q.reached = 1; }
    else q.force_zero = 1;
  }
}

// lossless0: every component is reversible and no block can lose a sample (ENC_CHECK_NEGZERO), so the unconstrained
// selection decodes to the source: its error, 0, is known without a measurement
__global__ void rq_init_kernel(RcTables t, unsigned long long limit, uint32_t ncomp, uint32_t lossless0)
{
  RqState& q = *t.q;
  q.limit = limit; q.ncomp = ncomp;
  q.t_pass = 0; q.t_fail = 1ull << 32;
  q.body0 = q.body_pass = t.state->sum0; q.body_fail = 0;
  q.c = 1.0;
  q.pass_measured = lossless0;
  rq_close(q);
}

// one warp per block: block b coded at p + k decodes to sign | ((m >> k) << (p + k)) | 2^(p + k - 1) for every
// sample whose m >> k is not 0, and to 0 for the others; to_output turns that into the value the decoder stores (its
// integer shift is 31 - K_max, the p of the static block array geom: a transcoded block starts at or below K_max)
__global__ void __launch_bounds__(128)
rq_recon_kernel(const EncBlock* __restrict__ geom, const EncBlock* __restrict__ blocks, uint32_t nblocks, const uint32_t* __restrict__ coef,
                uint32_t* __restrict__ out, RcTables t)
{
  const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
  if (b >= nblocks || t.q->done) return;
  const EncBlock blk = blocks[b];
  const uint32_t p = blk.p, k = t.chosen[b], pk = p + k;
  const uint32_t mode = t.irv[b] ? (uint32_t)DEC_OUT_FLOAT : (uint32_t)DEC_OUT_INT, shift = geom[b].p;
  const float delta = t.delta[b];
  const uint32_t* src = coef + blk.src_off;
  uint32_t* dst = out + blk.src_off;
  for (uint32_t y = 0; y < blk.h; ++y)
    for (uint32_t x = lane; x < blk.w; x += 32) {
      const uint32_t w = src[(size_t)y * blk.stride + x];
      const uint32_t m = ((w & 0x7FFFFFFFu) >> p) >> k;
      dst[(size_t)y * blk.stride + x] = m ? to_output((w & 0x80000000u) | (m << pk) | (1u << (pk - 1)), mode, shift, delta) : 0u;
    }
}

__device__ __forceinline__ long long rq_sample(const ImgComp& c, uint32_t type, uint32_t x, uint32_t y) {
  const uint8_t* row = reinterpret_cast<const uint8_t*>(c.base) + (size_t)y * c.pitch;
  const size_t i = (size_t)x * c.col;
  if (type == 0) return row[i];
  if (type == 1) return reinterpret_cast<const uint16_t*>(row)[i];
  return reinterpret_cast<const int32_t*>(row)[i];
}

// (lo, hi) += (vlo, vhi)
__device__ __forceinline__ void add128(unsigned long long& lo, unsigned long long& hi, unsigned long long vlo, unsigned long long vhi) {
  const unsigned long long s = lo + vlo;
  hi += vhi + (s < lo ? 1ull : 0ull); lo = s;
}

// sum over component blockIdx.y of (decoded - source)^2: rows over CTAs, columns over threads; each thread sums in
// 128 bits, a warp reduces, one lane adds to the component's total with a carry into the high word
#define RQ_SSE_THREADS 256u
__global__ void __launch_bounds__(RQ_SSE_THREADS)
rq_sse_kernel(const ImgComp* __restrict__ dec, const ImgComp* __restrict__ src, RqImage im, RcTables t)
{
  const uint32_t c = blockIdx.y;
  if (t.q->done || c >= im.ncomp) return;
  const ImgComp a = dec[c], s = src[c];
  unsigned long long lo = 0, hi = 0;
  for (uint32_t y = blockIdx.x; y < im.h[c]; y += gridDim.x)
    for (uint32_t x = threadIdx.x; x < im.w[c]; x += blockDim.x) {
      const long long d = rq_sample(a, im.sample_type, x, y) - rq_sample(s, im.sample_type, x, y);
      const unsigned long long m = (unsigned long long)(d < 0 ? -d : d);
      add128(lo, hi, m * m, 0);
    }
  #pragma unroll
  for (int o = 16; o; o >>= 1) {
    const unsigned long long l = __shfl_xor_sync(0xFFFFFFFFu, lo, o), h = __shfl_xor_sync(0xFFFFFFFFu, hi, o);
    add128(lo, hi, l, h);
  }
  if ((threadIdx.x & 31u) == 0 && (lo | hi)) {
    unsigned long long* acc = t.q->comp_cur[c];
    const unsigned long long old = atomicAdd(&acc[0], lo);
    const unsigned long long carry = (old + lo < old) ? 1ull : 0ull;
    if (hi + carry) atomicAdd(&acc[1], hi + carry);
  }
}

// the round's measurement into the bracket (see the top of the file)
__global__ void rq_update_kernel(RcTables t)
{
  RqState& q = *t.q;
  if (q.done) return;
  unsigned long long lo = 0, hi = 0;
  for (uint32_t c = 0; c < q.ncomp; ++c) add128(lo, hi, q.comp_cur[c][0], q.comp_cur[c][1]);
  if (q.rounds < RQ_MAX_ROUNDS) q.round[q.rounds] = RqRound{ q.key, lo, hi, q.body };
  q.rounds += 1;
  const bool pass = hi == 0 && lo <= q.limit;
  if (pass || q.key == 0) {      // a pass; or key 0 failing, which is returned as it is (reached stays 0)
    q.t_pass = q.key; q.body_pass = q.body; q.sse_pass[0] = lo; q.sse_pass[1] = hi; q.pass_measured = 1;
    for (uint32_t c = 0; c < q.ncomp; ++c) { q.comp_pass[c][0] = q.comp_cur[c][0]; q.comp_pass[c][1] = q.comp_cur[c][1]; }
    if (!pass) { q.done = 1; return; }
  } else {
    q.t_fail = q.key; q.body_fail = q.body; q.fail_measured = 1;
  }
  const double sse = (double)hi * 18446744073709551616.0 + (double)lo;
  q.c = sse > 0.0 ? q.c * (double)q.limit / sse : q.c * 2.0;
  rq_close(q);
  if (q.rounds >= RQ_MAX_ROUNDS && !q.done) q.done = 1;      // not reached: the bracket closes within RQ_BODY_ROUNDS + 34
}

} // namespace

// squared norm of component c's column of the inverse colour transform: what one unit of error in that component
// costs summed over the three output components
double colour_weight(bool ict, uint32_t c) {
  if (c == 0) return 3.0;
  if (!ict) return 11.0 / 16.0;           // RCT: G = Y - (Cb + Cr) / 4, R = Cr + G, B = Cb + G (linearised)
  if (c == 1) return (double)ICT_GAMMA_CB2G * ICT_GAMMA_CB2G + (double)ICT_GAMMA_CB2B * ICT_GAMMA_CB2B;
  return (double)ICT_GAMMA_CR2G * ICT_GAMMA_CR2G + (double)ICT_GAMMA_CR2R * ICT_GAMMA_CR2R;
}

void launch_rc_prepare(const EncBlock* blocks, uint32_t nblocks, const uint32_t* coef, const RcTables& t, cudaStream_t st) {
  OJB_LAUNCH(rc_dist_kernel, dim3((nblocks + 3) / 4), dim3(128), 0, st, blocks, nblocks, coef, t);
}
void launch_rc_hull(const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res, const RcTables& t, cudaStream_t st) {
  OJB_LAUNCH(rc_hull_kernel, dim3((nblocks + 127) / 128), dim3(128), 0, st, blocks, nblocks, t);
  OJB_LAUNCH(rc_init_kernel, dim3((nblocks + 127) / 128), dim3(128), 0, st, blocks, nblocks, work, res, t);
}
void launch_rc_round(const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res, const RcTables& t, cudaStream_t st) {
  OJB_LAUNCH(rc_select_kernel<false>, dim3(1), dim3(RS_THREADS), 0, st, nblocks, t);
  OJB_LAUNCH(rc_apply_kernel<0>, dim3((nblocks + 127) / 128), dim3(128), 0, st, blocks, nblocks, work, res, t);
}
void launch_rc_check(const RcTables& t, const uint64_t* total, uint64_t target, uint64_t min_bytes, bool first, cudaStream_t st) {
  OJB_LAUNCH(rc_check_kernel, dim3(1), dim3(1), 0, st, t.state, total, (unsigned long long)target, (unsigned long long)min_bytes, first ? 1u : 0u);
}

void launch_rq_init(const RcTables& t, uint64_t limit, uint32_t ncomp, bool lossless0, cudaStream_t st) {
  OJB_LAUNCH(rq_init_kernel, dim3(1), dim3(1), 0, st, t, (unsigned long long)limit, ncomp, lossless0 ? 1u : 0u);
}
void launch_rq_select(const EncBlock* geom, const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res,
                      const uint32_t* coef, uint32_t* recon, const RcTables& t, cudaStream_t st) {
  OJB_LAUNCH(rc_select_kernel<true>, dim3(1), dim3(RS_THREADS), 0, st, nblocks, t);
  OJB_LAUNCH(rc_apply_kernel<1>, dim3((nblocks + 127) / 128), dim3(128), 0, st, blocks, nblocks, work, res, t);
  OJB_LAUNCH(rq_recon_kernel, dim3((nblocks + 3) / 4), dim3(128), 0, st, geom, blocks, nblocks, coef, recon, t);
}
void launch_rq_measure(const ImgComp* decoded, const ImgComp* source, const RqImage& im, const RcTables& t, cudaStream_t st) {
  uint32_t rows = 1;
  for (uint32_t c = 0; c < im.ncomp; ++c) rows = std::max(rows, im.h[c]);
  OJB_LAUNCH(rq_sse_kernel, dim3(std::min(rows, 1024u), im.ncomp), dim3(RQ_SSE_THREADS), 0, st, decoded, source, im, t);
  OJB_LAUNCH(rq_update_kernel, dim3(1), dim3(1), 0, st, t);
}
void launch_rq_final(const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res, const RcTables& t, cudaStream_t st) {
  OJB_LAUNCH(rc_apply_kernel<2>, dim3((nblocks + 127) / 128), dim3(128), 0, st, blocks, nblocks, work, res, t);
}

} // namespace ojb
