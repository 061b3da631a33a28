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
#include "ojb_device.h"
#include "ojb_kernels.h"
#include "dwt_common.cuh"

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

__global__ void __launch_bounds__(128)
rc_init_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks, EncBlock* __restrict__ work, EncResult* __restrict__ res, RcTables t)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  work[b] = blocks[b];
  t.chosen[b] = 0;
  const uint32_t r0 = t.ncand[b] ? rc_len(t.cand[(size_t)b * t.kc]) : 0u;
  res[b].len_head = r0 == RC_LEN_INVALID ? 0u : r0; res[b].len_tail = 0;
}

#define RS_THREADS 1024u
__global__ void __launch_bounds__(RS_THREADS)
rc_select_kernel(uint32_t nblocks, RcTables t)
{
  __shared__ unsigned long long red[RS_THREADS];
  if (t.state->done) return;
  const unsigned long long budget = t.state->budget > 0 ? (unsigned long long)t.state->budget : 0ull;
  const uint32_t tid = threadIdx.x;
  auto body = [&](unsigned long long key_t) -> unsigned long long {
    unsigned long long s = 0;
    for (uint32_t b = tid; b < nblocks; b += RS_THREADS) {
      const uint32_t j = rc_taken(t, b, key_t);
      if (j) s += t.hull_len[(size_t)b * t.kc + j - 1];
    }
    red[tid] = s;
    __syncthreads();
    for (uint32_t d = RS_THREADS / 2; d; d >>= 1) { if (tid < d) red[tid] += red[tid + d]; __syncthreads(); }
    const unsigned long long r = red[0];
    __syncthreads();
    return r;
  };
  // the smallest key t with body(t) <= budget; body(2^32) = 0 (no key reaches it)
  unsigned long long lo = 0, hi = 1ull << 32;
  if (body(0) <= budget) hi = 0;
  else
    while (hi - lo > 1) { const unsigned long long mid = (lo + hi) >> 1; if (body(mid) <= budget) hi = mid; else lo = mid; }
  const unsigned long long fin = body(hi);
  if (tid == 0) { t.state->thresh = (uint32_t)min(hi, 0xFFFFFFFFull); t.state->body = fin; }
}

__global__ void __launch_bounds__(128)
rc_apply_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks, EncBlock* __restrict__ work, EncResult* __restrict__ res, RcTables t)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks || t.state->done) return;
  const RcState& s = *t.state;
  const unsigned long long key_t = s.thresh == 0xFFFFFFFFu ? (1ull << 32) : s.thresh;
  const uint32_t j = rc_taken(t, b, key_t);
  const uint32_t k = t.hull_k[(size_t)b * (t.kc + 1) + j];
  EncBlock e = blocks[b];
  if (k >= 31u - e.p) e.flags &= (uint16_t)~ENC_CHECK_NEGZERO;     // left out: nothing may keep it coded
  e.p = (uint16_t)(e.p + k);
  work[b] = e;
  t.chosen[b] = (uint8_t)k;
  res[b].len_head = j ? t.hull_len[(size_t)b * t.kc + j - 1] : 0u; res[b].len_tail = 0;
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
  OJB_LAUNCH(rc_select_kernel, dim3(1), dim3(RS_THREADS), 0, st, nblocks, t);
  OJB_LAUNCH(rc_apply_kernel, dim3((nblocks + 127) / 128), dim3(128), 0, st, blocks, nblocks, work, res, t);
}
void launch_rc_check(const RcTables& t, const uint64_t* total, uint64_t target, uint64_t min_bytes, bool first, cudaStream_t st) {
  OJB_LAUNCH(rc_check_kernel, dim3(1), dim3(1), 0, st, t.state, total, (unsigned long long)target, (unsigned long long)min_bytes, first ? 1u : 0u);
}

} // namespace ojb
