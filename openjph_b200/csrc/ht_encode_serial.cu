// ht_encode_serial.cu -- HTJ2K cleanup-pass block encoder, one THREAD per code-block.
//
// Computes what ojph_encode_codeblock32 computes (src/core/coding/ojph_block_encoder.cpp:542-1016),
// byte for byte, like ht_encode.cu.  The three bit-streams of a block are inherently sequential
// (byte stuffing and the adaptive MEL coder make every bit position depend on all earlier data), so
// the warp-per-block kernel spends most of its instructions on warp-wide scans, shared-memory bit
// scatter and stuffing fix-ups that keep 32 lanes in lock step.  Here every lane walks its own block
// quad by quad with the three writers in registers -- far fewer instructions per sample --
// and a warp advances 32 independent blocks.  Latency (one serial chain per thread) is covered by
// software prefetch of the next quad pair and by the other frames in flight on the device.
//   * MagSgn goes through a 128-bit window: one append per quad (its four fields fit 64 bits when K_max <= 15),
//     flushed straight to the block's slot as aligned 8-byte groups whose stuffing (7-bit byte after 0xFF,
//     :483-488) is done on the whole group by SWAR -- the flush is the same straight-line code for every lane
//     of the warp, not a byte loop a few lanes take at a time;
//   * VLC is written backward from the slot end as aligned 4-byte groups (7-bit byte 0x7F after a byte > 0x8F,
//     :393-404, tested on four bytes at once; the byte-wise path runs only when it applies);
//   * MEL bytes (<= 192, the reference's limit) stay in shared memory until termination;
//   * the previous quad-row's significance / exponents live in a per-thread shared-memory row.
#include "ojb_device.h"
#include "ojb_kernels.h"
#include "ojb_async.cuh"

namespace ojb {

#define ES_THREADS 128
#define ES_MEL_BYTES 200
#define MEL_EXP(k) ((uint32_t)((0x5433222111000ull >> (4 * (k))) & 7ull))

namespace {

template <bool WIDE> struct WordOf;
template <> struct WordOf<false> { typedef uint32_t W; };
template <> struct WordOf<true> { typedef unsigned long long W; };

struct MsWriter {            // forward, LSB first: a 128-bit window (w1:w0), fewer than 64 bits pending between puts
  unsigned long long w0, w1; uint32_t nbits, words; uint32_t last_ff;
};
struct VlcWriter {           // backward, LSB first
  unsigned long long acc; uint32_t nbits, words, prev;
};
struct MelWriter {
  uint32_t k, run, tmp, rem, pos;
};

// Emit eight MagSgn bytes (needs nbits >= 64).  Byte stuffing (a byte after 0xFF carries 7 bits, :483-488)
// is done on the whole 64-bit group: the 0xFF bytes are located with SWAR tests and a zero bit is opened
// above each of them, lowest first -- no byte loop, and groups without 0xFF (the usual case) take the
// straight path.  One 8-byte store per group.
template <bool ST = true>
__device__ __forceinline__ void ms_flush8(MsWriter& s, uint2* dst) {
  const unsigned long long M = 0x0080808080808080ull;         // bytes 0..6: a 0xFF in byte 7 shortens the NEXT group
  const unsigned long long M7 = 0x0101010101010101ull;
  const uint32_t lf = s.last_ff;
  unsigned long long x = (s.w0 & 0x7Full) | ((s.w0 >> 7) << (7 + lf));   // 7-bit first byte after a 0xFF
  uint32_t c = 64u - lf;                                                  // data bits this group takes
  // bit 8i+7 <=> byte i == 0xFF (low seven bits all ones: adding 1 carries into bit 7; and bit 7 set)
  unsigned long long ff = ((x & 0x7F7F7F7F7F7F7F7Full) + M7) & x & M;
  while (ff) {
    const uint32_t pos = (uint32_t)__ffsll((long long)ff) + 7u;           // top bit of the byte after the 0xFF
    x = (x & ((1ull << pos) - 1ull)) | (((x >> pos) << pos) << 1);
    --c;
    ff = ((x & 0x7F7F7F7F7F7F7F7Full) + M7) & x & M & (~0ull << pos);
  }
  if (ST) dst[s.words >> 1] = make_uint2((uint32_t)x, (uint32_t)(x >> 32));
  s.words += 2;
  s.last_ff = ((uint32_t)(x >> 56) == 0xFFu) ? 1u : 0u;
  // drop c (56..64) bits from the window
  const uint32_t a1 = (uint32_t)(s.w0 >> 32), a2 = (uint32_t)s.w1, a3 = (uint32_t)(s.w1 >> 32), r = c - 32u;
  const uint32_t n0 = __funnelshift_rc(a1, a2, r), n1 = __funnelshift_rc(a2, a3, r), n2 = __funnelshift_rc(a3, 0u, r);
  s.w0 = (unsigned long long)n0 | ((unsigned long long)n1 << 32);
  s.w1 = (unsigned long long)n2;
  s.nbits -= c;
}
// append up to 64 bits; fewer than 64 bits are pending on entry and on exit
template <bool ST = true>
__device__ __forceinline__ void ms_put(MsWriter& s, unsigned long long cwd, uint32_t len, uint2* dst) {
  s.w1 = (cwd >> 1) >> (63u - s.nbits);                     // the part that does not fit the low word
  s.w0 |= cwd << s.nbits; s.nbits += len;
  while (s.nbits >= 64) ms_flush8<ST>(s, dst);
}

// emit four VLC bytes (needs nbits >= 32); `end` = one past the slot, words grow downward
template <bool ST = true>
__device__ __forceinline__ void vlc_flush4(VlcWriter& v, uint32_t* end) {
  const uint32_t lo = (uint32_t)v.acc;
  const uint32_t pv = (lo << 8) | v.prev;
  uint32_t w, used;
  if (((((lo & 0x7F7F7F7Fu) + 0x01010101u) & pv & ((pv & 0x70707070u) + 0x70707070u)) & 0x80808080u) == 0) {
    w = lo; used = 32;
  } else {
    unsigned long long a = v.acc;
    uint32_t p = v.prev;
    w = 0; used = 0;
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint32_t b = (uint32_t)a & 0xFFu, n = 8;
      if (p > 0x8F && (b & 0x7F) == 0x7F) { b = 0x7F; n = 7; }
      w |= b << (8 * i); a >>= n; used += n; p = b;
    }
  }
  v.prev = w >> 24;
  ++v.words;
  if (ST) end[-(int)v.words] = __byte_perm(w, 0, 0x0123);
  v.acc >>= used; v.nbits -= used;
}
template <bool ST = true>
__device__ __forceinline__ void vlc_put(VlcWriter& v, uint32_t cwd, uint32_t len, uint32_t* end) {
  v.acc |= (unsigned long long)cwd << v.nbits; v.nbits += len;
  while (v.nbits >= 32) vlc_flush4<ST>(v, end);
}

template <int MS = ES_THREADS>
__device__ __forceinline__ void mel_bit(MelWriter& m, uint32_t v, uint8_t* buf) {
  m.tmp = (m.tmp << 1) | v;
  if (--m.rem == 0) {
    if (m.pos < ES_MEL_BYTES) buf[m.pos * MS] = (uint8_t)m.tmp;
    m.pos++;
    m.rem = (m.tmp == 0xFF) ? 7 : 8;
    m.tmp = 0;
  }
}
template <int MS = ES_THREADS>
__device__ __forceinline__ void mel_event(MelWriter& m, bool one, uint8_t* buf) {     // mel_encode :321-348
  if (!one) {
    if (++m.run >= (1u << MEL_EXP(m.k))) { mel_bit<MS>(m, 1, buf); m.run = 0; m.k = m.k < 12 ? m.k + 1 : 12; }
  } else {
    mel_bit<MS>(m, 0, buf);
    for (uint32_t t = MEL_EXP(m.k); t > 0; ) { --t; mel_bit<MS>(m, (m.run >> t) & 1u, buf); }
    m.run = 0; m.k = m.k > 0 ? m.k - 1 : 0;
  }
}

// terminate_mel_vlc :413-441, ms_terminate :517-533: the pending bits of the three streams, the MEL / VLC byte
// fusion, MEL bytes moved behind MagSgn, Scup.  ST = false: lengths only (nothing is stored; a block the final
// encode would refuse gets the length RC_LEN_INVALID instead of a status bit)
template <int MS = ES_THREADS, bool ST = true>
__device__ __forceinline__ void terminate_block(MsWriter& ms, VlcWriter& vlc, MelWriter& mel, uint8_t* mel_buf, uint8_t* slot,
                                                uint32_t slot_cap, uint32_t* status, EncResult& res)
{
  // ---- termination (terminate_mel_vlc :413-441, ms_terminate :517-533)
  uint32_t ms_pos = ms.words * 4;
  {
    unsigned long long acc = ms.w0; uint32_t nb = ms.nbits;        // < 64 raw bits: cut them into bytes
    bool lf = ms.last_ff != 0;
    for (;;) {
      const uint32_t n = lf ? 7u : 8u;
      if (nb < n) break;
      const uint32_t b = (uint32_t)acc & ((1u << n) - 1u);
      if (ST) slot[ms_pos] = (uint8_t)b;
      ++ms_pos; acc >>= n; nb -= n; lf = (b == 0xFF);
    }
    const uint32_t cap = lf ? 7u : 8u;
    if (nb) {
      const uint32_t t = cap - nb;
      const uint32_t byte = (uint32_t)acc | ((0xFFu & ((1u << t) - 1u)) << nb);
      if (byte != 0xFF) { if (ST) slot[ms_pos] = (uint8_t)byte; ++ms_pos; }
    } else if (cap == 7) ms_pos--;
  }
  if (mel.run > 0) mel_bit<MS>(mel, 1, mel_buf);
  const uint32_t mel_tmp = (mel.tmp << mel.rem) & 0xFFu;
  const uint32_t mel_mask = (0xFFu << mel.rem) & 0xFFu;
  uint32_t vl_pos = vlc.words * 4;
  uint8_t* vend = slot + slot_cap;
  uint32_t vl_tmp, vl_mask;
  {
    unsigned long long acc = vlc.acc;
    uint32_t nb = vlc.nbits, pv = vlc.prev;
    for (;;) {                           // complete bytes of the pending bits, with their stuffing
      uint32_t b = (uint32_t)acc & 0xFFu, n = 8;
      if (pv > 0x8F && nb >= 7 && (b & 0x7F) == 0x7F) { b = 0x7F; n = 7; }
      if (nb < n) break;
      ++vl_pos; if (ST) vend[-(int)vl_pos] = (uint8_t)b;
      acc >>= n; nb -= n; pv = b;
    }
    // the unfinished byte: after a byte > 0x8F only 7 bits are available at first (vlc_encode :379-405)
    vl_tmp = (uint32_t)acc & 0xFFu;
    vl_mask = 0xFFu >> (8 - nb);
  }
  if ((mel_mask | vl_mask) != 0) {
    const uint32_t fuse = mel_tmp | vl_tmp;
    if ((((fuse ^ mel_tmp) & mel_mask) | ((fuse ^ vl_tmp) & vl_mask)) == 0 && fuse != 0xFF && vl_pos > 1) {
      if (mel.pos < ES_MEL_BYTES) mel_buf[mel.pos * MS] = (uint8_t)fuse;
      mel.pos++;
    } else {
      if (mel.pos < ES_MEL_BYTES) mel_buf[mel.pos * MS] = (uint8_t)mel_tmp;
      mel.pos++;
      ++vl_pos; if (ST) vend[-(int)vl_pos] = (uint8_t)vl_tmp;
    }
  }
  if (mel.pos > 192 || ms_pos + mel.pos + vl_pos + 8 > slot_cap) {
    if (!ST) { res.len_head = RC_LEN_INVALID; res.len_tail = 0; return; }
    atomicOr(status, mel.pos > 192 ? 2u : 1u);          // the reference errors out on MEL > 192 bytes
    res.len_head = 0; res.len_tail = 0;
    return;
  }
  if (!ST) { res.len_head = ms_pos + mel.pos; res.len_tail = vl_pos; return; }
  for (uint32_t i = 0; i < mel.pos; ++i) slot[ms_pos + i] = mel_buf[i * MS];
  const uint32_t scup = mel.pos + vl_pos;
  vend[-1] = (uint8_t)(scup >> 4);
  vend[-2] = (uint8_t)((vend[-2] & 0xF0) | (scup & 0xF));
  res.len_head = ms_pos + mel.pos;
  res.len_tail = vl_pos;
}

// WIDE: 64-bit sign-magnitude samples (ojph_encode_codeblock64, src/core/coding/ojph_block_encoder.cpp:1026-1523): the same
// pass with p = 62 - missing_msbs, exponents up to 6 bits, MagSgn fields of up to 43 bits appended one sample at a time,
// and the 4-bit U-VLC extension for u_q > 32 (uvlc_tbl entries 33.., :236-247) after the two suffixes (:1491-1492)
// COUNT: the candidate lengths of rate control (rate_ctrl.cu).  Thread i codes block i / kc with its k = i % kc lowest
// magnitude planes dropped (p + k; only k < ncand[block]) and records the length alone in results[i]; nothing is stored
template <bool WIDE, bool COUNT = false>
__global__ void __launch_bounds__(ES_THREADS)
ht_encode_serial_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks,
                        const uint32_t* __restrict__ coef32, uint8_t* __restrict__ slots,
                        EncResult* __restrict__ results, const uint16_t* __restrict__ tables,
                        uint32_t* __restrict__ status, uint32_t prev_quads, uint32_t kc = 1, const uint8_t* __restrict__ ncand = nullptr)
{
  __shared__ uint16_t s_vlc[2 * 2048];
  __shared__ uint16_t s_uvlc[36];
  __shared__ uint8_t s_mel[ES_MEL_BYTES * ES_THREADS];
  OJB_DYN_SMEM(uint16_t, s_prev);          // prev_quads x ES_THREADS: rho | e1 << 4 | e3 << 9 of the row above

  for (uint32_t i = threadIdx.x; i < 2 * 2048; i += blockDim.x) s_vlc[i] = tables[i];
  if (threadIdx.x < 33) s_uvlc[threadIdx.x] = tables[2 * 2048 + threadIdx.x];
  __syncthreads();

  const uint32_t bidx = blockIdx.x * ES_THREADS + threadIdx.x;
  if (bidx >= nblocks) return;
  EncBlock blk;
  if (COUNT) {
    const uint32_t b = bidx / kc, k = bidx - b * kc;
    if (k >= ncand[b]) return;
    blk = blocks[b]; blk.p = (uint16_t)(blk.p + k);
  } else {
    blk = blocks[bidx];
    if (blk.flags & ENC_FLAG_FAST) return;               // coded by ht_encode_split_kernel
  }
  typedef typename WordOf<WIDE>::W W;
  constexpr uint32_t WB = WIDE ? 64u : 32u, EB = WIDE ? 6u : 5u, EM = (1u << EB) - 1u;     // word bits; bits of a stored exponent
  const uint32_t width = blk.w, height = blk.h, stride = blk.stride, p = blk.p;
  const W* __restrict__ src = reinterpret_cast<const W*>(coef32) + blk.src_off;
  uint8_t* slot = COUNT ? nullptr : slots + blk.slot_off;
  uint2* ms_dst = reinterpret_cast<uint2*>(slot);          // slots are 16-byte aligned
  uint32_t* vl_end = reinterpret_cast<uint32_t*>(slot + blk.slot_cap);
  uint8_t* mel_buf = s_mel + threadIdx.x;
  uint16_t* prev = s_prev + threadIdx.x;
  const uint32_t nq = (width + 1) >> 1;
  const uint32_t slot_words = blk.slot_cap >> 2;

  MsWriter ms; ms.w0 = 0; ms.w1 = 0; ms.nbits = 0; ms.words = 0; ms.last_ff = 0;
  // VLC starts as byte 0xFF (later the Scup byte) followed by the four bits 0xF (vlc_init, :365-375)
  VlcWriter vlc; vlc.acc = 0xFFFull; vlc.nbits = 12; vlc.words = 0; vlc.prev = 0;
  MelWriter mel; mel.k = 0; mel.run = 0; mel.tmp = 0; mel.rem = 8; mel.pos = 0;
  uint32_t any_sig = 0, negzero = 0;
  bool overflow = false;
  // aligned block rows: a quad pair of one row is one 16-byte load
  const bool vec4 = !WIDE && ((blk.src_off | stride) & 3u) == 0;
  const bool narrow = !WIDE && p >= 16;    // m_n <= K_max + 1 = 32 - p: four fields of a quad fit 64 bits

  for (uint32_t q = 0; q <= nq; ++q) prev[q * ES_THREADS] = 0;

  for (uint32_t y = 0; y < height; y += 2) {
    const W* r0 = src + (size_t)y * stride;
    const W* r1 = r0 + stride;
    const bool has_r1 = y + 1 < height;
    const uint16_t* vtab = s_vlc + (y ? 2048u : 0u);
    uint32_t rho_left = 0;
    uint32_t pl = 0, pc = prev[0];               // row above: quad q-1, quad q (before being overwritten)

    auto load_pair = [&](uint32_t q, W (&a)[4], W (&b)[4]) {
      // samples 2q .. 2q+3 of the two rows (zero outside the block)
      if (!WIDE && vec4 && 2 * q + 3 < width) {
        const uint4 t = *reinterpret_cast<const uint4*>(r0 + 2 * q);
        a[0] = t.x; a[1] = t.y; a[2] = t.z; a[3] = t.w;
        if (has_r1) { const uint4 u = *reinterpret_cast<const uint4*>(r1 + 2 * q); b[0] = u.x; b[1] = u.y; b[2] = u.z; b[3] = u.w; }
        else { b[0] = b[1] = b[2] = b[3] = 0; }
      } else {
        #pragma unroll
        for (uint32_t i = 0; i < 4; ++i) {
          const bool in = 2 * q + i < width;
          a[i] = in ? r0[2 * q + i] : (W)0;
          b[i] = (in && has_r1) ? r1[2 * q + i] : (W)0;
        }
      }
    };

    W na[4], nb[4];
    load_pair(0, na, nb);
    for (uint32_t q = 0; q < nq; q += 2) {
      W ca[4], cb[4];
      #pragma unroll
      for (int i = 0; i < 4; ++i) { ca[i] = na[i]; cb[i] = nb[i]; }
      if (q + 2 < nq) load_pair(q + 2, na, nb);          // next pair in flight while this one is coded

      uint32_t uq[2] = {0, 0};
      uint32_t pair_bits = 0, pair_len = 0;      // CxtVLC codewords of the pair, then its U-VLC bits (<= 30)
      #pragma unroll
      for (uint32_t h = 0; h < 2; ++h) {
        const uint32_t qq = q + h;
        if (qq >= nq) break;
        // ---- per-sample quantities (:591-643); quad order TL, BL, TR, BR
        const W t[4] = { ca[2 * h], cb[2 * h], ca[2 * h + 1], cb[2 * h + 1] };
        uint32_t rho = 0, e[4] = {0, 0, 0, 0};
        W s[4] = {0, 0, 0, 0};
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          // branch-free: v = 2 * magnitude (0 when insignificant); exponent of 2*mag - 1, MagSgn value
          // 2*(mag - 1) + sign (only read when the sample is significant)
          const W v = ((W)(t[i] + t[i]) >> p) & ~(W)1;
          const uint32_t sig = v ? 1u : 0u;
          rho |= sig << i;
          e[i] = WIDE ? 64u - (uint32_t)__clzll((long long)(v - sig)) : 32u - (uint32_t)__clz((int)(uint32_t)(v - sig));   // v = 0 -> 0
          s[i] = v - 2u + (t[i] >> (WB - 1));
        }
        any_sig |= rho;
        if (blk.flags & ENC_CHECK_NEGZERO) {          // magnitude-overflow words keep the block coded
          const W nz = (W)1 << (WB - 1);
          negzero |= (t[0] == nz) | (t[1] == nz) | (t[2] == nz) | (t[3] == nz);
        }
        const uint32_t emax = max(max(e[0], e[1]), max(e[2], e[3]));
        // ---- context and exponent predictor from the row above
        const uint32_t pr = prev[(qq + 1) * ES_THREADS];      // quad qq+1 of the row above
        uint32_t kappa = 1, cq;
        if (y == 0) cq = (rho_left >> 1) | (rho_left & 1);
        else {
          // max exponent of the four samples above (:862,:950): e3 of NW quad, e1/e3 of N quad, e1 of NE quad
          const uint32_t me = max(max((pl >> (4 + EB)) & EM, (pc >> 4) & EM), max((pc >> (4 + EB)) & EM, (pr >> 4) & EM));
          if (rho & (rho - 1)) kappa = max(1u, me > 0 ? me - 1 : 0u);
          const uint32_t a = ((pl >> 3) | (pc >> 1)) & 1u;
          const uint32_t b = ((rho_left >> 2) | (rho_left >> 3)) & 1u;
          const uint32_t c = ((pc >> 3) | (pr >> 1)) & 1u;
          cq = a | (b << 1) | (c << 2);
        }
        prev[qq * ES_THREADS] = (uint16_t)(rho | (e[1] << 4) | (e[3] << (4 + EB)));
        pl = pc; pc = pr;
        const uint32_t Uq = max(emax, kappa);
        const uint32_t u = Uq - kappa;
        uq[h] = u;
        // which samples reach the maximum exponent (only coded when u > 0); branch-free
        const uint32_t eps = ((e[0] == emax ? 1u : 0u) | (e[1] == emax ? 2u : 0u) | (e[2] == emax ? 4u : 0u) | (e[3] == emax ? 8u : 0u))
                             & (0u - min(u, 1u));
        const uint32_t tuple = vtab[(cq << 8) + (rho << 4) + eps];
        pair_bits |= (tuple >> 8) << pair_len; pair_len += (tuple >> 4) & 7u;      // :661-662
        if (cq == 0) mel_event(mel, rho != 0, mel_buf);                          // :664-665
        {                                                                         // :667-674
          // m_n = sigma_n * (U_q - emb_n) for the four samples at once, one byte each (U_q >= 1, emb_n <= 1)
          uint32_t m[4];
          {
            const uint32_t rb = (rho * 0x00204081u) & 0x01010101u, eb = ((tuple & 15u) * 0x00204081u) & 0x01010101u;
            const uint32_t mb = (Uq * 0x01010101u - eb) & (rb * 0xFFu);
            m[0] = mb & 0xFFu; m[1] = (mb >> 8) & 0xFFu; m[2] = (mb >> 16) & 0xFFu; m[3] = mb >> 24;
          }
          if (WIDE) {                         // fields of up to 43 bits: one append per sample (ms_encode64, :1477-1484)
            #pragma unroll
            for (int i = 0; i < 4; ++i)
              ms_put<!COUNT>(ms, (unsigned long long)s[i] & ((1ull << m[i]) - 1ull), m[i], ms_dst);
          } else {
            const unsigned long long A = (unsigned long long)((uint32_t)s[0] & ((1u << m[0]) - 1u)) |
                                         ((unsigned long long)((uint32_t)s[1] & ((1u << m[1]) - 1u)) << m[0]);
            const unsigned long long B = (unsigned long long)((uint32_t)s[2] & ((1u << m[2]) - 1u)) |
                                         ((unsigned long long)((uint32_t)s[3] & ((1u << m[3]) - 1u)) << m[2]);
            // one append per quad while its four fields fit 64 bits (K_max <= 15), else one per column
            const uint32_t la = m[0] + m[1], lb = m[2] + m[3];
            if (narrow) ms_put<!COUNT>(ms, A | (B << la), la + lb, ms_dst);
            else { ms_put<!COUNT>(ms, A, la, ms_dst); ms_put<!COUNT>(ms, B, lb, ms_dst); }
          }
        }
        rho_left = rho;
      }
      // ---- U-VLC of the pair (:763-785, :985-988)
      {
        const uint32_t u0 = uq[0], u1 = uq[1];
        uint32_t c0, c1;
        // U-VLC code of u: table for u <= 32; beyond it (64-bit samples only) prefix "000", suffix 28 + (u - 33) % 4 and a
        // 4-bit extension (u - 33) / 4
        uint32_t x0 = 0, x1 = 0, xl0 = 0, xl1 = 0;
        auto code = [&](uint32_t u, uint32_t& ext, uint32_t& extl) -> uint32_t {
          if (!WIDE || u <= 32) return s_uvlc[u];
          ext = (u - 33u) >> 2; extl = 4;
          return (3u << 3) | ((28u + ((u - 33u) & 3u)) << 6) | (5u << 11);
        };
        if (y == 0) {
          if (u0 > 0 && u1 > 0) mel_event(mel, min(u0, u1) > 2, mel_buf);
          if (u0 > 2 && u1 > 2) { c0 = code(u0 - 2, x0, xl0); c1 = code(u1 - 2, x1, xl1); }
          else if (u0 > 2 && u1 > 0) { c0 = code(u0, x0, xl0); c1 = (u1 - 1) | (1u << 3); }     // one-bit u1
          else { c0 = code(u0, x0, xl0); c1 = code(u1, x1, xl1); }
        } else { c0 = code(u0, x0, xl0); c1 = code(u1, x1, xl1); }
        // prefixes of both quads, then both suffixes, as one field of at most 3+3+5+5 bits
        uint32_t bits = pair_bits, len = pair_len;
        bits |= (c0 & 7u) << len; len += (c0 >> 3) & 7u;
        bits |= (c1 & 7u) << len; len += (c1 >> 3) & 7u;
        bits |= ((c0 >> 6) & 31u) << len; len += (c0 >> 11) & 31u;
        bits |= ((c1 >> 6) & 31u) << len; len += (c1 >> 11) & 31u;
        vlc_put<!COUNT>(vlc, bits, len, vl_end);
        if (WIDE && (xl0 | xl1)) vlc_put<!COUNT>(vlc, x0 | (x1 << xl0), xl0 + xl1, vl_end);
      }
    }
    if (ms.words + vlc.words + 24 >= slot_words) { overflow = true; break; }
  }

  if (overflow) {
    if (!COUNT) atomicOr(status, 1u);
    results[bidx].len_head = COUNT ? RC_LEN_INVALID : 0; results[bidx].len_tail = 0; return;
  }
  if (any_sig == 0 && negzero == 0) { results[bidx].len_head = 0; results[bidx].len_tail = 0; return; }   // block not included

  terminate_block<ES_THREADS, !COUNT>(ms, vlc, mel, mel_buf, slot, blk.slot_cap, status, results[bidx]);
}

// ---- fast path: two threads per code-block -------------------------------------------------------------------
// The same encoder for the blocks the host marks ENC_FLAG_FAST: width a multiple of 4 and at most 64, even
// height, 16-byte aligned rows, K_max <= 15 (the four MagSgn fields of a quad fit 64 bits; 2 * magnitude - 1 fits
// 16 bits), no magnitude-overflow check.  Without the per-quad bounds / width / precision tests, and with the
// row above kept as
//   * a 64-bit register of bottom-sample significance bits (two per quad, walked four bits per pair) and
//   * one word per quad pair of g[q] = x(br of quad q-1) | x(bl of quad q), x = 2 * magnitude - 1: the largest
//     exponent of the four samples above a quad is 32 - clz(g[q] | g[q+1]) -- one CLZ instead of a 4-way max of
//     stored exponents; inside the quad the largest exponent is 32 - clz(x0 | x1 | x2 | x3) and a sample reaches it
//     iff x_i >> (e_max - 1) is non-zero.
// Thread A of a block (warps 0-1 of the CTA) does everything that touches the samples: magnitudes, exponents,
// contexts, the CxtVLC table look-up, and the MagSgn stream; per quad pair it hands thread B (warps 2-3) one word
// -- the pair's CxtVLC bits and length, the two u_q, and which MEL events the pair produces -- through a
// double-buffered shared-memory row.  B runs the adaptive MEL coder, the U-VLC tables and the backward VLC writer,
// and terminates the block.  One direction only (A never needs anything from B), hand-over per quad-row with named
// barriers as in the decoder.  The serial chain per block -- what bounds this kernel when one frame's 49 152 blocks
// are all that is in flight -- loses the VLC / MEL part, and a CTA holds twice the warps.
#define SE_BLOCKS 64
struct SplitTail { unsigned long long w0; uint32_t nbits, words, last_ff, any_sig, overflow, pad; };
__global__ void __launch_bounds__(2 * SE_BLOCKS)
ht_encode_split_kernel(const EncBlock* __restrict__ blocks, uint32_t nblocks,
                       const uint32_t* __restrict__ coef, uint8_t* __restrict__ slots,
                       EncResult* __restrict__ results, const uint16_t* __restrict__ tables,
                       uint32_t* __restrict__ status)
{
  __shared__ uint16_t s_vlc[2 * 2048];
  __shared__ uint16_t s_uvlc[36];
  __shared__ uint8_t s_mel[ES_MEL_BYTES * SE_BLOCKS];
  __shared__ uint32_t s_g[17 * SE_BLOCKS];
  __shared__ uint32_t s_rec[2 * 16 * SE_BLOCKS];            // [stage][pair][block]
  __shared__ SplitTail s_tail[SE_BLOCKS];
  __shared__ uint32_t s_rows;

  for (uint32_t i = threadIdx.x; i < 2 * 2048; i += blockDim.x) s_vlc[i] = tables[i];
  if (threadIdx.x < 33) s_uvlc[threadIdx.x] = tables[2 * 2048 + threadIdx.x];
  if (threadIdx.x == 0) s_rows = 0;
  __syncthreads();

  const bool side_a = threadIdx.x < SE_BLOCKS;
  const uint32_t tid = side_a ? threadIdx.x : threadIdx.x - SE_BLOCKS;
  const uint32_t bidx = blockIdx.x * SE_BLOCKS + tid;
  EncBlock blk;
  bool active = bidx < nblocks;
  if (active) { blk = blocks[bidx]; active = (blk.flags & ENC_FLAG_FAST) != 0; }
  const uint32_t npairs = active ? (uint32_t)(blk.w >> 2) : 0u, myrows = active ? (uint32_t)(blk.h >> 1) : 0u;
  if (side_a && myrows) atomicMax(&s_rows, myrows);
  __syncthreads();
  const uint32_t rows = s_rows;
  enum { BAR_FULL = 1, BAR_EMPTY = 3 };
  uint8_t* slot = active ? slots + blk.slot_off : nullptr;
  // the VLC segment's worst case (30 bits per quad pair, one stuffing bit in seven, margin), as the host sized it
  uint32_t vl_worst = 0;
  if (active) {
    const uint32_t nqp = ((uint32_t)(blk.w >> 1) * (uint32_t)(blk.h >> 1) + 1u) / 2u;
    vl_worst = (nqp * 30u + 12u + 7u) / 8u; vl_worst += vl_worst / 7u + 8u;
  }

  if (side_a) {
    const uint32_t stride = active ? blk.stride : 0u, p = active ? (uint32_t)blk.p : 16u;
    const uint32_t* __restrict__ src = active ? coef + blk.src_off : coef;
    uint2* ms_dst = reinterpret_cast<uint2*>(slot);
    uint32_t* gw = s_g + tid;
    const uint32_t pm1 = p - 1u, vmask = (2u << (31u - p)) - 2u;
    // MagSgn cannot exceed its worst case ((K_max + 1) bits per sample, a stuffing bit per 15, as the host sized the
    // slot); the test below is a safety net that keeps a faulty run out of the VLC side's part of the slot
    uint32_t ms_limit = 0;
    if (active) {
      uint32_t mw = ((uint32_t)blk.w * blk.h * (32u - p) + 7u) / 8u; mw += mw / 15u + 8u;
      ms_limit = (mw + 48u) >> 2;
    }
    MsWriter ms; ms.w0 = 0; ms.w1 = 0; ms.nbits = 0; ms.words = 0; ms.last_ff = 0;
    uint32_t any_sig = 0, overflow = 0;
    if (active) for (uint32_t j = 0; j <= 16; ++j) gw[j * SE_BLOCKS] = 0;
    uint32_t sg_lo = 0, sg_hi = 0;
    for (uint32_t r = 0; r < rows; ++r) {
      if (r >= 2) named_bar_sync(BAR_EMPTY + (r & 1), 2 * SE_BLOCKS);
      if (r < myrows && !overflow) {
        const bool first = (r == 0);
        const uint4* r0 = reinterpret_cast<const uint4*>(src + (size_t)(2 * r) * stride);
        const uint4* r1 = reinterpret_cast<const uint4*>(src + (size_t)(2 * r + 1) * stride);
        const uint16_t* vtab = s_vlc + (first ? 0u : 2048u);
        uint32_t* out = s_rec + (size_t)(r & 1) * 16 * SE_BLOCKS + tid;
        uint32_t rho_left = 0;
        uint32_t rs_lo = sg_lo, rs_hi = sg_hi, rs_carry = 0;
        uint32_t cu_lo = 0, cu_hi = 0;
        uint32_t wj = gw[0], x_carry = 0;
        uint4 na = ld_stream16(r0), nb = ld_stream16(r1);
        #pragma unroll 1
        for (uint32_t j = 0; j < npairs; ++j) {
          const uint4 ca = na, cb = nb;
          if (j + 1 < npairs) { na = ld_stream16(r0 + j + 1); nb = ld_stream16(r1 + j + 1); }
          const uint32_t wj1 = gw[(j + 1) * SE_BLOCKS];
          const uint32_t y6 = rs_carry | ((rs_lo & 0x1Fu) << 1);
          const uint32_t z = y6 | (y6 >> 1);
          rs_carry = (rs_lo >> 3) & 1u;
          rs_lo = __funnelshift_r(rs_lo, rs_hi, 4); rs_hi >>= 4;
          const uint32_t gor[2] = { (wj | (wj >> 16)) & 0xFFFFu, (wj >> 16) | (wj1 & 0xFFFFu) };
          wj = wj1;
          uint32_t uq[2], xb[2][2], rr[2], cwl[2], melf = 0;
          unsigned long long cwd[2];
          uint32_t pair_bits = 0, pair_len = 0;
          #pragma unroll
          for (uint32_t h = 0; h < 2; ++h) {
            const uint32_t t[4] = { h ? ca.z : ca.x, h ? cb.z : cb.x, h ? ca.w : ca.y, h ? cb.w : cb.y };
            uint32_t rho = 0, x[4], s[4];
            #pragma unroll
            for (int i = 0; i < 4; ++i) {
              const uint32_t v = (t[i] >> pm1) & vmask;
              const uint32_t sig = min(v, 1u);
              rho |= sig << i;
              x[i] = v - sig;
              s[i] = v - 2u + (t[i] >> 31);
            }
            any_sig |= rho;
            rr[h] = rho;
            xb[h][0] = x[1]; xb[h][1] = x[3];
            const uint32_t emax = 32u - (uint32_t)__clz((int)(x[0] | x[1] | x[2] | x[3]));
            uint32_t kappa = 1, cq;
            if (first) cq = (rho_left >> 1) | (rho_left & 1);
            else {
              const int me = 32 - __clz((int)gor[h]);
              if (rho & (rho - 1)) kappa = (uint32_t)max(1, me - 1);
              cq = ((z >> (2 * h)) & 5u) | (rho_left > 3u ? 2u : 0u);
            }
            const uint32_t Uq = max(emax, kappa);
            const uint32_t u = Uq - kappa;
            uq[h] = u;
            const uint32_t sh = max(emax, 1u) - 1u;
            const uint32_t eps = ((x[0] >> sh) | ((x[1] >> sh) << 1) | ((x[2] >> sh) << 2) | ((x[3] >> sh) << 3)) & (0u - min(u, 1u));
            const uint32_t tuple = vtab[(cq << 8) + (rho << 4) + eps];
            pair_bits |= (tuple >> 8) << pair_len; pair_len += (tuple >> 4) & 7u;
            melf |= ((cq == 0 ? 1u : 0u) | (rho != 0 ? 2u : 0u)) << (2 * h);       // MEL event of this quad, and its value
            {
              const uint32_t rb = (rho * 0x00204081u) & 0x01010101u, eb = ((tuple & 15u) * 0x00204081u) & 0x01010101u;
              const uint32_t mb = (Uq * 0x01010101u - eb) & (rb * 0xFFu);
              const uint32_t m0 = mb & 0xFFu, m1 = (mb >> 8) & 0xFFu, m2 = (mb >> 16) & 0xFFu, m3 = mb >> 24;
              const uint32_t A = (s[0] & ((1u << m0) - 1u)) | ((s[1] & ((1u << m1) - 1u)) << m0);
              const uint32_t B = (s[2] & ((1u << m2) - 1u)) | ((s[3] & ((1u << m3) - 1u)) << m2);
              const uint32_t la = m0 + m1, lb = m2 + m3;
              cwd[h] = (unsigned long long)A | ((unsigned long long)B << la); cwl[h] = la + lb;
            }
            rho_left = rho;
          }
          // the pair's hand-over word: CxtVLC bits (<= 14) | their length << 14 | MEL flags << 18 | u_q0 << 22 | u_q1 << 27
          out[j * SE_BLOCKS] = pair_bits | (pair_len << 14) | (melf << 18) | (uq[0] << 22) | (uq[1] << 27);
          ms_put(ms, cwd[0], cwl[0], ms_dst);
          ms_put(ms, cwd[1], cwl[1], ms_dst);
          {
            const uint32_t ta = (rr[0] >> 1) & 5u, tb = (rr[1] >> 1) & 5u;
            const uint32_t nbits4 = ((ta | (ta >> 1)) & 3u) | (((tb | (tb >> 1)) & 3u) << 2);
            cu_lo = __funnelshift_r(cu_lo, cu_hi, 4); cu_hi = (cu_hi >> 4) | (nbits4 << 28);
            gw[j * SE_BLOCKS] = (x_carry | xb[0][0]) | ((xb[0][1] | xb[1][0]) << 16);
            x_carry = xb[1][1];
          }
        }
        gw[npairs * SE_BLOCKS] = x_carry;
        const uint32_t sh = 64u - 4u * npairs;
        const uint32_t a0 = sh >= 32 ? cu_hi : cu_lo, a1 = sh >= 32 ? 0u : cu_hi;
        sg_lo = __funnelshift_r(a0, a1, sh & 31u); sg_hi = a1 >> (sh & 31u);
        if (ms.words > ms_limit) overflow = 1;
      }
      __threadfence_block();
      named_bar_arrive(BAR_FULL + (r & 1), 2 * SE_BLOCKS);
    }
    if (active) {
      SplitTail& t = s_tail[tid];
      t.w0 = ms.w0; t.nbits = ms.nbits; t.words = ms.words; t.last_ff = ms.last_ff; t.any_sig = any_sig; t.overflow = overflow;
    }
    __syncthreads();
    return;
  }

  // ---- side B: MEL, U-VLC, the VLC stream, termination
  uint32_t* vl_end = active ? reinterpret_cast<uint32_t*>(slot + blk.slot_cap) : nullptr;
  uint8_t* mel_buf = s_mel + tid;
  VlcWriter vlc; vlc.acc = 0xFFFull; vlc.nbits = 12; vlc.words = 0; vlc.prev = 0;
  MelWriter mel; mel.k = 0; mel.run = 0; mel.tmp = 0; mel.rem = 8; mel.pos = 0;
  uint32_t overflow_b = 0;
  for (uint32_t r = 0; r < rows; ++r) {
    named_bar_sync(BAR_FULL + (r & 1), 2 * SE_BLOCKS);
    if (r < myrows && !overflow_b) {
      const bool first = (r == 0);
      const uint32_t* in = s_rec + (size_t)(r & 1) * 16 * SE_BLOCKS + tid;
      #pragma unroll 1
      for (uint32_t j = 0; j < npairs; ++j) {
        const uint32_t w = in[j * SE_BLOCKS];
        const uint32_t melf = (w >> 18) & 15u, u0 = (w >> 22) & 31u, u1 = w >> 27;
        if (melf & 1u) mel_event<SE_BLOCKS>(mel, (melf & 2u) != 0, mel_buf);                  // :664-665
        if (melf & 4u) mel_event<SE_BLOCKS>(mel, (melf & 8u) != 0, mel_buf);
        uint32_t c0, c1;
        if (first) {
          if (u0 > 0 && u1 > 0) mel_event<SE_BLOCKS>(mel, min(u0, u1) > 2, mel_buf);
          if (u0 > 2 && u1 > 2) { c0 = s_uvlc[u0 - 2]; c1 = s_uvlc[u1 - 2]; }
          else if (u0 > 2 && u1 > 0) { c0 = s_uvlc[u0]; c1 = (u1 - 1) | (1u << 3); }     // one-bit u1
          else { c0 = s_uvlc[u0]; c1 = s_uvlc[u1]; }
        } else { c0 = s_uvlc[u0]; c1 = s_uvlc[u1]; }
        uint32_t bits = w & 0x3FFFu, len = (w >> 14) & 15u;
        bits |= (c0 & 7u) << len; len += (c0 >> 3) & 7u;
        bits |= (c1 & 7u) << len; len += (c1 >> 3) & 7u;
        bits |= ((c0 >> 6) & 31u) << len; len += (c0 >> 11) & 31u;
        bits |= ((c1 >> 6) & 31u) << len; len += (c1 >> 11) & 31u;
        vlc_put(vlc, bits, len, vl_end);
      }
      if (vlc.words * 4u >= vl_worst + 48u) overflow_b = 1;      // (cannot happen: vl_worst bounds the segment; the reserve is vl_worst + 64)
    }
    if (r + 2 < rows) named_bar_arrive(BAR_EMPTY + (r & 1), 2 * SE_BLOCKS);
  }
  __syncthreads();
  if (!active) return;
  const SplitTail t = s_tail[tid];
  if (t.overflow || overflow_b) { atomicOr(status, 1u); results[bidx].len_head = 0; results[bidx].len_tail = 0; return; }
  if (t.any_sig == 0) { results[bidx].len_head = 0; results[bidx].len_tail = 0; return; }   // block not included
  MsWriter ms; ms.w0 = t.w0; ms.w1 = 0; ms.nbits = t.nbits; ms.words = t.words; ms.last_ff = t.last_ff;
  terminate_block<SE_BLOCKS>(ms, vlc, mel, mel_buf, slot, blk.slot_cap, status, results[bidx]);
}

} // namespace

void launch_ht_encode_serial(const EncBlock* blocks, uint32_t nblocks, uint32_t nfast, uint32_t max_width, const uint32_t* coef,
                             uint8_t* slots, EncResult* results, const uint16_t* tables, uint32_t* status,
                             cudaStream_t st, bool wide, const SideStream* side)
{
  if (nblocks == 0) return;
  if (wide) nfast = 0;
  // both kernels to run: the general one goes to the side stream
  const bool forked = side && side->st && nfast && nfast < nblocks && !wide;
  cudaStream_t sg = forked ? side->st : st;
  if (forked) { cudaEventRecord(side->fork, st); cudaStreamWaitEvent(side->st, side->fork, 0); }
  const uint32_t prev_quads = (max_width + 1) / 2 + 2;
  const size_t smem = (size_t)prev_quads * ES_THREADS * sizeof(uint16_t);
  cudaFuncSetAttribute(ht_encode_serial_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(ht_encode_serial_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((nblocks + ES_THREADS - 1) / ES_THREADS), block(ES_THREADS);
  if (nfast) {           // blocks flagged ENC_FLAG_FAST: two threads per block
    dim3 g2((nblocks + SE_BLOCKS - 1) / SE_BLOCKS), b2(2 * SE_BLOCKS);
    OJB_LAUNCH(ht_encode_split_kernel, g2, b2, 0, st, blocks, nblocks, coef, slots, results, tables, status);
  }
  if (wide)
    OJB_LAUNCH(ht_encode_serial_kernel<true>, grid, block, smem, st, blocks, nblocks, coef, slots, results, tables, status,
               prev_quads);
  else if (nfast < nblocks)
    OJB_LAUNCH(ht_encode_serial_kernel<false>, grid, block, smem, sg, blocks, nblocks, coef, slots, results, tables, status,
               prev_quads);
  if (forked) { cudaEventRecord(side->join, side->st); cudaStreamWaitEvent(st, side->join, 0); }
}

void launch_ht_encode_lengths(const EncBlock* blocks, uint32_t nblocks, uint32_t kc, const uint8_t* ncand, uint32_t max_width,
                              const uint32_t* coef, EncResult* lengths, const uint16_t* tables, cudaStream_t st)
{
  const uint32_t n = nblocks * kc;
  if (n == 0) return;
  const uint32_t prev_quads = (max_width + 1) / 2 + 2;
  const size_t smem = (size_t)prev_quads * ES_THREADS * sizeof(uint16_t);
  cudaFuncSetAttribute(ht_encode_serial_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  OJB_LAUNCH((ht_encode_serial_kernel<false, true>), dim3((n + ES_THREADS - 1) / ES_THREADS), dim3(ES_THREADS), smem, st,
             blocks, n, coef, nullptr, lengths, tables, nullptr, prev_quads, kc, ncand);
}

} // namespace ojb
