// ht_decode.cu -- HTJ2K block decoder for sm_90a: cleanup pass (+ SigProp + MagRef).
//
// Results are those of the reference's ojph_decode_codeblock32
// (src/core/coding/ojph_block_decoder32.cpp:742-1612).  One kernel per block class:
//   * ht_decode_split_kernel: cleanup-only blocks of the common shape (DEC_FLAG_FAST), a producer /
//     consumer thread pair per code-block, see the comment above it;
//   * ht_decode_serial_kernel: every other block, the whole cleanup pass by ONE THREAD per code-block
//     (lock-step 64-bit refills of 128-bit bit windows), then SPP / MRP (only present in streams from
//     other encoders);
//   * ht_decode_wide_kernel: 64-bit samples.
// The de-quantisation the reference does line by line afterwards (tx_from_cb32,
// src/core/codestream/ojph_codestream_gen.cpp:124-168) is fused into the final store.
#include "ojb_device.h"
#include "ojb_kernels.h"
#include "ojb_async.cuh"
#include "dequant.cuh"

namespace ojb {

#define DEC_WARPS 4

// block status bits
#define DST_FAIL 1u
#define DST_EMPTY 2u              // serial decoder: block not included, to be zero-filled
#define DEC1_THREADS 128        // thread-per-block kernels: threads per CTA

namespace {

struct DecTables {            // shared-memory copy
  uint16_t vlc0[1024], vlc1[1024], uvlc0[320], uvlc1[256];
};

// ---- MEL / VLC readers (thread-private): 32 bits per refill, as the reference's mel_read /
// rev_read do (ojph_block_decoder32.cpp:92-152, :307-357), built from aligned word loads

struct MelDec {
  const uint8_t* p; int size; unsigned long long tmp; int bits; bool unstuff; int k;
  // the aligned words that hold the next four bytes, requested one refill ahead (the funnel shift
  // that needs them runs at the next refill, so the load latency is off the critical chain)
  const uint32_t* wp; uint32_t lo, hi, sh;
};
__device__ __forceinline__ void mel_prime(MelDec& m) {
  m.wp = reinterpret_cast<const uint32_t*>((size_t)m.p & ~(size_t)3);
  m.sh = (uint32_t)((size_t)m.p & 3) * 8;
  m.lo = m.wp[0]; m.hi = m.wp[1];
}
__device__ __forceinline__ void mel_fill(MelDec& m) {       // MSB first; needs bits <= 32 on entry
  if (m.bits > 32) return;
  uint32_t val;
  if (m.size > 4) {
    val = m.sh ? __funnelshift_r(m.lo, m.hi, m.sh) : m.lo;
    m.p += 4; m.size -= 4;
    m.lo = m.hi; m.wp += 1; m.hi = m.wp[1];
  } else {
    val = 0xFFFFFFFFu;                                        // 0xFF fed past the end
    int i = 0;
    while (m.size > 0) {
      uint32_t v = *m.p++;
      if (m.size == 1) v |= 0xF;                              // MEL and VLC may share the last byte
      val = (val & ~(0xFFu << i)) | (v << i);
      --m.size; i += 8;
    }
  }
  uint32_t t = 0; int nb = 0;
  bool us = m.unstuff;
  uint32_t ff = val & (val >> 1); ff &= ff >> 2; ff &= ff >> 4;      // bit 8i set <=> byte i == 0xFF
  if (!us && (ff & 0x00010101u) == 0) {                              // no stuffed byte among the four
    t = __byte_perm(val, 0, 0x0123); nb = 32; us = (ff >> 24) & 1u;
  } else {
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t d = (val >> (8 * i)) & 0xFFu;
      const int n = 8 - (us ? 1 : 0);
      t = (t << n) | (d & ((1u << n) - 1u));
      nb += n;
      us = (d == 0xFF);
    }
  }
  m.unstuff = us;
  m.tmp |= (unsigned long long)t << (64 - nb - m.bits);
  m.bits += nb;
}
// one run code (mel_decode, :170-208): 2*z+1 = z zero events then a one; 2*(2^E - 1) = 2^E zeros
__device__ __forceinline__ int mel_next_run(MelDec& m) {
  if (m.bits < 6) mel_fill(m);
  const int eval = (int)((0x5433222111000ull >> (4 * m.k)) & 7ull);
  int run;
  if (m.tmp & (1ull << 63)) {
    run = ((1 << eval) - 1) << 1;
    m.k = m.k < 12 ? m.k + 1 : 12;
    m.tmp <<= 1; m.bits -= 1;
  } else {
    run = (int)(m.tmp >> (63 - eval)) & ((1 << eval) - 1);
    m.k = m.k > 0 ? m.k - 1 : 0;
    m.tmp <<= eval + 1; m.bits -= eval + 1;
    run = (run << 1) + 1;
  }
  return run;
}

struct RevDec {               // backward-growing stream (VLC, MRP)
  const uint8_t* p; int size; unsigned long long tmp; uint32_t bits; bool unstuff;
  // rev_fill32: the stream is read backward one aligned word per refill.  The words are requested
  // VLC_RING-1 refills ahead with cp.async into a per-thread ring in shared memory (global/L2
  // latency is several refill periods for one serial chain per thread); `lo`/`hi` hold the two
  // words the next refill's funnel shift needs.
  const uint32_t* wnext; const uint32_t* wbase; uint32_t* ring; uint32_t ridx, lo, hi, sh;
};
#ifndef VLC_RING
#define VLC_RING 8
#endif
template <int STRIDE = DEC1_THREADS>
__device__ __forceinline__ void rev_ring_issue(RevDec& v) {
  uint32_t* slot = v.ring + v.ridx * STRIDE;
  if (v.wnext >= v.wbase) cp_async<4>(slot, v.wnext); else *slot = 0u;
  cp_commit();
  --v.wnext; v.ridx = (v.ridx + 1) & (VLC_RING - 1);
}
template <int STRIDE = DEC1_THREADS>
__device__ __forceinline__ void rev_prime(RevDec& v, const uint8_t* buffer_start, uint32_t* ring) {
  const uint8_t* q = v.p - 3;
  const uint32_t* wp = reinterpret_cast<const uint32_t*>((size_t)q & ~(size_t)3);
  v.wbase = reinterpret_cast<const uint32_t*>((size_t)buffer_start & ~(size_t)3);
  v.sh = (uint32_t)((size_t)q & 3) * 8;
  v.lo = (wp >= v.wbase) ? wp[0] : 0u;
  v.hi = (wp + 1 >= v.wbase) ? wp[1] : 0u;
  v.ring = ring; v.ridx = 0; v.wnext = wp - 1;
  #pragma unroll
  for (int i = 0; i < VLC_RING - 1; ++i) rev_ring_issue<STRIDE>(v);
  v.ridx = 0;                                  // oldest request sits in slot 0
}
// byte-wise refill (refinement passes)
__device__ __forceinline__ void rev_fill(RevDec& v) {       // LSB first
  while (v.bits <= 56) {
    uint32_t d = 0;
    if (v.size > 0) { d = *v.p--; --v.size; }
    uint32_t nb = 8 - ((v.unstuff && (d & 0x7F) == 0x7F) ? 1u : 0u);
    v.unstuff = d > 0x8F;
    d &= (1u << nb) - 1u;
    v.tmp |= (unsigned long long)d << v.bits;
    v.bits += nb;
  }
}
// 32 bits per refill; needs bits <= 32 on entry
template <int STRIDE = DEC1_THREADS>
__device__ __forceinline__ void rev_fill32(RevDec& v) {
  if (v.bits > 32) return;
  uint32_t val = 0;                                           // bytes p-3 .. p, byte p in the MSB
  if (v.size > 3) {
    val = v.sh ? __funnelshift_r(v.lo, v.hi, v.sh) : v.lo;
    v.p -= 4; v.size -= 4;
    v.hi = v.lo;
    cp_wait<VLC_RING - 2>();                                  // the oldest request has landed
    const uint32_t take = v.ridx;
    v.lo = v.ring[take * STRIDE];
    // the freed slot takes the request VLC_RING-1 words further down the stream
    v.ridx = (take + VLC_RING - 1) & (VLC_RING - 1);
    rev_ring_issue<STRIDE>(v);
    v.ridx = (take + 1) & (VLC_RING - 1);
  } else {
    int i = 24;
    while (v.size > 0) { val |= (uint32_t)(*v.p--) << i; --v.size; i -= 8; }
  }
  uint32_t t = 0, nb = 0;
  bool us = v.unstuff;
  // a byte whose low 7 bits are 0x7F and whose predecessor (the byte consumed before it) is > 0x8F
  // carries 7 bits; all four bytes are tested at once and the byte loop runs only when one does
  const uint32_t pv = (val >> 8) | (us ? 0x90000000u : 0u);
  if (((((val & 0x7F7F7F7Fu) + 0x01010101u) & pv & ((pv & 0x70707070u) + 0x70707070u)) & 0x80808080u) == 0) {
    t = __byte_perm(val, 0, 0x0123); nb = 32; us = (val & 0xFFu) > 0x8Fu;
  } else {
    #pragma unroll
    for (int i = 3; i >= 0; --i) {
      const uint32_t d = (val >> (8 * i)) & 0xFFu;
      const uint32_t n = 8 - ((us && (d & 0x7F) == 0x7F) ? 1u : 0u);
      t |= (d & ((1u << n) - 1u)) << nb;
      nb += n;
      us = d > 0x8F;
    }
  }
  v.unstuff = us;
  v.tmp |= (unsigned long long)t << v.bits;
  v.bits += nb;
}

// simple byte-wise readers for the refinement passes
struct FwdBits {              // SPP: forward, 0 fed when exhausted, 7-bit byte after 0xFF
  const uint8_t* p; int size; unsigned long long tmp; uint32_t bits; bool unstuff;
};
__device__ __forceinline__ void fwd_fill(FwdBits& f) {
  while (f.bits <= 56) {
    uint32_t d = 0;
    if (f.size > 0) { d = *f.p++; --f.size; }
    uint32_t nb = 8 - (f.unstuff ? 1u : 0u);
    f.unstuff = (d == 0xFF);
    d &= (1u << nb) - 1u;
    f.tmp |= (unsigned long long)d << f.bits; f.bits += nb;
  }
}
__device__ __forceinline__ uint32_t fwd_get(FwdBits& f) {
  if (f.bits == 0) fwd_fill(f);
  uint32_t b = (uint32_t)f.tmp & 1u; f.tmp >>= 1; --f.bits; return b;
}

__device__ __forceinline__ uint32_t rec_rho(const uint32_t* rec, uint32_t qstride, uint32_t x, uint32_t y,
                                            uint32_t width, uint32_t height) {
  if (x >= width || y >= height) return 0;
  uint32_t r = rec[(size_t)(y >> 1) * qstride + (x >> 1)];
  return ((r >> 4) >> (2 * (x & 1) + (y & 1))) & 1u;
}

// SigProp + MagRef, serial restatement executed by the block's thread on its sign-magnitude
// samples (ojph_block_decoder32.cpp:1318-1612)
__device__ void refine_passes(const DecBlock& blk, uint32_t np, const uint8_t* data, uint32_t* dst,
                              const uint32_t* rec, uint32_t qstride, uint32_t p)
{
  const uint32_t width = blk.w, height = blk.h, stride = blk.stride;
  const bool causal = (blk.flags & 1) != 0;
  // ---- significance propagation
  {
    FwdBits sp; sp.p = data + blk.len1; sp.size = (int)blk.len2; sp.tmp = 0; sp.bits = 0; sp.unstuff = false;
    const uint32_t val = 3u << (p - 2);
    for (uint32_t y0 = 0; y0 < height; y0 += 4) {
      uint32_t prev_col = 0;    // final neighbourhood flags (rows 0..3) of the column left of the group
      for (uint32_t x0 = 0; x0 < width; x0 += 4) {
        // V(c, j): vertically integrated significance of column c at stripe row j, CUP-only
        // for columns of this and the next group (plus row above: final, row below: CUP)
        uint32_t V[6];           // columns x0-1 .. x0+4
        uint32_t cs[4];
        for (int ci = 0; ci < 5; ++ci) {
          const uint32_t c = x0 + (uint32_t)ci;
          uint32_t col = 0;
          for (uint32_t j = 0; j < 4; ++j) col |= rec_rho(rec, qstride, c, y0 + j, width, height) << j;
          if (ci < 4) cs[ci] = col;
          uint32_t v = col | ((col & 7u) << 1) | ((col & 14u) >> 1);
          if (c < width) {
            if (y0 > 0 && dst[(size_t)(y0 - 1) * stride + c] != 0) v |= 1u;          // row above: final state
            if (!causal && rec_rho(rec, qstride, c, y0 + 4, width, height)) v |= 8u;  // row below: CUP only
          }
          V[ci + 1] = v;
        }
        V[0] = prev_col;
        uint32_t cand[4], newsig[4] = {0, 0, 0, 0};
        uint32_t inside[4];
        for (int i = 0; i < 4; ++i) {
          uint32_t in = 0;
          for (uint32_t j = 0; j < 4; ++j) if (x0 + i < width && y0 + j < height) in |= 1u << j;
          inside[i] = in;
          cand[i] = (V[i] | V[i + 1] | V[i + 2]) & in & ~cs[i];
        }
        uint32_t nnew = 0;
        for (int i = 0; i < 4; ++i)
          for (uint32_t j = 0; j < 4; ++j) {
            if (!((cand[i] >> j) & 1u)) continue;
            if (fwd_get(sp)) {
              newsig[i] |= 1u << j; ++nnew;
              // neighbours later in scan order become candidates (:1452-1492)
              uint32_t own = (j < 3 ? (2u << j) : 0u);                         // sample below
              uint32_t nxt = (1u << j) | (j ? (1u << (j - 1)) : 0u) | (j < 3 ? (2u << j) : 0u);
              cand[i] |= own & inside[i] & ~cs[i];
              if (i < 3) cand[i + 1] |= nxt & inside[i + 1] & ~cs[i + 1];
            }
          }
        if (nnew)
          for (int i = 0; i < 4; ++i)
            for (uint32_t j = 0; j < 4; ++j)
              if ((newsig[i] >> j) & 1u)
                dst[(size_t)(y0 + j) * stride + x0 + i] = (fwd_get(sp) << 31) | val;
        // state handed to the next group: last column, final significance, vertically integrated
        {
          uint32_t f = cs[3] | newsig[3];
          uint32_t v = f | ((f & 7u) << 1) | ((f & 14u) >> 1);
          v |= V[4] & 9u & ~0u;    // row-above / row-below contributions of that column
          prev_col = v;
        }
      }
    }
  }
  // ---- magnitude refinement
  if (np > 2) {
    RevDec mr; mr.p = data + blk.len1 + blk.len2 - 1; mr.size = (int)blk.len2; mr.tmp = 0; mr.bits = 0;
    mr.unstuff = true;
    const uint32_t half = 1u << (p - 2);
    for (uint32_t y0 = 0; y0 < height; y0 += 4)
      for (uint32_t x0 = 0; x0 < width; x0 += 8) {
        for (uint32_t i = 0; i < 8; ++i)
          for (uint32_t j = 0; j < 4; ++j) {
            if (!rec_rho(rec, qstride, x0 + i, y0 + j, width, height)) continue;
            if (mr.bits == 0) rev_fill(mr);
            uint32_t sym = (uint32_t)mr.tmp & 1u; mr.tmp >>= 1; --mr.bits;
            dst[(size_t)(y0 + j) * stride + x0 + i] ^= ((1u - sym) << (p - 1)) | half;
          }
      }
  }
}

// ---- whole cleanup pass, one thread per code-block ---------------------------------------------
// The serial form of the decoder (what ojph_decode_codeblock32 does, :742-1316, in one pass instead of
// its two): the thread that decodes a quad pair's VLC / U-VLC codewords reads the pair's MagSgn bits
// right away, so no quad records travel through memory.  Blocks that carry SPP / MRP passes still write
// their quad records to the scratch area (refine_passes needs the CUP significance).
// ---- bit readers of the thread-per-block decoder ------------------------------------------------
// Both streams are read as aligned 8-byte groups through per-thread cp.async rings; a group is un-stuffed
// as a whole (the positions to delete come from one SWAR test, the usual group has none) and appended to a
// 128-bit window (w1:w0).  The caller tops a window up to >= 64 bits at ONE point per quad (MagSgn) or
// quad pair (VLC) -- the same point for every lane of the warp, so the refill is a piece of straight-line
// code the whole warp runs together instead of a branch a few lanes take at a time -- and then reads its
// fields from w0 without further checks.
struct Win128 { unsigned long long w0, w1; uint32_t bits; };
// append the low c bits of val (upper bits zero); needs bits < 64
__device__ __forceinline__ void win_append(Win128& w, unsigned long long val, uint32_t c) {
  w.w1 = (val >> 1) >> (63u - w.bits);
  w.w0 |= val << w.bits;
  w.bits += c;
}
// drop n (0..64) bits
__device__ __forceinline__ void win_drop(Win128& w, uint32_t n) {
  uint32_t a0 = (uint32_t)w.w0, a1 = (uint32_t)(w.w0 >> 32), a2 = (uint32_t)w.w1, a3 = (uint32_t)(w.w1 >> 32);
  const bool big = n >= 32;
  a0 = big ? a1 : a0; a1 = big ? a2 : a1; a2 = big ? a3 : a2; a3 = big ? 0u : a3;
  const uint32_t rr = (n == 64) ? 32u : (n & 31u);
  const uint32_t b0 = __funnelshift_rc(a0, a1, rr), b1 = __funnelshift_rc(a1, a2, rr), b2 = __funnelshift_rc(a2, a3, rr),
                 b3 = __funnelshift_rc(a3, 0u, rr);
  w.w0 = (unsigned long long)b0 | ((unsigned long long)b1 << 32);
  w.w1 = (unsigned long long)b2 | ((unsigned long long)b3 << 32);
  w.bits -= n;
}
// delete the bits of val marked in del (highest first, so lower positions stay valid); returns how many
__device__ __forceinline__ uint32_t delete_bits(unsigned long long& val, unsigned long long del) {
  uint32_t n = 0;
  while (del) {
    const uint32_t pos = 63u - (uint32_t)__clzll((long long)del);
    val = (val & ((1ull << pos) - 1ull)) | (((val >> pos) >> 1) << pos);
    del &= ~(1ull << pos);
    ++n;
  }
  return n;
}
__device__ __forceinline__ unsigned long long u64_of(uint2 v) { return (unsigned long long)v.x | ((unsigned long long)v.y << 32); }

// MagSgn: forward, LSB first, bytes past the segment read as 0xFF; the bit after every 0xFF byte is a
// stuffing bit (frwd_read / frwd_init<0xFF>, :340-421)
struct MsDec {
  const uint2* wnext; const uint8_t* seg_end; uint2* ring; uint32_t ridx;
  int left; Win128 w; uint32_t unstuff;
};
template <int STRIDE = DEC1_THREADS>
__device__ __forceinline__ void ms_ring_issue(MsDec& m) {
  uint2* slot = m.ring + m.ridx * STRIDE;
  if (reinterpret_cast<const uint8_t*>(m.wnext) < m.seg_end) cp_async<8>(slot, m.wnext); else *slot = make_uint2(0xFFFFFFFFu, 0xFFFFFFFFu);
  cp_commit();
  ++m.wnext; m.ridx = (m.ridx + 1) & (VLC_RING - 1);
}
// take a group of nv (1..8) bytes, first byte in the low byte of val
__device__ __forceinline__ void ms_ingest(MsDec& m, unsigned long long val, uint32_t nv) {
  if (m.left < (int)nv) val |= (m.left <= 0) ? ~0ull : (~0ull << (8 * m.left));
  if (nv < 8) val &= (1ull << (8 * nv)) - 1ull;
  m.left -= (int)nv;
  // bit 8i+7 <=> byte i == 0xFF: the low seven bits are all ones (adding 1 carries into bit 7) and bit 7 is set
  const unsigned long long ff = ((val & 0x7F7F7F7F7F7F7F7Full) + 0x0101010101010101ull) & val & 0x8080808080808080ull;
  // bits to delete: the top bit of the byte after each 0xFF (of byte 0 when the previous group ended in 0xFF)
  unsigned long long del = ((ff << 8) | ((unsigned long long)m.unstuff << 7)) & ((nv < 8) ? ((1ull << (8 * nv)) - 1ull) : ~0ull);
  m.unstuff = (uint32_t)(ff >> (8 * (nv - 1) + 7)) & 1u;
  const uint32_t c = 8 * nv - delete_bits(val, del);
  win_append(m.w, val, c);
}
template <int STRIDE = DEC1_THREADS>
__device__ __forceinline__ void ms_prime(MsDec& m, const uint8_t* p, int len, const uint8_t* seg_end, uint2* ring) {
  const uint2* wp = reinterpret_cast<const uint2*>((size_t)p & ~(size_t)7);
  const uint32_t a = (uint32_t)((size_t)p & 7);
  m.seg_end = seg_end; m.left = len; m.w.w0 = 0; m.w.w1 = 0; m.w.bits = 0; m.unstuff = 0;
  m.ring = ring; m.ridx = 0; m.wnext = wp + 1;
  #pragma unroll
  for (int i = 0; i < VLC_RING - 1; ++i) ms_ring_issue<STRIDE>(m);
  m.ridx = 0;
  ms_ingest(m, u64_of(wp[0]) >> (8 * a), 8 - a);           // the bytes up to the next 8-byte boundary: groups are aligned from here on
}
template <int STRIDE = DEC1_THREADS>
__device__ __forceinline__ void ms_fill(MsDec& m) {            // adds 56..64 bits; needs bits < 64
  cp_wait<VLC_RING - 2>();
  const uint32_t take = m.ridx;
  const unsigned long long val = u64_of(m.ring[take * STRIDE]);
  m.ridx = (take + VLC_RING - 1) & (VLC_RING - 1);
  ms_ring_issue<STRIDE>(m);
  m.ridx = (take + 1) & (VLC_RING - 1);
  ms_ingest(m, val, 8);
}

// VLC: backward from the end of the segment, LSB first, zeros once the segment is exhausted; a byte whose
// low seven bits are ones and whose predecessor in reading order is > 0x8F carries seven bits (rev_read,
// :220-302).  A group holds eight bytes in READING order (byte-reversed memory word).
struct VlcDec {
  const uint2* wnext; const uint2* wbase; uint2* ring; uint32_t ridx;
  int left; Win128 w; uint32_t unstuff;
};
__device__ __forceinline__ void vlc_ring_issue(VlcDec& v) {
  uint2* slot = v.ring + v.ridx * DEC1_THREADS;
  if (v.wnext >= v.wbase) cp_async<8>(slot, v.wnext); else *slot = make_uint2(0u, 0u);
  cp_commit();
  --v.wnext; v.ridx = (v.ridx + 1) & (VLC_RING - 1);
}
__device__ __forceinline__ unsigned long long bswap64(unsigned long long x) {
  return ((unsigned long long)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | (unsigned long long)__byte_perm((uint32_t)(x >> 32), 0, 0x0123);
}
__device__ __forceinline__ void vlc_ingest(VlcDec& v, unsigned long long val, uint32_t nv) {
  if (v.left < (int)nv) val &= (v.left <= 0) ? 0ull : ((1ull << (8 * v.left)) - 1ull);
  v.left -= (int)nv;
  const unsigned long long pv = (val << 8) | (v.unstuff ? 0x90ull : 0ull);        // predecessor of every byte
  const unsigned long long del = ((val & 0x7F7F7F7F7F7F7F7Full) + 0x0101010101010101ull) & pv &
                                 ((pv & 0x7070707070707070ull) + 0x7070707070707070ull) & 0x8080808080808080ull;
  v.unstuff = ((uint32_t)(val >> (8 * (nv - 1))) & 0xFFu) > 0x8Fu ? 1u : 0u;
  const uint32_t c = 8 * nv - delete_bits(val, del);
  win_append(v.w, val, c);
}
// p = the first byte to read (then downward), size = bytes available from p down; the window already
// holds the bits of the Scup nibble byte
__device__ __forceinline__ void vlc_prime(VlcDec& v, const uint8_t* p, int size, const uint8_t* buffer_start, uint2* ring) {
  const uint2* wp = reinterpret_cast<const uint2*>((size_t)p & ~(size_t)7);
  const uint32_t a = (uint32_t)((size_t)p & 7);
  v.wbase = reinterpret_cast<const uint2*>((size_t)buffer_start & ~(size_t)7);
  v.left = size;
  v.ring = ring; v.ridx = 0; v.wnext = wp - 1;
  #pragma unroll
  for (int i = 0; i < VLC_RING - 1; ++i) vlc_ring_issue(v);
  v.ridx = 0;
  vlc_ingest(v, bswap64(u64_of(wp[0])) >> (8 * (7 - a)), a + 1);   // down to the 8-byte boundary: groups are aligned from here on
}
__device__ __forceinline__ void vlc_fill(VlcDec& v) {         // adds 56..64 bits; needs bits < 64
  cp_wait<VLC_RING - 2>();
  const uint32_t take = v.ridx;
  const unsigned long long val = bswap64(u64_of(v.ring[take * DEC1_THREADS]));
  v.ridx = (take + VLC_RING - 1) & (VLC_RING - 1);
  vlc_ring_issue(v);
  v.ridx = (take + 1) & (VLC_RING - 1);
  vlc_ingest(v, val, 8);
}

template <int MODE>       // 0: integer output, 1: float output, 2: per-block mode / blocks with refinement passes, 3: DEC_OUT_CODED
__global__ void __launch_bounds__(DEC1_THREADS)
ht_decode_serial_kernel(const DecBlock* __restrict__ blocks, uint32_t nblocks,
                        const uint8_t* __restrict__ cs, uint32_t* __restrict__ coef,
                        uint32_t* __restrict__ scratch, const uint16_t* __restrict__ tables,
                        uint32_t out_mode, uint32_t* __restrict__ block_status, uint32_t prev_quads)
{
  __shared__ DecTables T;
  __shared__ uint2 s_ring[VLC_RING * DEC1_THREADS];        // per-thread FIFO of VLC 8-byte groups (slot-major)
  __shared__ uint2 s_mring[VLC_RING * DEC1_THREADS];       // per-thread FIFO of MagSgn 8-byte groups
  OJB_DYN_SMEM(uint16_t, s_prev);       // prev_quads x threads: msb(v_n) of the bottom samples of the row above
  {
    uint16_t* d = reinterpret_cast<uint16_t*>(&T);
    for (uint32_t i = threadIdx.x; i < sizeof(DecTables) / 2; i += blockDim.x) d[i] = tables[i];
  }
  __syncthreads();
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  const DecBlock blk = blocks[b];
  if (blk.flags & DEC_FLAG_FAST) return;                 // decoded by ht_decode_split_kernel
  uint32_t np = blk.num_passes;
  if (np == 0 || blk.len1 == 0) { block_status[b] = DST_EMPTY; return; }     // zero-filled by the fill kernel
  // validity gates (:752-820)
  if (np > 1 && blk.len2 == 0) np = 1;
  bool ok = true;
  if (np > 3 || blk.missing_msbs >= 30 || blk.len1 < 2) ok = false;
  if (blk.missing_msbs == 29 && np > 1) np = 1;      // p == 1: refinement passes are skipped
  const uint8_t* data = cs + blk.data_off;
  int lcup = (int)blk.len1, scup = 0;
  if (ok) {
    scup = ((int)data[lcup - 1] << 4) + (data[lcup - 2] & 0xF);
    if (scup < 2 || scup > lcup || scup > 4079) ok = false;
  }
  if (!ok || (blk.w + 1u) / 2 + 2 > prev_quads) { block_status[b] = DST_FAIL; return; }

  MelDec mel; mel.p = data + lcup - scup; mel.size = scup - 1; mel.tmp = 0; mel.bits = 0;
  mel.unstuff = false; mel.k = 0;
  VlcDec vlc;
  {
    const uint32_t d = data[lcup - 2];                     // the byte that shares the Scup nibble (rev_init, :270-302)
    vlc.w.w0 = d >> 4; vlc.w.w1 = 0;
    vlc.w.bits = 4 - (((vlc.w.w0 & 7) == 7) ? 1u : 0u);
    vlc.unstuff = (d | 0xF) > 0x8F ? 1u : 0u;
  }
  vlc_prime(vlc, data + lcup - 3, scup - 2, cs, s_ring + threadIdx.x);
  mel_prime(mel);
  MsDec ms;
  ms_prime(ms, data, lcup - scup, data + lcup, s_mring + threadIdx.x);
  int run = mel_next_run(mel);

  const uint32_t width = blk.w, height = blk.h, stride = blk.stride;
  const uint32_t nq = (width + 1) >> 1, qstride = (nq + 1) & ~1u;   // quads per row (even stride)
  uint32_t* rec = scratch + blk.scratch_off;
  uint32_t* dst = coef + blk.dst_off;
  uint16_t* prev = s_prev + threadIdx.x;
  const uint32_t mmsbp2 = blk.missing_msbs + 2u;
  const uint32_t p = 30u - blk.missing_msbs;
  const uint32_t shift = 31u - blk.K_max;
  const float delta = blk.delta;
  if (out_mode == DEC_OUT_PER_BLOCK) out_mode = (blk.flags & 2) ? (uint32_t)DEC_OUT_FLOAT : (uint32_t)DEC_OUT_INT;
  // MODE 0 / 1: the launch has cleanup passes only and one output type, known at compile time
  const uint32_t om = MODE == 0 ? (uint32_t)DEC_OUT_INT : MODE == 1 ? (uint32_t)DEC_OUT_FLOAT
                                : ((np > 1) ? (uint32_t)DEC_OUT_SIGNMAG : out_mode);
  // MODE 3: a cleanup-only block drops its bin centre (bit p - 1) at once; a block with refinement passes is decoded
  // whole, as the passes need the bin centre, and cut below its lowest plane p - 1 afterwards
  const uint32_t cut = (MODE == 3 && np == 1) ? 1u << (p - 1) : 0u;
  const bool vec4 = ((blk.dst_off | stride) & 3u) == 0;
  const bool narrow = mmsbp2 <= 16;          // m_n <= missing_msbs + 2: the four fields of a quad fit 64 bits
  const uint32_t pscale = 1u << (p - 1);
  bool fail = false;
  // significance of the row above as bit masks over up to 32 quads per word is not enough for wide
  // blocks: the row-above state (sigma of the two bottom samples, msb of their v_n) lives in s_prev
  for (uint32_t q = 0; q <= nq; ++q) prev[q * DEC1_THREADS] = 0;

  for (uint32_t y = 0; y < height && !fail; y += 2) {
    const uint16_t* vtab = y ? T.vlc1 : T.vlc0;
    uint32_t rho_left = 0;
    uint32_t* rrow = rec + (size_t)(y >> 1) * qstride;
    uint32_t pl = 0, pc = prev[0];             // row above: quad q-1, quad q (read before being overwritten)
    uint32_t* r0 = dst + (size_t)y * stride;
    uint32_t* r1 = r0 + stride;
    const bool has_r1 = y + 1 < height;
    for (uint32_t q = 0; q < nq; q += 2) {
      uint32_t t[2] = {0, 0}, pq[3];
      // one top-up per quad pair: the pair reads at most 2 x 7 + 6 + 10 bits
      while (vlc.w.bits < 64) vlc_fill(vlc);
      unsigned long long vt = vlc.w.w0;
      uint32_t vused = 0;
      pq[0] = pl; pq[1] = pc;
      pq[2] = prev[(q + 1) * DEC1_THREADS];
      const uint32_t pq3 = (q + 2 <= nq) ? prev[(q + 2) * DEC1_THREADS] : 0u;
      #pragma unroll
      for (uint32_t i = 0; i < 2; ++i) {
        const uint32_t qq = q + i;
        if (qq < nq) {
          uint32_t c;
          if (y == 0) c = (rho_left & 1) | (rho_left >> 1);
          else {
            // sigma bits of the row above: bit 10 = bottom-left, bit 11 = bottom-right of a quad
            const uint32_t pw = i ? pq[1] : pq[0], pn = i ? pq[2] : pq[1], pe = i ? pq3 : pq[2];
            const uint32_t a = ((pw >> 11) | (pn >> 10)) & 1u;
            const uint32_t l = ((rho_left >> 2) | (rho_left >> 3)) & 1u;
            const uint32_t r = ((pn >> 11) | (pe >> 10)) & 1u;
            c = a | (l << 1) | (r << 2);
          }
          uint32_t e = vtab[(c << 7) | ((uint32_t)vt & 0x7F)];
          if (c == 0) {               // significance of an all-zero context comes from MEL
            run -= 2;
            if (run != -1) e = 0;
            if (run < 0) run = mel_next_run(mel);
          }
          vt >>= (e & 7); vused += (e & 7);
          t[i] = e;
          rho_left = (e >> 4) & 15u;
        }
      }
      // U-VLC of the pair (:940-974 initial row, :1066-1085 others)
      uint32_t mode = ((t[0] >> 3) & 1u) | (((t[1] >> 3) & 1u) << 1);
      uint32_t ent;
      if (y == 0) {
        if (mode == 3) {
          run -= 2;
          if (run == -1) mode = 4;
          if (run < 0) run = mel_next_run(mel);
        }
        ent = T.uvlc0[(mode << 6) | ((uint32_t)vt & 0x3F)];
      } else
        ent = T.uvlc1[(mode << 6) | ((uint32_t)vt & 0x3F)];
      vt >>= (ent & 7); vused += (ent & 7);
      ent >>= 3;
      uint32_t len = ent & 0xF;
      uint32_t suf = (uint32_t)vt & ((1u << len) - 1u);
      vused += len;
      win_drop(vlc.w, vused);
      ent >>= 4;
      len = ent & 7; ent >>= 3;
      const uint32_t kap = (y == 0) ? 1u : 0u;
      const uint32_t uu[2] = { kap + (ent & 7) + (suf & ~(0xFFu << len)), kap + (ent >> 3) + (suf >> len) };
      if (np > 1)                       // the refinement passes look the CUP significance up
        *reinterpret_cast<uint2*>(rrow + q) = make_uint2((t[0] & 0xFFFF) | (uu[0] << 16), (t[1] & 0xFFFF) | (uu[1] << 16));

      // ---- MagSgn of the two quads (:1087-1316)
      uint32_t o[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
      #pragma unroll
      for (uint32_t i = 0; i < 2; ++i) {
        const uint32_t qq = q + i;
        if (qq >= nq) break;
        const uint32_t inf = t[i] & 0xFFFF;
        const uint32_t rho = (inf >> 4) & 15u, ek = inf >> 12, e1 = (inf >> 8) & 15u;
        uint32_t Uq = uu[i];
        if (y != 0) {
          // exponent predictor: msb of v_n of the four samples above (stored as 31 - clz(v | 2))
          const uint32_t pw = i ? pq[1] : pq[0], pn = i ? pq[2] : pq[1], pe = i ? pq3 : pq[2];
          const uint32_t emax = max(max((pw >> 5) & 31u, pn & 31u), max((pn >> 5) & 31u, pe & 31u));
          Uq += (rho & (rho - 1)) ? max(emax, 1u) : 1u;
        }
        if (Uq > mmsbp2) { fail = true; break; }
        uint32_t vbl = 0, vbr = 0;
        // m_n = sigma_n * (U_q - ek_n) for the four samples at once, one byte each
        uint32_t mk[4];
        {
          const uint32_t rb = (rho * 0x00204081u) & 0x01010101u, eb = (ek * 0x00204081u) & 0x01010101u;
          const uint32_t mb = (Uq * 0x01010101u - eb) & (rb * 0xFFu);
          mk[0] = mb & 0xFFu; mk[1] = (mb >> 8) & 0xFFu; mk[2] = (mb >> 16) & 0xFFu; mk[3] = mb >> 24;
        }
        // the window is topped up at the same two points of the quad in every lane; a quad whose four
        // fields fit 64 bits (K_max <= 15) needs the first one only
        #pragma unroll
        for (int half = 0; half < 2; ++half) {
          if (half == 0 || !narrow) { while (ms.w.bits < 64) ms_fill(ms); }
          uint32_t off = (half == 1 && narrow) ? mk[0] + mk[1] : 0u;
          #pragma unroll
          for (int kk = 0; kk < 2; ++kk) {
            const int k = 2 * half + kk;
            const uint32_t m = mk[k];
            const uint32_t bits = (uint32_t)(ms.w.w0 >> off);
            off += m;
            // (multiplications by powers of two on purpose: IMAD issues on the FMA pipe, not on the integer ALU
            // pipe that the shifts, logic and adds of this kernel load)
            const uint32_t pow = 1u << m;
            uint32_t v = (bits & (pow - 1u)) | 1u;
            v = ((e1 >> k) & 1u) * pow + v;                           // bit m is clear: + is |
            const bool sig = (rho >> k) & 1u;
            if (k == 1) vbl = sig ? v : 0u;
            if (k == 3) vbr = sig ? v : 0u;
            const uint32_t mag = v * pscale + 2u * pscale;            // (v + 2) << (p - 1): magnitude with the half-LSB bin centre, bit 30 down
            uint32_t val;
            if (MODE == 0) { const uint32_t a = mag >> shift; val = a * (1u - 2u * (bits & 1u)); }   // two's complement: +a or -a
            else if (MODE == 1) val = __float_as_uint(__fmul_rn((float)mag, delta)) | (bits << 31);
            else if (MODE == 3) val = (bits << 31) | (mag - cut);
            else val = to_output((bits << 31) | mag, om, shift, delta);
            o[i][k] = sig ? val : 0u;
          }
          if (!narrow) win_drop(ms.w, mk[2 * half] + mk[2 * half + 1]);
          else if (half == 1) win_drop(ms.w, off);
        }
        // row-above record of this quad for the next quad-row
        prev[qq * DEC1_THREADS] = (uint16_t)((31u - (uint32_t)__clz((int)(vbl | 2u))) | ((31u - (uint32_t)__clz((int)(vbr | 2u))) << 5)
                                             | (((rho >> 1) & 1u) << 10) | (((rho >> 3) & 1u) << 11));
      }
      pl = pq[2]; pc = pq3;
      if (fail) break;
      // ---- store the pair: samples 2q .. 2q+3 of the two rows
      if (vec4 && 2 * q + 3 < width) {
        *reinterpret_cast<uint4*>(r0 + 2 * q) = make_uint4(o[0][0], o[0][2], o[1][0], o[1][2]);
        if (has_r1) *reinterpret_cast<uint4*>(r1 + 2 * q) = make_uint4(o[0][1], o[0][3], o[1][1], o[1][3]);
      } else {
        #pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
          const uint32_t x = 2 * q + k;
          if (x < width) {
            r0[x] = o[k >> 1][(k & 1) * 2];
            if (has_r1) r1[x] = o[k >> 1][(k & 1) * 2 + 1];
          }
        }
      }
    }
  }
  if (fail) { block_status[b] = DST_FAIL; return; }

  if (np > 1) {
    refine_passes(blk, np, data, dst, rec, qstride, p);
    if (MODE == 3)
      for (uint32_t yy = 0; yy < height; ++yy)
        for (uint32_t xx = 0; xx < width; ++xx) dst[(size_t)yy * stride + xx] &= ~((1u << (p - 1)) - 1u);
    else if (out_mode != DEC_OUT_SIGNMAG)
      for (uint32_t yy = 0; yy < height; ++yy)
        for (uint32_t xx = 0; xx < width; ++xx) {
          uint32_t* qp = dst + (size_t)yy * stride + xx;
          *qp = to_output(*qp, out_mode, shift, delta);
        }
  }
  block_status[b] = 0;
}


// ---- fast path: two threads per code-block ----------------------------------------------------------------------
// The cleanup pass of the blocks the host marks DEC_FLAG_FAST: one coding pass, width a multiple of 4 and at most 64,
// even height, 16-byte aligned rows, missing_msbs + 2 <= 16 (so the four MagSgn fields of a quad fit 64 bits).
// Knowing that at compile time removes the per-quad bounds / pass / width tests of the general kernel, and the state
// of the row above shrinks to registers plus one word per quad pair:
//   * significance of the bottom samples of the row above: a 64-bit register, two bits per quad, walked four bits
//     per pair; the contexts of both quads of a pair come out of six consecutive bits;
//   * exponent predictor: per quad boundary q the OR g[q] = h(br of quad q-1) | h(bl of quad q) with h = v_n >> 1
//     (16 bits, v_n < 2^17); kappa of quad q is 32 - clz(g[q] | g[q+1] | 1): one word load, one word store and one
//     CLZ per quad instead of per-sample exponents, two 16-bit records and a 4-way max;
//   * VLC through a 64-bit window refilled 32 bits at a time (a pair reads at most 30 bits), MagSgn through the
//     128-bit window in 8-byte groups as in the general kernel.
// A U_q beyond missing_msbs + 2 (corrupt data) is clamped and flagged; the block is then zero-filled.
// The pass is two chains: MEL + VLC + U-VLC decoding (each codeword's position and context depend on the one
// before) and MagSgn extraction (positions depend on the row above through the exponent predictor).  The second
// needs the first's results but not the other way round, so the pair runs as a producer and a consumer thread in
// different warps of one CTA: warps 0-1 decode the quad records (rho, e_k, e_1, u) of 64 blocks one quad-row ahead
// into a double-buffered shared-memory row, warps 2-3 read them, extract the MagSgn fields and store the samples.
// Hand-over per quad-row through named barriers (producers bar.arrive on FULL, consumers bar.sync; the
// reverse on EMPTY), no polling.  Twice the threads per block: the serial chain of a block -- which bounds the
// kernel's duration when 49 152 blocks are all that is in flight -- is cut to the longer of the two halves.
#define SP_BLOCKS 64
template <int MODE>       // 0: integer output, 1: float output, 2: sign-magnitude, 3: DEC_OUT_CODED
__global__ void __launch_bounds__(2 * SP_BLOCKS)
ht_decode_split_kernel(const DecBlock* __restrict__ blocks, uint32_t nblocks,
                       const uint8_t* __restrict__ cs, uint32_t* __restrict__ coef,
                       const uint16_t* __restrict__ tables, uint32_t* __restrict__ block_status)
{
  __shared__ DecTables T;
  __shared__ uint32_t s_vring[VLC_RING * SP_BLOCKS];
  __shared__ uint2 s_mring[VLC_RING * SP_BLOCKS];
  __shared__ uint32_t s_g[17 * SP_BLOCKS];
  // [stage][pair][block]: the quad records of one quad-row, 16 bits per quad: bits 4-15 of the CxtVLC entry (rho, e_1,
  // e_k) and u_q - kappa in bits 0-3 (a larger u_q sets the block's bit in s_ufail)
  __shared__ uint32_t s_rec[2 * 16 * SP_BLOCKS];
  __shared__ uint4 s_stage[8 * SP_BLOCKS];                  // [row * 4 + pair][block ^ (row * 4 + pair)]: see the consumer
  __shared__ uint32_t s_rows, s_ufail[SP_BLOCKS / 32];
  {
    uint16_t* d = reinterpret_cast<uint16_t*>(&T);
    for (uint32_t i = threadIdx.x; i < sizeof(DecTables) / 2; i += blockDim.x) d[i] = tables[i];
  }
  if (threadIdx.x < SP_BLOCKS / 32) s_ufail[threadIdx.x] = 0;
  if (threadIdx.x == 0) s_rows = 0;
  __syncthreads();
  const bool producer = threadIdx.x < SP_BLOCKS;
  const uint32_t tid = producer ? threadIdx.x : threadIdx.x - SP_BLOCKS;
  const uint32_t b = blockIdx.x * SP_BLOCKS + tid;
  DecBlock blk;
  bool active = b < nblocks;
  if (active) { blk = blocks[b]; active = (blk.flags & DEC_FLAG_FAST) != 0; }
  const uint8_t* data = nullptr;
  int lcup = 0, scup = 0;
  if (active) {
    data = cs + blk.data_off;
    lcup = (int)blk.len1;
    scup = ((int)data[lcup - 1] << 4) + (data[lcup - 2] & 0xF);
    if (scup < 2 || scup > lcup || scup > 4079) { if (!producer) block_status[b] = DST_FAIL; active = false; }
  }
  const uint32_t npairs = active ? (uint32_t)(blk.w >> 2) : 0u, myrows = active ? (uint32_t)(blk.h >> 1) : 0u;
  if (producer && myrows) atomicMax(&s_rows, myrows);
  __syncthreads();
  const uint32_t rows = s_rows;
  enum { BAR_FULL = 1, BAR_EMPTY = 3 };

  if (producer) {
    MelDec mel; RevDec vlc; int run = 0;
    if (active) {
      mel.p = data + lcup - scup; mel.size = scup - 1; mel.tmp = 0; mel.bits = 0; mel.unstuff = false; mel.k = 0;
      vlc.p = data + lcup - 2; vlc.size = scup - 2;
      const uint32_t d = *vlc.p--;                            // the byte that shares the Scup nibble (rev_init, :270-302)
      vlc.tmp = d >> 4;
      vlc.bits = 4 - (((vlc.tmp & 7) == 7) ? 1u : 0u);
      vlc.unstuff = (d | 0xF) > 0x8F;
      rev_prime<SP_BLOCKS>(vlc, cs, s_vring + tid);
      mel_prime(mel);
      run = mel_next_run(mel);
    }
    uint32_t sg_lo = 0, sg_hi = 0;              // bottom-sample significance of the row above: bit 2q = left, 2q+1 = right
    for (uint32_t r = 0; r < rows; ++r) {
      if (r >= 2) named_bar_sync(BAR_EMPTY + (r & 1), 2 * SP_BLOCKS);
      if (r < myrows) {
        const bool first = (r == 0);
        const uint16_t* vtab = first ? T.vlc0 : T.vlc1;
        const uint16_t* utab = first ? T.uvlc0 : T.uvlc1;
        uint32_t* out = s_rec + (size_t)(r & 1) * 16 * SP_BLOCKS + tid;
        uint32_t rho_left = 0, ubig = 0;
        uint32_t rs_lo = sg_lo, rs_hi = sg_hi, rs_carry = 0;
        uint32_t cu_lo = 0, cu_hi = 0;
        #pragma unroll 1
        for (uint32_t j = 0; j < npairs; ++j) {
          while (vlc.bits <= 32) rev_fill32<SP_BLOCKS>(vlc);          // the pair reads at most 2 x 7 + 6 + 10 bits
          uint32_t vt = (uint32_t)vlc.tmp, vused = 0;
          const uint32_t y6 = rs_carry | ((rs_lo & 0x1Fu) << 1);
          const uint32_t z = y6 | (y6 >> 1);
          rs_carry = (rs_lo >> 3) & 1u;
          rs_lo = __funnelshift_r(rs_lo, rs_hi, 4); rs_hi >>= 4;
          uint32_t t[2];
          #pragma unroll
          for (uint32_t i = 0; i < 2; ++i) {
            uint32_t c;
            if (first) c = (rho_left & 1u) | (rho_left >> 1);
            else c = ((z >> (2 * i)) & 5u) | (rho_left > 3u ? 2u : 0u);
            uint32_t e = vtab[(c << 7) | (vt & 0x7Fu)];
            if (c == 0) {               // significance of an all-zero context comes from MEL
              run -= 2;
              if (run != -1) e = 0;
              if (run < 0) run = mel_next_run(mel);
            }
            vt >>= (e & 7u); vused += (e & 7u);
            t[i] = e;
            rho_left = (e >> 4) & 15u;
          }
          uint32_t mode = ((t[0] >> 3) & 1u) | ((t[1] >> 2) & 2u);
          if (first && mode == 3) {
            run -= 2;
            if (run == -1) mode = 4;
            if (run < 0) run = mel_next_run(mel);
          }
          uint32_t ent = utab[(mode << 6) | (vt & 0x3Fu)];
          vt >>= (ent & 7u); vused += (ent & 7u);
          ent >>= 3;
          uint32_t len = ent & 0xFu;
          const uint32_t suf = vt & ((1u << len) - 1u);
          vused += len;
          vlc.tmp >>= vused; vlc.bits -= vused;
          ent >>= 4;
          len = ent & 7u; ent >>= 3;
          const uint32_t u0 = (ent & 7u) + (suf & ~(0xFFu << len)), u1 = (ent >> 3) + (suf >> len);   // u_q without kappa
          {
            const uint32_t ta = (t[0] >> 5) & 5u, tb = (t[1] >> 5) & 5u;
            const uint32_t nb = ((ta | (ta >> 1)) & 3u) | (((tb | (tb >> 1)) & 3u) << 2);
            cu_lo = __funnelshift_r(cu_lo, cu_hi, 4); cu_hi = (cu_hi >> 4) | (nb << 28);
          }
          ubig |= u0 | u1;
          out[j * SP_BLOCKS] = (t[0] & 0xFFF0u) | (u0 & 15u) | (((t[1] & 0xFFF0u) | (u1 & 15u)) << 16);
        }
        // kappa >= 1, so u_q > 15 means U_q > 16 >= missing_msbs + 2: the block fails (the 4-bit field cannot carry it)
        if (ubig > 15u) atomicOr(&s_ufail[tid >> 5], 1u << (tid & 31));
        const uint32_t sh = 64u - 4u * npairs;
        const uint32_t a0 = sh >= 32 ? cu_hi : cu_lo, a1 = sh >= 32 ? 0u : cu_hi;
        sg_lo = __funnelshift_r(a0, a1, sh & 31u); sg_hi = a1 >> (sh & 31u);
      }
      __threadfence_block();
      named_bar_arrive(BAR_FULL + (r & 1), 2 * SP_BLOCKS);
    }
    return;
  }

  // ---- consumer: MagSgn extraction and output
  MsDec ms;
  uint32_t* dst = nullptr; uint32_t* gw = s_g + tid;
  uint32_t mmsbp2 = 0, pscale = 0, mul_a = 0, stride = 0, fail = 0;
  float delta = 0.f;
  if (active) {
    ms_prime<SP_BLOCKS>(ms, data, lcup - scup, data + lcup, s_mring + tid);
    dst = coef + blk.dst_off; stride = blk.stride;
    mmsbp2 = blk.missing_msbs + 2u;
    pscale = 1u << (29u - blk.missing_msbs);
    mul_a = 1u << (blk.K_max - blk.missing_msbs - 1u);
    delta = blk.delta;
    for (uint32_t j = 0; j <= 16; ++j) gw[j * SP_BLOCKS] = 0;
  }
  // The samples of a quad pair (16 bytes in each of two rows) go to a staging tile instead of global memory: chunk
  // (row, pair) of block t sits at s_stage[c * SP_BLOCKS + (t ^ c)], c = row * 4 + pair mod 4.  Every four pairs the
  // warp writes its 32 blocks' tiles out cooperatively, eight lanes per block (two 64-byte row pieces = four whole
  // sectors), so a store instruction touches 8 lines instead of 32 half-sectors in 32 lines.  The XOR keeps both the
  // owner's stores (a quarter-warp = 8 consecutive blocks, one chunk) and the write-out's loads (one block, 8 chunks)
  // on 8 different 16-byte bank groups.  Chunks of pairs a block does not have are never written out.
  const uint32_t lane = tid & 31u, wbase = tid & ~31u;
  for (uint32_t r = 0; r < rows; ++r) {
    named_bar_sync(BAR_FULL + (r & 1), 2 * SP_BLOCKS);
    const bool first = (r == 0);
    const uint32_t lp = (r < myrows && !fail) ? npairs : 0u;          // pairs this lane decodes in quad-row r
    const uint32_t wp = __reduce_max_sync(0xFFFFFFFFu, lp);
    // for the write-out: address of row 2r (16-byte aligned) | pairs - 1, or 0 when the lane writes nothing
    const unsigned long long rowa = lp ? reinterpret_cast<unsigned long long>(dst + (size_t)(2 * r) * stride) | (lp - 1u) : 0ull;
    const uint32_t* in = s_rec + (size_t)(r & 1) * 16 * SP_BLOCKS + tid;
    uint32_t wj = gw[0], h_carry = 0;
    #pragma unroll 1
    for (uint32_t j = 0; j < wp; ++j) {
      if (j < lp) {
        const uint32_t rec = in[j * SP_BLOCKS];
        const uint32_t wj1 = gw[(j + 1) * SP_BLOCKS];
        const uint32_t gor[2] = { (wj | (wj >> 16)) & 0xFFFFu, (wj >> 16) | (wj1 & 0xFFFFu) };
        wj = wj1;
        uint32_t o[2][4], hb[2][2];
        #pragma unroll
        for (uint32_t i = 0; i < 2; ++i) {
          const uint32_t inf = (rec >> (16 * i)) & 0xFFFFu;
          const uint32_t rho = (inf >> 4) & 15u, ek = inf >> 12, e1 = (inf >> 8) & 15u;
          uint32_t Uq = inf & 15u;
          Uq += (!first && (rho & (rho - 1u))) ? 32u - (uint32_t)__clz((int)(gor[i] | 1u)) : 1u;
          fail |= (Uq > mmsbp2) ? 1u : 0u;
          Uq = min(Uq, mmsbp2);
          const uint32_t rb = (rho * 0x00204081u) & 0x01010101u, eb = (ek * 0x00204081u) & 0x01010101u;
          const uint32_t mb = (Uq * 0x01010101u - eb) & (rb * 0xFFu);
          const uint32_t m0 = mb & 0xFFu, m1 = (mb >> 8) & 0xFFu, m2 = (mb >> 16) & 0xFFu, m3 = mb >> 24;
          while (ms.w.bits < 64) ms_fill<SP_BLOCKS>(ms);              // the quad reads at most 64 bits
          const uint32_t lo = (uint32_t)ms.w.w0, hi = (uint32_t)(ms.w.w0 >> 32);
          const uint32_t s01 = m0 + m1;                           // <= 32
          const uint32_t lo2 = __funnelshift_rc(lo, hi, s01), hi2 = __funnelshift_rc(hi, 0u, s01);
          const uint32_t f[4] = { lo, __funnelshift_r(lo, hi, m0), lo2, __funnelshift_r(lo2, hi2, m2) };
          const uint32_t mm[4] = { m0, m1, m2, m3 };
          win_drop(ms.w, s01 + m2 + m3);
          #pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint32_t m = mm[k], bits = f[k];
            const uint32_t pw = 1u << m;
            uint32_t v = (bits & (pw - 1u)) | 1u;
            v = ((e1 >> k) & 1u) * pw + v;                          // bit m is clear: + is |
            const bool sig = (rho >> k) & 1u;
            if (k & 1) hb[i][k >> 1] = sig ? (v >> 1) : 0u;
            uint32_t val;
            if (MODE == 0) { const uint32_t a = (v * mul_a + 2u * mul_a) >> 1; val = a * (1u - 2u * (bits & 1u)); }
            else {
              const uint32_t mag = v * pscale + 2u * pscale;
              if (MODE == 1) val = __float_as_uint(__fmul_rn((float)mag, delta)) | (bits << 31);
              else if (MODE == 3) val = (bits << 31) | (mag - pscale);     // without the bin centre
              else val = (bits << 31) | mag;
            }
            o[i][k] = sig ? val : 0u;
          }
        }
        gw[j * SP_BLOCKS] = (h_carry | hb[0][0]) | ((hb[0][1] | hb[1][0]) << 16);
        h_carry = hb[1][1];
        const uint32_t c = j & 3u;
        s_stage[c * SP_BLOCKS + (tid ^ c)] = make_uint4(o[0][0], o[0][2], o[1][0], o[1][2]);
        s_stage[(c + 4u) * SP_BLOCKS + (tid ^ (c + 4u))] = make_uint4(o[0][1], o[0][3], o[1][1], o[1][3]);
      }
      if ((j & 3u) == 3u || j + 1 == wp) {        // write out pairs j & ~3 .. j of the warp's blocks
        __syncwarp();
        const uint32_t c = lane & 7u, pr = (j & ~3u) + (c & 3u);          // this lane's chunk: row c >> 2, pair pr
        #pragma unroll 1
        for (uint32_t i = 0; i < 32; i += 4) {
          const uint32_t bb = i + (lane >> 3);
          const unsigned long long a = __shfl_sync(0xFFFFFFFFu, rowa, (int)bb);
          const uint32_t sb = __shfl_sync(0xFFFFFFFFu, stride, (int)bb);
          if (a && pr <= (uint32_t)(a & 15u))
            *reinterpret_cast<uint4*>(reinterpret_cast<uint32_t*>(a & ~15ull) + (c >> 2) * sb + 4 * pr) =
                s_stage[c * SP_BLOCKS + ((wbase + bb) ^ c)];
        }
        __syncwarp();
      }
    }
    if (lp) gw[npairs * SP_BLOCKS] = h_carry;
    if (r + 2 < rows) named_bar_arrive(BAR_EMPTY + (r & 1), 2 * SP_BLOCKS);
  }
  if (active) block_status[b] = (fail || ((s_ufail[tid >> 5] >> (tid & 31)) & 1u)) ? DST_FAIL : 0u;
}


// ---- 64-bit samples (precision beyond 32 bits) ------------------------------------------------------------------
// ojph_decode_codeblock64 (src/core/coding/ojph_block_decoder64.cpp:766-1316), cleanup pass, one thread per block,
// written for clarity rather than speed (the path serves 28..32-bit lossless content): p = 62 - missing_msbs, MagSgn
// fields of up to 43 bits read one sample at a time, exponents kept in 6 bits, and the 4-bit U-VLC extension for
// u_q > 32 (:1000-1010 initial row, with the bias of the table entry; :1122-1131 others).  Output: 64-bit two's
// complement integers (gen_rev_tx_from_cb64, ojph_codestream_gen.cpp:140-155) or the raw sign-magnitude words.
template <bool SIGNMAG>
__global__ void __launch_bounds__(DEC1_THREADS)
ht_decode_wide_kernel(const DecBlock* __restrict__ blocks, uint32_t nblocks,
                      const uint8_t* __restrict__ cs, unsigned long long* __restrict__ coef,
                      const uint16_t* __restrict__ tables, uint32_t* __restrict__ block_status, uint32_t prev_quads)
{
  __shared__ DecTables T;
  __shared__ uint2 s_ring[VLC_RING * DEC1_THREADS];
  __shared__ uint2 s_mring[VLC_RING * DEC1_THREADS];
  OJB_DYN_SMEM(uint16_t, s_prev);       // prev_quads x threads: exp(bl) | exp(br) << 6 | sigma(bl) << 12 | sigma(br) << 13
  {
    uint16_t* d = reinterpret_cast<uint16_t*>(&T);
    for (uint32_t i = threadIdx.x; i < sizeof(DecTables) / 2; i += blockDim.x) d[i] = tables[i];
  }
  __syncthreads();
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nblocks) return;
  const DecBlock blk = blocks[b];
  const uint32_t np = blk.num_passes;
  if (np == 0 || blk.len1 == 0) { block_status[b] = DST_EMPTY; return; }
  bool ok = np == 1 && blk.missing_msbs <= 60 && blk.len1 >= 2;       // (refinement passes are refused by the host)
  const uint8_t* data = cs + blk.data_off;
  const int lcup = (int)blk.len1;
  int scup = 0;
  if (ok) {
    scup = ((int)data[lcup - 1] << 4) + (data[lcup - 2] & 0xF);
    if (scup < 2 || scup > lcup || scup > 4079) ok = false;
  }
  if (!ok || (blk.w + 1u) / 2 + 2 > prev_quads) { block_status[b] = DST_FAIL; return; }

  MelDec mel; mel.p = data + lcup - scup; mel.size = scup - 1; mel.tmp = 0; mel.bits = 0; mel.unstuff = false; mel.k = 0;
  VlcDec vlc;
  {
    const uint32_t d = data[lcup - 2];
    vlc.w.w0 = d >> 4; vlc.w.w1 = 0;
    vlc.w.bits = 4 - (((vlc.w.w0 & 7) == 7) ? 1u : 0u);
    vlc.unstuff = (d | 0xF) > 0x8F ? 1u : 0u;
  }
  vlc_prime(vlc, data + lcup - 3, scup - 2, cs, s_ring + threadIdx.x);
  mel_prime(mel);
  MsDec ms;
  ms_prime(ms, data, lcup - scup, data + lcup, s_mring + threadIdx.x);
  int run = mel_next_run(mel);

  const uint32_t width = blk.w, height = blk.h, stride = blk.stride;
  const uint32_t nq = (width + 1) >> 1;
  unsigned long long* dst = coef + blk.dst_off;
  uint16_t* prev = s_prev + threadIdx.x;
  const uint32_t mmsbp2 = blk.missing_msbs + 2u;
  const uint32_t p = 62u - blk.missing_msbs;
  const uint32_t shift = 63u - blk.K_max;
  bool fail = false;
  for (uint32_t q = 0; q <= nq + 1 && q < prev_quads; ++q) prev[q * DEC1_THREADS] = 0;

  for (uint32_t y = 0; y < height && !fail; y += 2) {
    const bool first = y == 0;
    const uint16_t* vtab = first ? T.vlc0 : T.vlc1;
    uint32_t rho_left = 0;
    uint32_t pl = 0, pc = prev[0];
    unsigned long long* r0 = dst + (size_t)y * stride;
    unsigned long long* r1 = r0 + stride;
    const bool has_r1 = y + 1 < height;
    for (uint32_t q = 0; q < nq && !fail; q += 2) {
      uint32_t t[2] = {0, 0}, pq[3];
      while (vlc.w.bits < 64) vlc_fill(vlc);                  // the pair reads at most 2 x 7 + 6 + 10 + 8 bits
      unsigned long long vt = vlc.w.w0;
      uint32_t vused = 0;
      pq[0] = pl; pq[1] = pc;
      pq[2] = prev[(q + 1) * DEC1_THREADS];
      const uint32_t pq3 = (q + 2 <= nq) ? prev[(q + 2) * DEC1_THREADS] : 0u;
      for (uint32_t i = 0; i < 2; ++i) {
        if (q + i >= nq) break;
        uint32_t c;
        if (first) c = (rho_left & 1) | (rho_left >> 1);
        else {
          const uint32_t pw = i ? pq[1] : pq[0], pn = i ? pq[2] : pq[1], pe = i ? pq3 : pq[2];
          const uint32_t a = ((pw >> 13) | (pn >> 12)) & 1u;
          const uint32_t l = ((rho_left >> 2) | (rho_left >> 3)) & 1u;
          const uint32_t r = ((pn >> 13) | (pe >> 12)) & 1u;
          c = a | (l << 1) | (r << 2);
        }
        uint32_t e = vtab[(c << 7) | ((uint32_t)vt & 0x7F)];
        if (c == 0) {
          run -= 2;
          if (run != -1) e = 0;
          if (run < 0) run = mel_next_run(mel);
        }
        vt >>= (e & 7); vused += (e & 7);
        t[i] = e;
        rho_left = (e >> 4) & 15u;
      }
      uint32_t mode = ((t[0] >> 3) & 1u) | (((t[1] >> 3) & 1u) << 1);
      uint32_t ent;
      if (first) {
        if (mode == 3) {
          run -= 2;
          if (run == -1) mode = 4;
          if (run < 0) run = mel_next_run(mel);
        }
        ent = T.uvlc0[(mode << 6) | ((uint32_t)vt & 0x3F)];
      } else
        ent = T.uvlc1[(mode << 6) | ((uint32_t)vt & 0x3F)];
      vt >>= (ent & 7); vused += (ent & 7);
      ent >>= 3;
      uint32_t len = ent & 0xF;
      const uint32_t suf = (uint32_t)vt & ((1u << len) - 1u);
      vt >>= len; vused += len;
      ent >>= 4;
      len = ent & 7; ent >>= 3;
      uint32_t uq[2] = { (ent & 7) + (suf & ~(0xFFu << len)), (ent >> 3) + (suf >> len) };
      // extensions: u_q > 32 once the initial row's "+2" of the both-large mode is taken off
      const uint32_t bias = (first && mode == 4) ? 2u : 0u;
      for (uint32_t i = 0; i < 2; ++i)
        if (uq[i] - bias > 32u && uq[i] >= bias) {
          uq[i] += ((uint32_t)vt & 0xFu) << 2;
          vt >>= 4; vused += 4;
        }
      win_drop(vlc.w, vused);
      const uint32_t kap = first ? 1u : 0u;

      for (uint32_t i = 0; i < 2 && !fail; ++i) {
        const uint32_t qq = q + i;
        if (qq >= nq) break;
        const uint32_t inf = t[i] & 0xFFFF;
        const uint32_t rho = (inf >> 4) & 15u, ek = inf >> 12, e1 = (inf >> 8) & 15u;
        uint32_t Uq = uq[i] + kap;
        if (!first) {
          const uint32_t pw = i ? pq[1] : pq[0], pn = i ? pq[2] : pq[1], pe = i ? pq3 : pq[2];
          const uint32_t emax = max(max((pw >> 6) & 63u, pn & 63u), max((pn >> 6) & 63u, pe & 63u));
          Uq += (rho & (rho - 1)) ? max(emax, 1u) : 1u;
        }
        if (Uq > mmsbp2) { fail = true; break; }
        unsigned long long val[4] = {0, 0, 0, 0};
        uint32_t ex[4] = {0, 0, 0, 0};
        for (int k = 0; k < 4; ++k) {
          if (!((rho >> k) & 1u)) continue;
          const uint32_t m = Uq - ((ek >> k) & 1u);                   // <= 43
          while (ms.w.bits < 64) ms_fill(ms);
          const unsigned long long bits = ms.w.w0;
          win_drop(ms.w, m);
          unsigned long long v = (bits & ((1ull << m) - 1ull)) | ((unsigned long long)((e1 >> k) & 1u) << m) | 1ull;
          ex[k] = 63u - (uint32_t)__clzll((long long)(v | 2ull));
          const unsigned long long mag = (v + 2ull) << (p - 1);       // magnitude with the half-LSB bin centre, bit 62 down
          if (SIGNMAG) val[k] = ((bits & 1ull) << 63) | mag;
          else { const long long a = (long long)(mag >> shift); val[k] = (unsigned long long)((bits & 1ull) ? -a : a); }
        }
        prev[qq * DEC1_THREADS] = (uint16_t)(ex[1] | (ex[3] << 6) | (((rho >> 1) & 1u) << 12) | (((rho >> 3) & 1u) << 13));
        const uint32_t x = 2 * qq;
        r0[x] = val[0]; if (has_r1) r1[x] = val[1];
        if (x + 1 < width) { r0[x + 1] = val[2]; if (has_r1) r1[x + 1] = val[3]; }
      }
      pl = pq[2]; pc = pq3;
    }
  }
  block_status[b] = fail ? DST_FAIL : 0u;
}

// zero-fill of 64-bit blocks that are not included or failed to decode
__global__ void __launch_bounds__(DEC_WARPS * 32)
ht_dec_fill_wide_kernel(const DecBlock* __restrict__ blocks, uint32_t nblocks, unsigned long long* __restrict__ coef,
                        uint32_t* __restrict__ block_status)
{
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t b = blockIdx.x * DEC_WARPS + warp;
  if (b >= nblocks) return;
  const uint32_t st = block_status[b];
  if (st == 0) return;
  const DecBlock blk = blocks[b];
  unsigned long long* dst = coef + blk.dst_off;
  for (uint32_t yy = 0; yy < blk.h; ++yy)
    for (uint32_t xx = lane; xx < blk.w; xx += 32) dst[(size_t)yy * blk.stride + xx] = 0;
  __syncwarp();
  if (lane == 0) block_status[b] = (st & DST_FAIL) ? DST_FAIL : 0u;
}

// zero-fill of blocks that are not included or failed to decode (one warp per block)
__global__ void __launch_bounds__(DEC_WARPS * 32)
ht_dec_fill_kernel(const DecBlock* __restrict__ blocks, uint32_t nblocks, uint32_t* __restrict__ coef,
                   uint32_t* __restrict__ block_status)
{
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t b = blockIdx.x * DEC_WARPS + warp;
  if (b >= nblocks) return;
  const uint32_t st = block_status[b];
  if (st == 0) return;
  const DecBlock blk = blocks[b];
  uint32_t* dst = coef + blk.dst_off;
  for (uint32_t yy = 0; yy < blk.h; ++yy)
    for (uint32_t xx = lane; xx < blk.w; xx += 32) dst[(size_t)yy * blk.stride + xx] = 0;
  __syncwarp();                          // every lane has read the status before it is rewritten
  if (lane == 0) block_status[b] = (st & DST_FAIL) ? DST_FAIL : 0u;
}

} // namespace

void launch_ht_decode_wide(const DecBlock* blocks, uint32_t nblocks, uint32_t max_width, const uint8_t* codestream,
                           uint32_t* coef, const uint16_t* tables, bool signmag, uint32_t* block_status, cudaStream_t st)
{
  if (nblocks == 0) return;
  const uint32_t prev_quads = (max_width + 1) / 2 + 2;
  const size_t smem = (size_t)prev_quads * DEC1_THREADS * sizeof(uint16_t);
  auto k = signmag ? ht_decode_wide_kernel<true> : ht_decode_wide_kernel<false>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((nblocks + DEC1_THREADS - 1) / DEC1_THREADS), block(DEC1_THREADS);
  OJB_LAUNCH(k, grid, block, smem, st, blocks, nblocks, codestream, reinterpret_cast<unsigned long long*>(coef), tables, block_status,
             prev_quads);
  dim3 g2((nblocks + DEC_WARPS - 1) / DEC_WARPS), b2(DEC_WARPS * 32);
  OJB_LAUNCH(ht_dec_fill_wide_kernel, g2, b2, 0, st, blocks, nblocks, reinterpret_cast<unsigned long long*>(coef), block_status);
}

void launch_ht_decode_serial(const DecBlock* blocks, uint32_t nblocks, uint32_t nfast, uint32_t max_width, const uint8_t* codestream,
                             uint32_t* coef, uint32_t* scratch, const uint16_t* tables, uint32_t out_mode,
                             bool cleanup_only, uint32_t* block_status, cudaStream_t st, const SideStream* side)
{
  if (nblocks == 0) return;
  const bool forked = side && side->st && nfast && nfast < nblocks;      // both kernels to run: the general one on the side stream
  cudaStream_t sg = forked ? side->st : st;
  if (forked) { cudaEventRecord(side->fork, st); cudaStreamWaitEvent(side->st, side->fork, 0); }
  const uint32_t prev_quads = (max_width + 1) / 2 + 2;
  const size_t smem = (size_t)prev_quads * DEC1_THREADS * sizeof(uint16_t);
  // specialised on the output type when no block carries SigProp / MagRef passes
  auto k = (cleanup_only && out_mode == DEC_OUT_INT) ? ht_decode_serial_kernel<0>
         : (cleanup_only && out_mode == DEC_OUT_FLOAT) ? ht_decode_serial_kernel<1>
         : out_mode == DEC_OUT_CODED ? ht_decode_serial_kernel<3> : ht_decode_serial_kernel<2>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  dim3 grid((nblocks + DEC1_THREADS - 1) / DEC1_THREADS), block(DEC1_THREADS);
  if (nfast) {           // blocks flagged DEC_FLAG_FAST (cleanup pass only, one output type): the producer / consumer pair
    auto kf = out_mode == DEC_OUT_INT ? ht_decode_split_kernel<0> : out_mode == DEC_OUT_FLOAT ? ht_decode_split_kernel<1>
            : out_mode == DEC_OUT_CODED ? ht_decode_split_kernel<3> : ht_decode_split_kernel<2>;
    dim3 g2((nblocks + SP_BLOCKS - 1) / SP_BLOCKS), b2(2 * SP_BLOCKS);
    OJB_LAUNCH(kf, g2, b2, 0, st, blocks, nblocks, codestream, coef, tables, block_status);
  }
  if (nfast < nblocks) {
    OJB_LAUNCH(k, grid, block, smem, sg, blocks, nblocks, codestream, coef, scratch, tables, out_mode,
               block_status, prev_quads);
  }
  if (forked) { cudaEventRecord(side->join, side->st); cudaStreamWaitEvent(st, side->join, 0); }
  {
    dim3 grid((nblocks + DEC_WARPS - 1) / DEC_WARPS), block(DEC_WARPS * 32);
    OJB_LAUNCH(ht_dec_fill_kernel, grid, block, 0, st, blocks, nblocks, coef, block_status);
  }
}

} // namespace ojb
