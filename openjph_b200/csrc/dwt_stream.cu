// dwt_stream.cu -- register-streaming lifting kernels (the fast path for every resolution that is
// at least 2x2; dwt_fwd.cu / dwt_inv.cu remain the general shared-memory path for degenerate sizes).
//
// Same arithmetic, same order as the reference (forward: vertical lifting then horizontal on each
// produced line, src/core/codestream/ojph_resolution.cpp:572-600 / :649-682; inverse: horizontal
// synthesis then vertical, :738-781 / :841-898; step formulas src/core/transform/ojph_transform.cpp:
// 209-257, 336-411, 514-590, 691-849), but organised for the GPU instead of line buffers:
//   * one WARP owns a strip of 128 columns (120 produced + a halo lane each side) and streams down a
//     chunk of rows; lane l holds four consecutive columns (even, odd, even, odd) = (low, high, low, high);
//   * VERTICAL lifting is a software pipeline in registers (state: 2 values per column for 5/3,
//     4 for 9/7); every iteration consumes two input rows and emits one (low, high) output pair;
//   * HORIZONTAL lifting of an emitted row is done with __shfl_up / __shfl_down between neighbouring
//     lanes -- no shared memory, no block barrier anywhere in the kernel;
//   * loads and stores are 8/16-byte vectors wherever the four columns are contiguous and aligned,
//     and the next iteration's rows are requested before the current pair is finished;
//   * one lane per side is halo (recomputed by the neighbouring strip), a few rows per chunk are
//     pipeline priming; borders use mirrored coordinates (whole-sample symmetric
//     extension, ojph_transform.cpp:372-374).
// Level 1 fuses sample fetch, level shift / int->float and RCT / ICT on load (forward) and the
// inverse of those on store (inverse); quantisation to MSB-aligned sign-magnitude is fused into
// the sub-band store (forward).
#include <cstdlib>
#include "dwt_common.cuh"
#include "ojb_async.cuh"
#include "ojb_kernels.h"

namespace ojb {

#define DS_WARPS 4
#define DS_ROWS 64            // output rows per warp chunk (large resolutions; small ones use fewer)
#define DS_COLS 4             // columns per lane: (even, odd, even, odd) = (low, high, low, high)
#define DS_STAGES 4           // row-pair stages of a lane's cp.async FIFO (3 in flight)
#define DS_VALID 30           // lanes that produce output; lanes 0 and 31 are halo (4 columns reach)
#define FULL 0xFFFFFFFFu

namespace {

template <bool REV> struct Tp;
template <> struct Tp<true>  { typedef int T; };
template <> struct Tp<false> { typedef float T; };

__device__ __forceinline__ float lift(float d, float a, float b, float c) {     // d + c*(a+b), no FMA
  return __fadd_rn(d, __fmul_rn(c, __fadd_rn(a, b)));
}

// horizontal analysis of one line; a lane holds columns (a[0], a[1], a[2], a[3]) = (even, odd, even, odd)
template <bool REV, typename T>
__device__ __forceinline__ void horz_ana(T (&a)[4]) {
  if (REV) {
    const int r = __shfl_down_sync(FULL, (int)a[0], 1);
    a[1] = (T)((int)a[1] - (((int)a[0] + (int)a[2]) >> 1));
    a[3] = (T)((int)a[3] - (((int)a[2] + r) >> 1));
    const int l = __shfl_up_sync(FULL, (int)a[3], 1);
    a[0] = (T)((int)a[0] + ((l + (int)a[1] + 2) >> 2));
    a[2] = (T)((int)a[2] + (((int)a[1] + (int)a[3] + 2) >> 2));
  } else {
    float r = __shfl_down_sync(FULL, (float)a[0], 1);
    a[1] = (T)lift((float)a[1], (float)a[0], (float)a[2], IRV_ALPHA);
    a[3] = (T)lift((float)a[3], (float)a[2], r, IRV_ALPHA);
    float l = __shfl_up_sync(FULL, (float)a[3], 1);
    a[0] = (T)lift((float)a[0], l, (float)a[1], IRV_BETA);
    a[2] = (T)lift((float)a[2], (float)a[1], (float)a[3], IRV_BETA);
    r = __shfl_down_sync(FULL, (float)a[0], 1);
    a[1] = (T)lift((float)a[1], (float)a[0], (float)a[2], IRV_GAMMA);
    a[3] = (T)lift((float)a[3], (float)a[2], r, IRV_GAMMA);
    l = __shfl_up_sync(FULL, (float)a[3], 1);
    a[0] = (T)lift((float)a[0], l, (float)a[1], IRV_DELTA);
    a[2] = (T)lift((float)a[2], (float)a[1], (float)a[3], IRV_DELTA);
    a[0] = (T)__fmul_rn((float)a[0], 1.0f / IRV_K);
    a[2] = (T)__fmul_rn((float)a[2], 1.0f / IRV_K);
    a[1] = (T)__fmul_rn((float)a[1], IRV_K);
    a[3] = (T)__fmul_rn((float)a[3], IRV_K);
  }
}

// horizontal synthesis
template <bool REV, typename T>
__device__ __forceinline__ void horz_syn(T (&a)[4]) {
  if (REV) {
    const int l = __shfl_up_sync(FULL, (int)a[3], 1);
    a[0] = (T)((int)a[0] - ((l + (int)a[1] + 2) >> 2));
    a[2] = (T)((int)a[2] - (((int)a[1] + (int)a[3] + 2) >> 2));
    const int r = __shfl_down_sync(FULL, (int)a[0], 1);
    a[1] = (T)((int)a[1] + (((int)a[0] + (int)a[2]) >> 1));
    a[3] = (T)((int)a[3] + (((int)a[2] + r) >> 1));
  } else {
    a[0] = (T)__fmul_rn((float)a[0], IRV_K);
    a[2] = (T)__fmul_rn((float)a[2], IRV_K);
    a[1] = (T)__fmul_rn((float)a[1], 1.0f / IRV_K);
    a[3] = (T)__fmul_rn((float)a[3], 1.0f / IRV_K);
    float l = __shfl_up_sync(FULL, (float)a[3], 1);
    a[0] = (T)lift((float)a[0], l, (float)a[1], -IRV_DELTA);
    a[2] = (T)lift((float)a[2], (float)a[1], (float)a[3], -IRV_DELTA);
    float r = __shfl_down_sync(FULL, (float)a[0], 1);
    a[1] = (T)lift((float)a[1], (float)a[0], (float)a[2], -IRV_GAMMA);
    a[3] = (T)lift((float)a[3], (float)a[2], r, -IRV_GAMMA);
    l = __shfl_up_sync(FULL, (float)a[3], 1);
    a[0] = (T)lift((float)a[0], l, (float)a[1], -IRV_BETA);
    a[2] = (T)lift((float)a[2], (float)a[1], (float)a[3], -IRV_BETA);
    r = __shfl_down_sync(FULL, (float)a[0], 1);
    a[1] = (T)lift((float)a[1], (float)a[0], (float)a[2], -IRV_ALPHA);
    a[3] = (T)lift((float)a[3], (float)a[2], r, -IRV_ALPHA);
  }
}

__device__ __forceinline__ uint32_t to_signmag_rev(int v, uint32_t shift) {
  return (v < 0 ? 0x80000000u : 0u) | ((uint32_t)(v < 0 ? -v : v) << shift);
}
__device__ __forceinline__ uint32_t to_signmag_irv(float v, float scale) {
  const int q = __float2int_rn(__fmul_rn(v, scale));
  return (q < 0 ? 0x80000000u : 0u) | (uint32_t)(q < 0 ? -q : q);
}

struct StripGeom {
  int x0, y0, x1, y1;       // resolution rectangle
  int u0;                   // absolute (even) column of this lane's first column
  int c[4];                 // source column indices (mirrored, relative to x0)
  bool has[4];              // output lane and column u0+i inside [x0, x1)
  bool lane_valid;          // any has[]
  bool interior;            // all four columns exist unmirrored (any lane, halo included)
  bool fast;                // warp-uniform: every lane's requests are whole aligned vectors (set by strip_fast_*)
  int R0, R1;               // output rows of this chunk [R0, R1), R0 even (absolute)
};

__device__ __forceinline__ bool strip_setup(const DwtJob& J, uint32_t strip, uint32_t chunk, uint32_t lane, StripGeom& g) {
  g.x0 = (int)J.x0; g.y0 = (int)J.y0; g.x1 = g.x0 + (int)J.w; g.y1 = g.y0 + (int)J.h;
  const int ue = g.x0 & ~1;
  g.u0 = ue + (int)strip * DS_COLS * DS_VALID + DS_COLS * ((int)lane - 1);
  const bool inner = lane >= 1 && lane <= DS_VALID;
  g.lane_valid = false;
  #pragma unroll
  for (int i = 0; i < 4; ++i) {
    g.c[i] = reflect_coord(g.u0 + i, g.x0, g.x1 - 1) - g.x0;
    g.has[i] = inner && g.u0 + i >= g.x0 && g.u0 + i < g.x1;
    g.lane_valid = g.lane_valid || g.has[i];
  }
  g.interior = g.u0 >= g.x0 && g.u0 + 3 < g.x1;
  g.fast = false;
  const int ye = g.y0 & ~1;
  g.R0 = ye + (int)chunk * (int)J.chunk_rows;
  g.R1 = min(g.R0 + (int)J.chunk_rows, g.y1);
  return g.R0 < g.y1;
}

// ---- asynchronous global -> shared copies.  Every lane owns a private FIFO of shared-memory slots:
// it requests the rows of the next iterations with cp.async (no registers are held while the data is
// in flight) and later reads back exactly the bytes it requested, so no cross-lane synchronisation
// is needed -- cp.async.wait_group orders a lane's own copies.

// A row is addressed as a pointer plus 32-bit byte offsets (column c at row + c * step); alignment is tested on
// the address itself.  step is the element size where the columns are contiguous (the coefficient arena, planar
// image rows), a multiple of it for interleaved image rows, which take the per-sample requests.
// request four 32-bit elements row[c[0..3]] into a 16-byte slot
__device__ __forceinline__ void issue4_w(unsigned char* d, const unsigned char* row, uint32_t step, const StripGeom& g) {
  const unsigned char* p = row + step * (uint32_t)g.c[0];
  if (g.interior && step == 4u && ((uint32_t)(size_t)p & 15u) == 0) cp_async<16>(d, p);
  else {
    #pragma unroll
    for (int i = 0; i < 4; ++i) cp_async<4>(d + 4 * i, row + step * (uint32_t)g.c[i]);
  }
}
__device__ __forceinline__ void issue4_u16(unsigned char* d, const unsigned char* row, uint32_t step, const StripGeom& g) {
  const unsigned char* p = row + step * (uint32_t)g.c[0];
  const uint32_t a = (uint32_t)(size_t)p;
  if (g.interior && step == 2u && (a & 7u) == 0) cp_async<8>(d, p);
  else if (g.interior && step == 2u && (a & 3u) == 0) { cp_async<4>(d, p); cp_async<4>(d + 4, p + 4); }
  else {                                   // mirrored, odd-aligned or interleaved columns: plain loads
    unsigned short* ds = reinterpret_cast<unsigned short*>(d);
    #pragma unroll
    for (int i = 0; i < 4; ++i) ds[i] = *reinterpret_cast<const unsigned short*>(row + step * (uint32_t)g.c[i]);
  }
}
__device__ __forceinline__ void issue4_u8(unsigned char* d, const unsigned char* row, uint32_t step, const StripGeom& g) {
  const unsigned char* p = row + step * (uint32_t)g.c[0];
  if (g.interior && step == 1u && ((uint32_t)(size_t)p & 3u) == 0) cp_async<4>(d, p);
  else {
    #pragma unroll
    for (int i = 0; i < 4; ++i) d[i] = row[step * (uint32_t)g.c[i]];
  }
}
// two consecutive 32-bit words
// the arena (256-byte aligned) is addressed with 32-bit word indices here: the host selects these kernels
// only when the coefficient arena has fewer than 2^32 words
__device__ __forceinline__ void store2_w(uint32_t* base, uint32_t idx, uint32_t a, uint32_t b, bool ha, bool hb) {
  // idx may have wrapped below zero for a lane whose first column is outside the band (ha false):
  // element indices are formed in 32 bits before they meet the 64-bit base
  if (ha && hb && (idx & 1u) == 0) *reinterpret_cast<uint2*>(base + idx) = make_uint2(a, b);
  else { if (ha) base[idx] = a; if (hb) base[idx + 1u] = b; }
}
template <typename T> __device__ __forceinline__ uint32_t as_bits(T v) { uint32_t r; memcpy(&r, &v, 4); return r; }
template <typename T> __device__ __forceinline__ T from_bits(uint32_t v) { T r; memcpy(&r, &v, 4); return r; }

// Warp-uniform decision, once per strip: are all requests of all lanes whole aligned vectors?  (True for every
// strip that does not touch the left / right edge when offsets and strides are even enough, i.e. almost
// always; the per-request tests above otherwise get if-converted and both variants are issued every time.)
template <int NC, int SRC>
__device__ __forceinline__ bool strip_fast_fwd(const DwtJob& J, const ImgView* V, const StripGeom& g) {
  constexpr bool FIRST = SRC != SRC_COEF;
  constexpr uint32_t ES = (SRC == SRC_U16) ? 2u : (SRC == SRC_U8 ? 1u : 4u);
  bool ok = g.interior;
  #pragma unroll
  for (int k = 0; k < (FIRST ? NC : 1); ++k) {
    const uint32_t off = FIRST ? (uint32_t)(size_t)V[k].org : (uint32_t)J.full_off[0] * 4u;
    const uint32_t pitch = FIRST ? (uint32_t)V[k].pitch : J.full_stride[0] * ES;
    ok = ok && (!FIRST || V[k].step == ES) && ((off + (uint32_t)g.c[0] * ES) % (4u * ES)) == 0 && (pitch % (4u * ES)) == 0;
  }
  return __all_sync(0xFFFFFFFFu, ok);
}
template <int NC>
__device__ __forceinline__ bool strip_fast_inv(const DwtJob& J, const StripGeom& g) {
  bool ok = g.interior;
  #pragma unroll
  for (int i = 0; i < 2; ++i) {               // first column of the low (i = 0) and of the high (i = 1) band
    const int ua = g.c[i] + g.x0;
    const int bx = (ua >> 1) - ((i & 1) ? (g.x0 >> 1) : ((g.x0 + 1) >> 1));
    // ... and the second column of the pair must be its neighbour
    const int ub = g.c[i + 2] + g.x0;
    const int bx2 = (ub >> 1) - ((i & 1) ? (g.x0 >> 1) : ((g.x0 + 1) >> 1));
    ok = ok && bx2 == bx + 1;
    #pragma unroll
    for (int k = 0; k < NC; ++k) {
      #pragma unroll
      for (int b = i; b < 4; b += 2) {
        const uint32_t off = (b == 0 && !J.last) ? (uint32_t)J.ll_off[k] : (uint32_t)J.band_off[k][b];
        const uint32_t str = (b == 0 && !J.last) ? J.ll_stride[k] : J.band_stride[k][b];
        ok = ok && (((off + (uint32_t)bx) | str) & 1u) == 0;
      }
    }
  }
  return __all_sync(0xFFFFFFFFu, ok);
}

// ---- interleaved first level (ILV variant): the three components of a colour-transform job sit next to each other
// in memory, S = 3 or 4 samples per pixel (RGB / RGBA).  A lane's four pixels are then 4 S contiguous samples: they
// travel as S whole requests of 4 ES bytes each (12 / 24 / 48 or 16 / 32 / 64 bytes per row) and sit in the lane's
// FIFO slot (16 ES bytes) exactly as in memory.  Warp-uniform gate as strip_fast_*: every lane interior, the first
// pixel of every lane and the pitch multiples of 4 ES bytes.
template <int SRC>
__device__ __forceinline__ bool strip_fast_ilv(const ImgView* V, const StripGeom& g, uint32_t S) {
  constexpr uint32_t ES = (SRC == SRC_U16) ? 2u : (SRC == SRC_U8 ? 1u : 4u);
  const uint32_t a = (uint32_t)(size_t)V[0].org + (uint32_t)g.c[0] * S * ES;
  return __all_sync(0xFFFFFFFFu, g.interior && (a % (4u * ES)) == 0 && ((uint32_t)V[0].pitch % (4u * ES)) == 0);
}
template <int SRC>
__device__ __forceinline__ void ilv_issue_row(const StripGeom& g, const ImgView* V, int vr, unsigned char* st, uint32_t S) {
  constexpr uint32_t ES = (SRC == SRC_U16) ? 2u : (SRC == SRC_U8 ? 1u : 4u);
  if (g.fast) {
    const unsigned char* p = V[0].org + ((uint32_t)vr * (uint32_t)V[0].pitch + (uint32_t)g.c[0] * S * ES);
    #pragma unroll
    for (int j = 0; j < 3; ++j) cp_async<4 * ES>(st + j * 4 * ES, p + j * 4 * ES);
    if (S == 4) cp_async<4 * ES>(st + 12 * ES, p + 12 * ES);
    return;
  }
  #pragma unroll
  for (int k = 0; k < 3; ++k) {              // edge lanes (mirrored columns) or misaligned rows: plain loads
    const unsigned char* row = V[k].org + (uint32_t)vr * (uint32_t)V[k].pitch;
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
      const unsigned char* q = row + (uint32_t)g.c[i] * V[k].step;
      unsigned char* d = st + ((uint32_t)i * S + (uint32_t)k) * ES;
      if (ES == 1) *d = *q;
      else if (ES == 2) *reinterpret_cast<unsigned short*>(d) = *reinterpret_cast<const unsigned short*>(q);
      else *reinterpret_cast<uint32_t*>(d) = *reinterpret_cast<const uint32_t*>(q);
    }
  }
}
// sample (pixel i, component k) of the 4 S samples at d (4-byte aligned)
template <int S, uint32_t ES>
__device__ __forceinline__ void ilv_unpack(const unsigned char* d, int (&iv)[3][4]) {
  uint32_t w[S * ES];
  #pragma unroll
  for (int j = 0; j < (int)(S * ES); ++j) w[j] = reinterpret_cast<const uint32_t*>(d)[j];
  #pragma unroll
  for (int i = 0; i < 4; ++i)
    #pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int n = i * S + k;
      iv[k][i] = ES == 1 ? (int)((w[n >> 2] >> (8 * (n & 3))) & 0xFFu)
               : ES == 2 ? (int)((w[n >> 1] >> (16 * (n & 1))) & 0xFFFFu) : (int)w[n];
    }
}
// the three components of four pixels (container values) to memory at p (4 ES-byte aligned): S = 3, three whole
// vectors of 4 ES bytes; S = 4, per pixel one vector for the first two components and one for the third, so the
// fourth sample of each pixel (a channel the codec does not code) is left as it is
template <int S, uint32_t ES>
__device__ __forceinline__ void ilv_store(unsigned char* p, const uint32_t (&q)[3][4]) {
  if (S == 3) {
    uint32_t w[3 * ES];
    #pragma unroll
    for (int j = 0; j < (int)(3 * ES); ++j) w[j] = 0;
    #pragma unroll
    for (int i = 0; i < 4; ++i)
      #pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int n = i * 3 + k;
        if (ES == 1) w[n >> 2] |= q[k][i] << (8 * (n & 3));
        else if (ES == 2) w[n >> 1] |= q[k][i] << (16 * (n & 1));
        else w[n] = q[k][i];
      }
    #pragma unroll
    for (int j = 0; j < 3; ++j) {
      if (ES == 1) reinterpret_cast<uint32_t*>(p)[j] = w[j];
      else if (ES == 2) reinterpret_cast<uint2*>(p)[j] = make_uint2(w[2 * j], w[2 * j + 1]);
      else reinterpret_cast<uint4*>(p)[j] = make_uint4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
    }
  } else {
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
      unsigned char* px = p + i * 4 * ES;
      if (ES == 1) { *reinterpret_cast<unsigned short*>(px) = (unsigned short)(q[0][i] | (q[1][i] << 8)); px[2] = (unsigned char)q[2][i]; }
      else if (ES == 2) { *reinterpret_cast<uint32_t*>(px) = q[0][i] | (q[1][i] << 16); *reinterpret_cast<unsigned short*>(px + 4) = (unsigned short)q[2][i]; }
      else { *reinterpret_cast<uint2*>(px) = make_uint2(q[0][i], q[1][i]); *reinterpret_cast<uint32_t*>(px + 8) = q[2][i]; }
    }
  }
}

// ---- forward ---------------------------------------------------------------------------------
// request source row v (mirrored into the resolution) into the row slot `st` (lane offset included); cpitch = bytes
// between the components' slots, or (ILV) samples per pixel
template <int NC, int SRC, bool ILV>
__device__ __forceinline__ void fwd_issue_row(const DwtJob& J, const StripGeom& g, const ImgView* V,
                                              const uint32_t* coef, int v, unsigned char* st, uint32_t cpitch)
{
  constexpr bool FIRST = SRC != SRC_COEF;     // the full-resolution side is the image
  constexpr uint32_t ES = (SRC == SRC_U16) ? 2u : (SRC == SRC_U8 ? 1u : 4u);
  const int vr = reflect_coord(v, g.y0, g.y1 - 1) - g.y0;
  if constexpr (ILV) { ilv_issue_row<SRC>(g, V, vr, st, cpitch); return; }
  if (g.fast) {                               // one aligned vector per component, no per-request tests
    #pragma unroll
    for (int k = 0; k < (FIRST ? NC : 1); ++k) {
      const unsigned char* p = FIRST
        ? V[k].org + ((uint32_t)vr * (uint32_t)V[k].pitch + (uint32_t)g.c[0] * ES)
        : reinterpret_cast<const unsigned char*>(coef) + ((uint32_t)J.full_off[0] * 4u + ((uint32_t)vr * J.full_stride[0] + (uint32_t)g.c[0]) * ES);
      cp_async<4 * ES>(st + (size_t)k * cpitch, p);
    }
    return;
  }
  if (FIRST) {
    #pragma unroll
    for (int k = 0; k < NC; ++k) {
      const unsigned char* row = V[k].org + (uint32_t)vr * (uint32_t)V[k].pitch;
      unsigned char* d = st + (size_t)k * cpitch;
      if (SRC == SRC_U16) issue4_u16(d, row, V[k].step, g);
      else if (SRC == SRC_U8) issue4_u8(d, row, V[k].step, g);
      else issue4_w(d, row, V[k].step, g);
    }
  } else {
    issue4_w(st, reinterpret_cast<const unsigned char*>(coef) + ((uint32_t)J.full_off[0] + (uint32_t)vr * J.full_stride[0]) * 4u, 4u, g);
  }
}

// read a row slot back: level shift / int->float and RCT / ICT at level 1
template <bool REV, int NC, int SRC, bool ILV>
__device__ __forceinline__ void fwd_read_row(const DwtJob& J, const unsigned char* st, uint32_t cpitch,
                                             typename Tp<REV>::T (&a)[NC][4])
{
  constexpr bool FIRST = SRC != SRC_COEF;     // the full-resolution side is the image
  typedef typename Tp<REV>::T T;
  if (FIRST) {
    int iv[NC][4];
    if constexpr (ILV) {
      constexpr uint32_t ES = (SRC == SRC_U16) ? 2u : (SRC == SRC_U8 ? 1u : 4u);
      if (cpitch == 3) ilv_unpack<3, ES>(st, iv); else ilv_unpack<4, ES>(st, iv);
    } else {
    #pragma unroll
    for (int k = 0; k < NC; ++k) {
      const unsigned char* d = st + (size_t)k * cpitch;
      if (SRC == SRC_U16) {
        const uint2 t = *reinterpret_cast<const uint2*>(d);
        iv[k][0] = (int)(t.x & 0xFFFF); iv[k][1] = (int)(t.x >> 16); iv[k][2] = (int)(t.y & 0xFFFF); iv[k][3] = (int)(t.y >> 16);
      } else if (SRC == SRC_U8) {
        const uint32_t t = *reinterpret_cast<const uint32_t*>(d);
        iv[k][0] = (int)(t & 0xFF); iv[k][1] = (int)((t >> 8) & 0xFF); iv[k][2] = (int)((t >> 16) & 0xFF); iv[k][3] = (int)(t >> 24);
      } else {
        const uint4 t = *reinterpret_cast<const uint4*>(d);
        iv[k][0] = (int)t.x; iv[k][1] = (int)t.y; iv[k][2] = (int)t.z; iv[k][3] = (int)t.w;
      }
    }
    }
    if (J.nlt_mask) {
      const int bias = (1 << (J.bit_depth - 1)) + 1;
      #pragma unroll
      for (int k = 0; k < NC; ++k)
        if ((J.nlt_mask >> k) & 1u) {
          #pragma unroll
          for (int i = 0; i < 4; ++i) iv[k][i] = nlt_type3(iv[k][i], bias);
        }
    }
    if (REV) {
      const int shift = J.is_signed ? 0 : (1 << (J.bit_depth - 1));
      #pragma unroll
      for (int k = 0; k < NC; ++k)
        #pragma unroll
        for (int i = 0; i < 4; ++i) iv[k][i] -= shift;
      if (NC == 3) {
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int rr = iv[0][i], gg = iv[1][i], bb = iv[2][i];
          iv[0][i] = (rr + (gg << 1) + bb) >> 2; iv[1][i] = bb - gg; iv[2][i] = rr - gg;
        }
      }
      #pragma unroll
      for (int k = 0; k < NC; ++k)
        #pragma unroll
        for (int i = 0; i < 4; ++i) a[k][i] = (T)iv[k][i];
    } else {
      const float mul = (float)(1.0 / (double)(1ull << J.bit_depth));
      const int half = J.is_signed ? 0 : (1 << (J.bit_depth - 1));
      float f[NC][4];
      #pragma unroll
      for (int k = 0; k < NC; ++k)
        #pragma unroll
        for (int i = 0; i < 4; ++i) f[k][i] = __fmul_rn((float)(iv[k][i] - half), mul);
      if (NC == 3) {
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float rr = f[0][i], gg = f[1][i], bb = f[2][i];
          const float yy = __fadd_rn(__fadd_rn(__fmul_rn(ICT_ALPHA_RF, rr), __fmul_rn(ICT_ALPHA_GF, gg)), __fmul_rn(ICT_ALPHA_BF, bb));
          f[0][i] = yy; f[1][i] = __fmul_rn(ICT_BETA_CBF, __fsub_rn(bb, yy)); f[2][i] = __fmul_rn(ICT_BETA_CRF, __fsub_rn(rr, yy));
        }
      }
      #pragma unroll
      for (int k = 0; k < NC; ++k)
        #pragma unroll
        for (int i = 0; i < 4; ++i) a[k][i] = (T)f[k][i];
    }
  } else {
    const uint4 t = *reinterpret_cast<const uint4*>(st);
    a[0][0] = from_bits<T>(t.x); a[0][1] = from_bits<T>(t.y); a[0][2] = from_bits<T>(t.z); a[0][3] = from_bits<T>(t.w);
  }
}

// store one emitted (vertically low, vertically high) row pair after horizontal analysis
template <bool REV, int NC>
__device__ __forceinline__ void fwd_store_pair(const DwtJob& J, const StripGeom& g, uint32_t* coef, int vlow,
                                               typename Tp<REV>::T (&lo)[NC][4], typename Tp<REV>::T (&hi)[NC][4])
{
  typedef typename Tp<REV>::T T;
  #pragma unroll
  for (int k = 0; k < NC; ++k) { horz_ana<REV, T>(lo[k]); horz_ana<REV, T>(hi[k]); }
  if (!g.lane_valid) return;
  const int bxl = (g.u0 >> 1) - ((g.x0 + 1) >> 1);      // index in horizontally-low bands
  const int bxh = (g.u0 >> 1) - (g.x0 >> 1);            // index in horizontally-high bands
  #pragma unroll
  for (int vpar = 0; vpar < 2; ++vpar) {
    const int v = vlow + vpar;
    if (v < g.y0 || v >= g.y1 || v < g.R0 || v >= g.R1) continue;
    const int by = (v >> 1) - (vpar ? (g.y0 >> 1) : ((g.y0 + 1) >> 1));
    #pragma unroll
    for (int k = 0; k < NC; ++k) {
      const T (&r)[4] = vpar ? hi[k] : lo[k];
      const int bl = vpar ? 2 : 0, bh = vpar ? 3 : 1;
      if (bl == 0 && !J.last)
        store2_w(coef, (uint32_t)J.ll_off[k] + (uint32_t)by * J.ll_stride[k] + (uint32_t)bxl, as_bits(r[0]), as_bits(r[2]), g.has[0], g.has[2]);
      else if (REV)
        store2_w(coef, (uint32_t)J.band_off[k][bl] + (uint32_t)by * J.band_stride[k][bl] + (uint32_t)bxl,
                 to_signmag_rev((int)r[0], J.band_shift[k][bl]), to_signmag_rev((int)r[2], J.band_shift[k][bl]), g.has[0], g.has[2]);
      else
        store2_w(coef, (uint32_t)J.band_off[k][bl] + (uint32_t)by * J.band_stride[k][bl] + (uint32_t)bxl,
                 to_signmag_irv((float)r[0], J.band_scale[k][bl]), to_signmag_irv((float)r[2], J.band_scale[k][bl]), g.has[0], g.has[2]);
      if (REV)
        store2_w(coef, (uint32_t)J.band_off[k][bh] + (uint32_t)by * J.band_stride[k][bh] + (uint32_t)bxh,
                 to_signmag_rev((int)r[1], J.band_shift[k][bh]), to_signmag_rev((int)r[3], J.band_shift[k][bh]), g.has[1], g.has[3]);
      else
        store2_w(coef, (uint32_t)J.band_off[k][bh] + (uint32_t)by * J.band_stride[k][bh] + (uint32_t)bxh,
                 to_signmag_irv((float)r[1], J.band_scale[k][bh]), to_signmag_irv((float)r[3], J.band_scale[k][bh]), g.has[1], g.has[3]);
    }
  }
}

// ILV: the interleaved layout variant (see ilv_issue_row), colour-transform jobs only
template <bool REV, int NC, int SRC, bool ILV>
__global__ void __launch_bounds__(DS_WARPS * 32, (REV || NC == 1) ? 5 : 3)
dwt_fwd_stream_kernel(const DwtJob* __restrict__ jobs, uint32_t njobs, const ImgComp* __restrict__ img,
                      uint32_t* __restrict__ coef)
{
  typedef typename Tp<REV>::T T;
  constexpr bool FIRSTK = SRC != SRC_COEF;
  __shared__ DwtJob sj;
  __shared__ ImgView sv[FIRSTK ? NC : 1];
  {
    uint32_t ji = find_job(jobs, njobs, blockIdx.x);
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&jobs[ji]);
    uint32_t* d = reinterpret_cast<uint32_t*>(&sj);
    for (uint32_t i = threadIdx.x; i < sizeof(DwtJob) / 4; i += blockDim.x) d[i] = s[i];
  }
  __syncthreads();
  if (FIRSTK) {
    if (threadIdx.x < NC) sv[threadIdx.x] = img_view(img, sj, threadIdx.x);
    __syncthreads();
  }
  const DwtJob& J = sj;
  const ImgView* V = sv;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // CTA = DS_WARPS adjacent strips of one row chunk
  const uint32_t cta = blockIdx.x - J.cta_base;
  const uint32_t strips_per_row = (J.tiles_x + DS_WARPS - 1) / DS_WARPS;
  const uint32_t strip = (cta % strips_per_row) * DS_WARPS + warp, chunk = J.chunk0 + cta / strips_per_row;
  if (strip >= J.tiles_x) return;
  StripGeom g;
  if (!strip_setup(J, strip, chunk, lane, g)) return;
  constexpr uint32_t ESK = (SRC == SRC_U16) ? 2u : (SRC == SRC_U8 ? 1u : 4u);
  const uint32_t S = ILV ? V[0].step / ESK : 0u;                       // ILV: samples per pixel
  g.fast = ILV ? strip_fast_ilv<SRC>(V, g, S) : strip_fast_fwd<NC, SRC>(J, V, g);

  // the lane's FIFO: DS_STAGES stages of one row pair each
  OJB_DYN_SMEM(unsigned char, s_ring);
  // 4 samples in their container (ILV: 4 pixels of up to 4 samples)
  const uint32_t slot = ILV ? 16u * ESK : ((SRC == SRC_U8 || SRC == SRC_U16) ? 8u : 16u);
  // bytes between the components of a row slot (ILV: samples per pixel, one slot holds them all)
  const uint32_t cpitch = ILV ? S : 32 * slot;
  const uint32_t row_bytes = ILV ? 32 * slot : NC * cpitch, stage_bytes = 2 * row_bytes;
  unsigned char* ring = s_ring + (size_t)warp * DS_STAGES * stage_bytes + (size_t)lane * slot;

  // iteration k consumes rows (2k-1, 2k); 5/3 emits the pair (2k-2, 2k-1), 9/7 the pair (2k-4, 2k-3)
  const int k0 = REV ? g.R0 / 2 : g.R0 / 2 - 1;
  const int k1 = REV ? (g.R1 + 1) / 2 : (g.R1 + 1) / 2 + 1;     // last pair covers rows up to R1-1
  T xe[NC][4];                                                // x[2k-2]
  {                                                           // priming row through the last stage
    unsigned char* sp = ring + (size_t)(DS_STAGES - 1) * stage_bytes;
    fwd_issue_row<NC, SRC, ILV>(J, g, V, coef, 2 * k0 - 2, sp, cpitch);
    cp_commit(); cp_wait<0>();
    fwd_read_row<REV, NC, SRC, ILV>(J, sp, cpitch, xe);
  }
  int issued = k0;
  #pragma unroll
  for (int s = 0; s < DS_STAGES - 1; ++s) {
    // rows (2 * issued - 1, 2 * issued) into the stage of iteration `issued`.  Both lifting loops repeat this pair:
    // routed through one lambda or helper, nvcc 12.9 allocates registers differently and the SASS changes
    if (issued <= k1) {
      unsigned char* st = ring + (size_t)((issued - k0) % DS_STAGES) * stage_bytes;
      fwd_issue_row<NC, SRC, ILV>(J, g, V, coef, 2 * issued - 1, st, cpitch);
      fwd_issue_row<NC, SRC, ILV>(J, g, V, coef, 2 * issued, st + row_bytes, cpitch);
    }
    cp_commit(); ++issued;
  }

  if (REV) {
    T hp[NC][4];                      // H[k-2]
    #pragma unroll
    for (int c = 0; c < NC; ++c)
      #pragma unroll
      for (int i = 0; i < 4; ++i) hp[c][i] = 0;
    for (int k = k0; k <= k1; ++k) {
      T xo[NC][4], xn[NC][4], lo[NC][4], hi[NC][4];
      cp_wait<DS_STAGES - 2>();
      const unsigned char* st = ring + (size_t)((k - k0) % DS_STAGES) * stage_bytes;
      fwd_read_row<REV, NC, SRC, ILV>(J, st, cpitch, xo);
      fwd_read_row<REV, NC, SRC, ILV>(J, st + row_bytes, cpitch, xn);
      #pragma unroll
      for (int c = 0; c < NC; ++c)
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int h = (int)xo[c][i] - (((int)xe[c][i] + (int)xn[c][i]) >> 1);       // H[k-1]
          const int l = (int)xe[c][i] + (((int)hp[c][i] + h + 2) >> 2);               // L[k-1]
          lo[c][i] = (T)l; hi[c][i] = (T)h;
          hp[c][i] = (T)h; xe[c][i] = xn[c][i];
        }
      if (issued <= k1) {             // refill the stage consumed one iteration ago
        unsigned char* sn = ring + (size_t)((issued - k0) % DS_STAGES) * stage_bytes;
        fwd_issue_row<NC, SRC, ILV>(J, g, V, coef, 2 * issued - 1, sn, cpitch);
        fwd_issue_row<NC, SRC, ILV>(J, g, V, coef, 2 * issued, sn + row_bytes, cpitch);
      }
      cp_commit(); ++issued;
      fwd_store_pair<REV, NC>(J, g, coef, 2 * k - 2, lo, hi);      // rows 2k-2 (low), 2k-1 (high)
    }
  } else {
    T d1[NC][4], s1[NC][4], d2[NC][4];   // d1[k-2], s1[k-2], d2[k-3]
    #pragma unroll
    for (int c = 0; c < NC; ++c)
      #pragma unroll
      for (int i = 0; i < 4; ++i) { d1[c][i] = 0; s1[c][i] = 0; d2[c][i] = 0; }
    const float Kinv = 1.0f / IRV_K;
    for (int k = k0; k <= k1; ++k) {
      T xo[NC][4], xn[NC][4], lo[NC][4], hi[NC][4];
      cp_wait<DS_STAGES - 2>();
      const unsigned char* st = ring + (size_t)((k - k0) % DS_STAGES) * stage_bytes;
      fwd_read_row<REV, NC, SRC, ILV>(J, st, cpitch, xo);
      fwd_read_row<REV, NC, SRC, ILV>(J, st + row_bytes, cpitch, xn);
      #pragma unroll
      for (int c = 0; c < NC; ++c)
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float nd1 = lift((float)xo[c][i], (float)xe[c][i], (float)xn[c][i], IRV_ALPHA);     // d1[k-1]
          const float ns1 = lift((float)xe[c][i], (float)d1[c][i], nd1, IRV_BETA);                  // s1[k-1]
          const float nd2 = lift((float)d1[c][i], (float)s1[c][i], ns1, IRV_GAMMA);                 // d2[k-2]
          const float ns2 = lift((float)s1[c][i], (float)d2[c][i], nd2, IRV_DELTA);                 // s2[k-2]
          lo[c][i] = (T)__fmul_rn(ns2, Kinv); hi[c][i] = (T)__fmul_rn(nd2, IRV_K);
          xe[c][i] = xn[c][i]; d1[c][i] = (T)nd1; s1[c][i] = (T)ns1; d2[c][i] = (T)nd2;
        }
      if (issued <= k1) {
        unsigned char* sn = ring + (size_t)((issued - k0) % DS_STAGES) * stage_bytes;
        fwd_issue_row<NC, SRC, ILV>(J, g, V, coef, 2 * issued - 1, sn, cpitch);
        fwd_issue_row<NC, SRC, ILV>(J, g, V, coef, 2 * issued, sn + row_bytes, cpitch);
      }
      cp_commit(); ++issued;
      fwd_store_pair<REV, NC>(J, g, coef, 2 * k - 4, lo, hi);      // rows 2k-4 (low), 2k-3 (high)
    }
  }
}

// ---- inverse ---------------------------------------------------------------------------------
// request the sub-band samples that interleave into rows (2j, 2j+1), columns u0..u0+3: per component
// four 8-byte slots (LL|HL of the vertically-low row, LH|HH of the vertically-high row)
template <int NC>
__device__ __forceinline__ void inv_issue_pair(const DwtJob& J, const StripGeom& g, const uint32_t* coef, int j,
                                               unsigned char* st)
{
  // mirrored absolute coordinates keep their parity, so each sample maps to a definite band
  int bx[4];
  #pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ua = g.c[i] + g.x0;
    bx[i] = (ua >> 1) - ((i & 1) ? (g.x0 >> 1) : ((g.x0 + 1) >> 1));
  }
  const int va = reflect_coord(2 * j, g.y0, g.y1 - 1), vb = reflect_coord(2 * j + 1, g.y0, g.y1 - 1);
  const int byl = (va >> 1) - ((g.y0 + 1) >> 1), byh = (vb >> 1) - (g.y0 >> 1);
  if (g.fast) {                               // every pair is one aligned 8-byte request
    #pragma unroll
    for (int k = 0; k < NC; ++k) {
      #pragma unroll
      for (int b = 0; b < 4; ++b) {
        const uint32_t row = (b == 0 && !J.last) ? (uint32_t)J.ll_off[k] + (uint32_t)byl * J.ll_stride[k]
                                                 : (uint32_t)J.band_off[k][b] + (uint32_t)(b < 2 ? byl : byh) * J.band_stride[k][b];
        cp_async<8>(st + (size_t)(k * 4 + b) * 32 * 8, coef + (row + (uint32_t)bx[b & 1]));
      }
    }
    return;
  }
  #pragma unroll
  for (int k = 0; k < NC; ++k) {
    #pragma unroll
    for (int b = 0; b < 4; ++b) {
      // 32-bit word indices into the arena (fewer than 2^32 words when these kernels are selected)
      const uint32_t row = (b == 0 && !J.last) ? (uint32_t)J.ll_off[k] + (uint32_t)byl * J.ll_stride[k]
                                               : (uint32_t)J.band_off[k][b] + (uint32_t)(b < 2 ? byl : byh) * J.band_stride[k][b];
      const uint32_t i0 = row + (uint32_t)bx[b & 1], i1 = row + (uint32_t)bx[(b & 1) + 2];
      unsigned char* d = st + (size_t)(k * 4 + b) * 32 * 8;
      if (g.interior && (i0 & 1u) == 0) cp_async<8>(d, coef + i0);
      else { cp_async<4>(d, coef + i0); cp_async<4>(d + 4, coef + i1); }
    }
  }
}

// read a requested pair back and undo the horizontal transform: L[..] = vertically-low row,
// H[..] = vertically-high row
template <bool REV, int NC>
__device__ __forceinline__ void inv_read_pair(const unsigned char* st, typename Tp<REV>::T (&L)[NC][4],
                                              typename Tp<REV>::T (&H)[NC][4])
{
  typedef typename Tp<REV>::T T;
  #pragma unroll
  for (int k = 0; k < NC; ++k) {
    const uint2 ll = *reinterpret_cast<const uint2*>(st + (size_t)(k * 4 + 0) * 32 * 8);
    const uint2 hl = *reinterpret_cast<const uint2*>(st + (size_t)(k * 4 + 1) * 32 * 8);
    const uint2 lh = *reinterpret_cast<const uint2*>(st + (size_t)(k * 4 + 2) * 32 * 8);
    const uint2 hh = *reinterpret_cast<const uint2*>(st + (size_t)(k * 4 + 3) * 32 * 8);
    L[k][0] = from_bits<T>(ll.x); L[k][1] = from_bits<T>(hl.x); L[k][2] = from_bits<T>(ll.y); L[k][3] = from_bits<T>(hl.y);
    H[k][0] = from_bits<T>(lh.x); H[k][1] = from_bits<T>(hh.x); H[k][2] = from_bits<T>(lh.y); H[k][3] = from_bits<T>(hh.y);
    horz_syn<REV, T>(L[k]);
    horz_syn<REV, T>(H[k]);
  }
}

// float -> integer as the reference's SIMD builds do it (cvtps: round to nearest, ties to even;
// ojph_colour_avx2.cpp:303).  The generic C path rounds ties away from zero (ojph_arch.h:317-326); the two
// differ only on exact halves, which zero-decomposition 9/7 components produce systematically.
__device__ __forceinline__ int round_haz(float t) { return __float2int_rn(t); }

template <bool REV, int NC, int SRC, bool ILV>
__device__ __forceinline__ void inv_store_row(const DwtJob& J, const StripGeom& g, const ImgView* V, uint32_t* coef,
                                              int v, typename Tp<REV>::T (&x)[NC][4])
{
  constexpr bool FIRST = SRC != SRC_COEF;     // the full-resolution side is the image
  typedef typename Tp<REV>::T T;
  if (!g.lane_valid || v < g.y0 || v >= g.y1 || v < g.R0 || v >= g.R1) return;
  const int cx = g.u0 - g.x0;
  const bool all4 = g.has[0] && g.has[3];
  if (!FIRST) {
    const uint32_t idx = (uint32_t)J.full_off[0] + (uint32_t)(v - g.y0) * J.full_stride[0] + (uint32_t)cx;
    // (idx wraps below zero when the lane's first column lies left of the resolution: 32-bit sums)
    if (all4 && (idx & 3u) == 0)
      *reinterpret_cast<uint4*>(coef + idx) = make_uint4(as_bits(x[0][0]), as_bits(x[0][1]), as_bits(x[0][2]), as_bits(x[0][3]));
    else {
      #pragma unroll
      for (int i = 0; i < 4; ++i) if (g.has[i]) coef[idx + (uint32_t)i] = as_bits(x[0][i]);
    }
    return;
  }
  int out[NC][4];
  if (REV) {
    int a[NC][4];
    #pragma unroll
    for (int k = 0; k < NC; ++k)
      #pragma unroll
      for (int i = 0; i < 4; ++i) a[k][i] = (int)x[k][i];
    if (NC == 3) {
      #pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int yy = a[0][i], cb = a[1][i], cr = a[2][i], gg = yy - ((cb + cr) >> 2);
        a[0][i] = cr + gg; a[1][i] = gg; a[2][i] = cb + gg;
      }
    }
    const int shift = J.is_signed ? 0 : (1 << (J.bit_depth - 1));
    #pragma unroll
    for (int k = 0; k < NC; ++k)
      #pragma unroll
      for (int i = 0; i < 4; ++i) out[k][i] = a[k][i] + shift;
  } else {
    float f[NC][4];
    #pragma unroll
    for (int k = 0; k < NC; ++k)
      #pragma unroll
      for (int i = 0; i < 4; ++i) f[k][i] = (float)x[k][i];
    if (NC == 3) {
      #pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float yy = f[0][i], cb = f[1][i], cr = f[2][i];
        f[1][i] = __fsub_rn(__fsub_rn(yy, __fmul_rn(ICT_GAMMA_CR2G, cr)), __fmul_rn(ICT_GAMMA_CB2G, cb));
        f[0][i] = __fadd_rn(yy, __fmul_rn(ICT_GAMMA_CR2R, cr));
        f[2][i] = __fadd_rn(yy, __fmul_rn(ICT_GAMMA_CB2B, cb));
      }
    }
    const int B = (int)J.bit_depth;
    const float mul = (float)(1ull << B);
    const int lo = -(1 << (B - 1)), hi = (1 << (B - 1)) - 1;
    const float flo = (float)lo, fhi = -(float)lo;
    const int half = J.is_signed ? 0 : (1 << (B - 1));
    #pragma unroll
    for (int k = 0; k < NC; ++k)
      #pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float t = __fmul_rn(f[k][i], mul);
        int q = round_haz(t);
        q = t >= flo ? q : lo; q = t < fhi ? q : hi;
        out[k][i] = q + half;
      }
  }
  if (J.nlt_mask) {
    const int bias = (1 << (J.bit_depth - 1)) + 1;
    #pragma unroll
    for (int k = 0; k < NC; ++k)
      if ((J.nlt_mask >> k) & 1u) {
        #pragma unroll
        for (int i = 0; i < 4; ++i) out[k][i] = nlt_type3(out[k][i], bias);
      }
  }
  // 8 / 16-bit containers: clamp to the component's range as the reference's file writers do
  // (gen_cvrt_32b*_to_*, yuv_out::write: src/apps/others/ojph_img_io.cpp:99-235, :1477-1516)
  const int smax = (1 << J.bit_depth) - 1;
  if constexpr (ILV) {                        // four whole pixels at a pixel-aligned address: vectors (ilv_store)
    constexpr uint32_t ES = (SRC == SRC_U16) ? 2u : (SRC == SRC_U8 ? 1u : 4u);
    unsigned char* p = V[0].org + (uint32_t)(v - g.y0) * (uint32_t)V[0].pitch + (uint32_t)cx * V[0].step;
    if (all4 && ((uint32_t)(size_t)p & (4u * ES - 1u)) == 0) {
      uint32_t q[3][4];
      #pragma unroll
      for (int k = 0; k < 3; ++k)
        #pragma unroll
        for (int i = 0; i < 4; ++i) q[k][i] = SRC == SRC_I32 ? (uint32_t)out[k][i] : (uint32_t)min(max(out[k][i], 0), smax);
      if (V[0].step == 3u * ES) ilv_store<3, ES>(p, q); else ilv_store<4, ES>(p, q);
      return;
    }
  }
  #pragma unroll
  for (int k = 0; k < NC; ++k) {
    // the row, then 32-bit byte offsets along it; a lane's first column lies left of the resolution (cx < 0) only
    // when has[0] is false, so the vector stores below never see the wrapped offset
    unsigned char* row = V[k].org + (uint32_t)(v - g.y0) * (uint32_t)V[k].pitch;
    const uint32_t step = V[k].step;
    unsigned char* p = row + (uint32_t)cx * step;
    const uint32_t a = (uint32_t)(size_t)p;
    if (SRC == SRC_U16) {
      uint32_t q[4];
      #pragma unroll
      for (int i = 0; i < 4; ++i) q[i] = (uint32_t)min(max(out[k][i], 0), smax);
      if (all4 && step == 2u && (a & 7u) == 0) *reinterpret_cast<uint2*>(p) = make_uint2(q[0] | (q[1] << 16), q[2] | (q[3] << 16));
      else {
        #pragma unroll
        for (int i = 0; i < 4; ++i) if (g.has[i]) *reinterpret_cast<unsigned short*>(row + (uint32_t)(cx + i) * step) = (unsigned short)q[i];
      }
    } else if (SRC == SRC_U8) {
      uint32_t q[4];
      #pragma unroll
      for (int i = 0; i < 4; ++i) q[i] = (uint32_t)min(max(out[k][i], 0), smax);
      if (all4 && step == 1u && (a & 3u) == 0) *reinterpret_cast<uint32_t*>(p) = q[0] | (q[1] << 8) | (q[2] << 16) | (q[3] << 24);
      else {
        #pragma unroll
        for (int i = 0; i < 4; ++i) if (g.has[i]) row[(uint32_t)(cx + i) * step] = (unsigned char)q[i];
      }
    } else {
      if (all4 && step == 4u && (a & 15u) == 0)
        *reinterpret_cast<uint4*>(p) = make_uint4((uint32_t)out[k][0], (uint32_t)out[k][1], (uint32_t)out[k][2], (uint32_t)out[k][3]);
      else {
        #pragma unroll
        for (int i = 0; i < 4; ++i) if (g.has[i]) *reinterpret_cast<int*>(row + (uint32_t)(cx + i) * step) = out[k][i];
      }
    }
  }
}

template <bool REV, int NC, int SRC, bool ILV>
__global__ void __launch_bounds__(DS_WARPS * 32, (REV || NC == 1) ? 5 : 3)
dwt_inv_stream_kernel(const DwtJob* __restrict__ jobs, uint32_t njobs, const ImgComp* __restrict__ img,
                      uint32_t* __restrict__ coef)
{
  typedef typename Tp<REV>::T T;
  constexpr bool FIRSTK = SRC != SRC_COEF;
  __shared__ DwtJob sj;
  __shared__ ImgView sv[FIRSTK ? NC : 1];
  {
    uint32_t ji = find_job(jobs, njobs, blockIdx.x);
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&jobs[ji]);
    uint32_t* d = reinterpret_cast<uint32_t*>(&sj);
    for (uint32_t i = threadIdx.x; i < sizeof(DwtJob) / 4; i += blockDim.x) d[i] = s[i];
  }
  __syncthreads();
  if (FIRSTK) {
    if (threadIdx.x < NC) sv[threadIdx.x] = img_view(img, sj, threadIdx.x);
    __syncthreads();
  }
  const DwtJob& J = sj;
  const ImgView* V = sv;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t cta = blockIdx.x - J.cta_base;
  const uint32_t strips_per_row = (J.tiles_x + DS_WARPS - 1) / DS_WARPS;
  const uint32_t strip = (cta % strips_per_row) * DS_WARPS + warp, chunk = J.chunk0 + cta / strips_per_row;
  if (strip >= J.tiles_x) return;
  StripGeom g;
  if (!strip_setup(J, strip, chunk, lane, g)) return;
  g.fast = strip_fast_inv<NC>(J, g);

  OJB_DYN_SMEM(unsigned char, s_ring);
  constexpr int NS = (NC == 3) ? DS_STAGES - 1 : DS_STAGES;       // three components: 3 KB per stage
  const uint32_t stage_bytes = NC * 4 * 32 * 8;
  unsigned char* ring = s_ring + (size_t)warp * NS * stage_bytes + (size_t)lane * 8;

  // iteration j consumes the band-row pair j; 5/3 emits rows (2j-1, 2j), 9/7 rows (2j-3, 2j-2)
  const int j0 = REV ? g.R0 / 2 : g.R0 / 2 - 1;
  const int j1 = REV ? (g.R1 + 1) / 2 : (g.R1 + 1) / 2 + 1;
  T hp[NC][4];                                                // H[j-1] (9/7: scaled)
  {
    T L[NC][4];
    unsigned char* sp = ring + (size_t)(NS - 1) * stage_bytes;   // priming pair through the last stage
    inv_issue_pair<NC>(J, g, coef, j0 - 1, sp);               // only H[j0-1] is needed
    cp_commit(); cp_wait<0>();
    inv_read_pair<REV, NC>(sp, L, hp);
  }
  int issued = j0;
  #pragma unroll
  for (int s = 0; s < NS - 1; ++s) {
    if (issued <= j1) inv_issue_pair<NC>(J, g, coef, issued, ring + (size_t)((issued - j0) % NS) * stage_bytes);
    cp_commit(); ++issued;
  }

  if (REV) {
    T xe[NC][4];                     // x[2j-2]
    #pragma unroll
    for (int c = 0; c < NC; ++c)
      #pragma unroll
      for (int i = 0; i < 4; ++i) xe[c][i] = 0;
    for (int j = j0; j <= j1; ++j) {
      T L[NC][4], H[NC][4], xo[NC][4], xn[NC][4];
      cp_wait<NS - 2>();
      inv_read_pair<REV, NC>(ring + (size_t)((j - j0) % NS) * stage_bytes, L, H);
      #pragma unroll
      for (int c = 0; c < NC; ++c)
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int e = (int)L[c][i] - (((int)hp[c][i] + (int)H[c][i] + 2) >> 2);     // x[2j]
          const int o = (int)hp[c][i] + (((int)xe[c][i] + e) >> 1);                   // x[2j-1]
          xn[c][i] = (T)e; xo[c][i] = (T)o;
          hp[c][i] = H[c][i]; xe[c][i] = (T)e;
        }
      if (issued <= j1) inv_issue_pair<NC>(J, g, coef, issued, ring + (size_t)((issued - j0) % NS) * stage_bytes);
      cp_commit(); ++issued;
      inv_store_row<REV, NC, SRC, ILV>(J, g, V, coef, 2 * j - 1, xo);
      inv_store_row<REV, NC, SRC, ILV>(J, g, V, coef, 2 * j, xn);
    }
  } else {
    T s1[NC][4], d1[NC][4], xe[NC][4];      // s1[j-1], d1[j-2], x_e[j-2]
    #pragma unroll
    for (int c = 0; c < NC; ++c)
      #pragma unroll
      for (int i = 0; i < 4; ++i) { hp[c][i] = (T)__fmul_rn((float)hp[c][i], 1.0f / IRV_K); s1[c][i] = 0; d1[c][i] = 0; xe[c][i] = 0; }
    for (int j = j0; j <= j1; ++j) {
      T L[NC][4], H[NC][4], xo[NC][4], xn[NC][4];
      cp_wait<NS - 2>();
      inv_read_pair<REV, NC>(ring + (size_t)((j - j0) % NS) * stage_bytes, L, H);
      #pragma unroll
      for (int c = 0; c < NC; ++c)
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float lr = __fmul_rn((float)L[c][i], IRV_K), hr = __fmul_rn((float)H[c][i], 1.0f / IRV_K);
          const float ns1 = lift(lr, (float)hp[c][i], hr, -IRV_DELTA);                          // s1[j]
          const float nd1 = lift((float)hp[c][i], (float)s1[c][i], ns1, -IRV_GAMMA);            // d1[j-1]
          const float nxe = lift((float)s1[c][i], (float)d1[c][i], nd1, -IRV_BETA);             // x_e[j-1]
          const float nxo = lift((float)d1[c][i], (float)xe[c][i], nxe, -IRV_ALPHA);            // x_o[j-2]
          xo[c][i] = (T)nxo; xn[c][i] = (T)nxe;
          hp[c][i] = (T)hr; s1[c][i] = (T)ns1; d1[c][i] = (T)nd1; xe[c][i] = (T)nxe;
        }
      if (issued <= j1) inv_issue_pair<NC>(J, g, coef, issued, ring + (size_t)((issued - j0) % NS) * stage_bytes);
      cp_commit(); ++issued;
      inv_store_row<REV, NC, SRC, ILV>(J, g, V, coef, 2 * j - 3, xo);
      inv_store_row<REV, NC, SRC, ILV>(J, g, V, coef, 2 * j - 2, xn);
    }
  }
}

template <bool REV, int NC, int SRC>
void launch_fwd(const DwtJob* jobs, uint32_t njobs, uint32_t ctas, const ImgComp* img, uint32_t* coef, cudaStream_t st,
                bool interleaved) {
  const size_t slot = (SRC == SRC_U8 || SRC == SRC_U16) ? 8 : 16;
  if constexpr (NC == 3 && SRC != SRC_COEF) {
    if (interleaved) {
      auto k = dwt_fwd_stream_kernel<REV, NC, SRC, true>;
      const size_t smem = (size_t)DS_WARPS * DS_STAGES * 2 * 32 * (4 * slot);     // 16 ES bytes per lane and row
      cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      OJB_LAUNCH(k, dim3(ctas), dim3(DS_WARPS * 32), smem, st, jobs, njobs, img, coef);
      return;
    }
  }
  auto k = dwt_fwd_stream_kernel<REV, NC, SRC, false>;
  const size_t smem = (size_t)DS_WARPS * DS_STAGES * 2 * NC * 32 * slot;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  OJB_LAUNCH(k, dim3(ctas), dim3(DS_WARPS * 32), smem, st, jobs, njobs, img, coef);
}
template <bool REV, int NC, int SRC>
void launch_inv(const DwtJob* jobs, uint32_t njobs, uint32_t ctas, const ImgComp* img, uint32_t* coef, cudaStream_t st,
                bool interleaved) {
  const size_t smem = (size_t)DS_WARPS * ((NC == 3) ? DS_STAGES - 1 : DS_STAGES) * NC * 4 * 32 * 8;
  if constexpr (NC == 3 && SRC != SRC_COEF) {
    if (interleaved) {
      auto k = dwt_inv_stream_kernel<REV, NC, SRC, true>;
      cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      OJB_LAUNCH(k, dim3(ctas), dim3(DS_WARPS * 32), smem, st, jobs, njobs, img, coef);
      return;
    }
  }
  auto k = dwt_inv_stream_kernel<REV, NC, SRC, false>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  OJB_LAUNCH(k, dim3(ctas), dim3(DS_WARPS * 32), smem, st, jobs, njobs, img, coef);
}

} // namespace

// strips across / row chunks down; the launch uses ceil(strips / DS_WARPS) * chunks CTAs
void dwt_stream_tiling(uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, bool reversible, bool forward,
                       uint32_t& strips, uint32_t& chunks, uint32_t& chunk_rows, uint32_t& ctas)
{
  const uint32_t SW = DS_COLS * DS_VALID;          // output columns per strip
  const uint32_t ue = x0 & ~1u, ye = y0 & ~1u;
  strips = (x0 + w - ue + SW - 1) / SW;
  // Rows per warp chunk.  A warp walks its chunk serially and re-reads the 2 (5/3) or 4 (9/7) rows above it;
  // measured on the 8K frame alone on one H100 80GB HBM3 at a 400 W power limit (OJB_DWT_CHUNK_ROWS 8 / 16 / 32 / 64):
  // forward 5/3 0.75 / 0.80 / 0.87 / 0.94 ms, forward 9/7 1.09 / 0.98 / 0.95 / 0.99 ms, inverse 5/3 0.71-0.74 ms
  // throughout, inverse 9/7 1.03 / 0.90 / 0.85 / 0.81 ms
  chunk_rows = forward ? (reversible ? 8u : 32u) : (uint32_t)DS_ROWS;
  {   // tuning knob: rows per warp chunk of the large resolutions (even)
    static const uint32_t knob = [] { const char* e = getenv("OJB_DWT_CHUNK_ROWS"); return e ? (uint32_t)atoi(e) & ~1u : 0u; }();
    if (knob >= 8) chunk_rows = knob;
  }
  // at least 8 warp chunks per SM of an H100 SXM (132 SMs)
  while (chunk_rows > 8 && strips * ((y0 + h - ye + chunk_rows - 1) / chunk_rows) < 132u * 8u) chunk_rows >>= 1;
  chunks = (y0 + h - ye + chunk_rows - 1) / chunk_rows;
  ctas = ((strips + DS_WARPS - 1) / DS_WARPS) * chunks;
}

void launch_dwt_fwd_stream(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                           uint32_t ncomp, bool first, uint32_t src_type, const ImgComp* img, bool interleaved, uint32_t* coef, cudaStream_t st)
{
  if (total_ctas == 0) return;
#define OJB_FWD(REV, NC, SRC) launch_fwd<REV, NC, SRC>(jobs, njobs, total_ctas, img, coef, st, interleaved)
#define OJB_FWD_SRC(REV, NC) do { if (src_type == SRC_U8) OJB_FWD(REV, NC, SRC_U8); else if (src_type == SRC_U16) OJB_FWD(REV, NC, SRC_U16); \
                                  else OJB_FWD(REV, NC, SRC_I32); } while (0)
  if (reversible) {
    if (!first) OJB_FWD(true, 1, SRC_COEF);
    else if (ncomp == 3) OJB_FWD_SRC(true, 3); else OJB_FWD_SRC(true, 1);
  } else {
    if (!first) OJB_FWD(false, 1, SRC_COEF);
    else if (ncomp == 3) OJB_FWD_SRC(false, 3); else OJB_FWD_SRC(false, 1);
  }
#undef OJB_FWD_SRC
#undef OJB_FWD
}

void launch_dwt_inv_stream(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                           uint32_t ncomp, bool first, uint32_t src_type, const ImgComp* img, bool interleaved, uint32_t* coef, cudaStream_t st)
{
  if (total_ctas == 0) return;
#define OJB_INV(REV, NC, SRC) launch_inv<REV, NC, SRC>(jobs, njobs, total_ctas, img, coef, st, interleaved)
#define OJB_INV_SRC(REV, NC) do { if (src_type == SRC_U8) OJB_INV(REV, NC, SRC_U8); else if (src_type == SRC_U16) OJB_INV(REV, NC, SRC_U16); \
                                  else OJB_INV(REV, NC, SRC_I32); } while (0)
  if (reversible) {
    if (!first) OJB_INV(true, 1, SRC_COEF);
    else if (ncomp == 3) OJB_INV_SRC(true, 3); else OJB_INV_SRC(true, 1);
  } else {
    if (!first) OJB_INV(false, 1, SRC_COEF);
    else if (ncomp == 3) OJB_INV_SRC(false, 3); else OJB_INV_SRC(false, 1);
  }
#undef OJB_INV_SRC
#undef OJB_INV
}

} // namespace ojb
