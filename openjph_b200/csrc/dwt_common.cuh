// dwt_common.cuh -- shared pieces of the forward / inverse lifting kernels.
#pragma once
#include "ojb_device.h"

namespace ojb {

#define DW_TW 128            // tile width  (samples of the resolution being split/merged)
#define DW_TH 32             // tile height
#define DW_H 8               // halo on every side: one sample per lifting step (9/7 needs 4; ATK kernels up to 8)
#define DW_COLS (DW_TW + 2 * DW_H)
#define DW_ROWS (DW_TH + 2 * DW_H)
#define DW_PITCH (DW_COLS + 1)
#define DW_THREADS 256
#define DW_TILE_WORDS (DW_ROWS * DW_PITCH)

// 9/7 lifting constants and K exactly as the reference rounds them to float
// (src/core/codestream/ojph_params.cpp:2870-2881)
#define IRV_ALPHA ((float)-1.586134342059924)
#define IRV_BETA  ((float)-0.052980118572961)
#define IRV_GAMMA ((float)0.882911075530934)
#define IRV_DELTA ((float)0.443506852043971)
#define IRV_K     ((float)1.230174104914001)

// ICT constants derived in double then rounded (src/core/transform/ojph_colour.cpp:220-230)
#define ICT_ALPHA_RF 0.299f
#define ICT_ALPHA_GF 0.587f
#define ICT_ALPHA_BF 0.114f
#define ICT_BETA_CBF ((float)(0.5 / (1.0 - (double)0.114f)))
#define ICT_BETA_CRF ((float)(0.5 / (1.0 - (double)0.299f)))
#define ICT_GAMMA_CB2G ((float)(2.0 * (double)0.114f * (1.0 - (double)0.114f) / (double)0.587f))
#define ICT_GAMMA_CR2G ((float)(2.0 * (double)0.299f * (1.0 - (double)0.299f) / (double)0.587f))
#define ICT_GAMMA_CB2B ((float)(2.0 * (1.0 - (double)0.114f)))
#define ICT_GAMMA_CR2R ((float)(2.0 * (1.0 - (double)0.299f)))

// whole-sample symmetric extension of coordinate u into [lo, hi] (hi inclusive)
__device__ __forceinline__ int reflect_coord(int u, int lo, int hi) {
  if (u >= lo && u <= hi) return u;
  int n = hi - lo;
  if (n == 0) return lo;
  int period = 2 * n;
  int t = (u - lo) % period;
  if (t < 0) t += period;
  if (t > n) t = period - t;
  return lo + t;
}

// NLT type 3, both directions (gen_rev_convert_nlt_type3, ojph_colour.cpp:273-310; the irreversible
// conversions apply the same map, :343-351 and :405-411): two's complement <-> a sign-magnitude ordering of
// the negative values, bias = 2^(B-1) + 1; an involution
__device__ __forceinline__ int nlt_type3(int v, int bias) { return v >= 0 ? v : -v - bias; }

__device__ __forceinline__ uint32_t src_esize(uint32_t src_type) { return src_type == SRC_U8 ? 1u : (src_type == SRC_U16 ? 2u : 4u); }

// component slot k of a first-level job as the kernels address it: sample (u, v) of the resolution (relative to its
// origin) at org + v * pitch + u * step, all in bytes
struct ImgView { unsigned char* org; uint64_t pitch; uint32_t step, pad; };
__device__ __forceinline__ ImgView img_view(const ImgComp* img, const DwtJob& J, uint32_t k) {
  const ImgComp c = img[J.img_comp[k]];
  ImgView w;
  w.step = c.col * src_esize(J.src_type); w.pitch = c.pitch; w.pad = 0;
  w.org = reinterpret_cast<unsigned char*>(c.base) + (size_t)J.img_y[k] * c.pitch + (size_t)J.img_x[k] * w.step;
  return w;
}

// locate the job a CTA belongs to (jobs sorted by cta_base)
__device__ __forceinline__ uint32_t find_job(const DwtJob* jobs, uint32_t njobs, uint32_t cta) {
  uint32_t lo = 0, hi = njobs;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (jobs[mid].cta_base <= cta) lo = mid; else hi = mid;
  }
  return lo;
}

} // namespace ojb
