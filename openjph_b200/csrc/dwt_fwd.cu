// dwt_fwd.cu -- one forward DWT level (reversible 5/3 on int32, irreversible 9/7 on fp32) per
// launch, fused with what sits either side of it on the reference's encode path:
//   level 1 : sample fetch (u8 / u16 / i32) -> level shift or int->float -> RCT / ICT
//             (tile::push, src/core/codestream/ojph_tile.cpp:332-420; rev_convert,
//              irv_convert_to_float, rct_forward, ict_forward in src/core/transform/ojph_colour.cpp)
//   lifting : VERTICAL first, then horizontal on every produced line -- the order matters
//             for bit-exactness with integer rounding (resolution::push_line,
//             src/core/codestream/ojph_resolution.cpp:572-600 / :649-682; rev_vert_step,
//             rev_horz_ana, irv_* in src/core/transform/ojph_transform.cpp:209-783)
//   store   : LL raw (input of the next level) and HL/LH/HH quantised to MSB-aligned
//             sign-magnitude ready for the block coder (tx_to_cb32,
//             src/core/codestream/ojph_codestream_gen.cpp:59-121)
// One CTA owns a 128x32 tile (+4 halo) of the resolution in shared memory: one HBM read and
// one HBM write per sample per level, no intermediate round trip.  Border handling is
// whole-sample symmetric extension done at load time (mirrored coordinates), which is what
// the reference's per-step lp[-1]/lp[w] extension amounts to.
#include "dwt_common.cuh"
#include "ojb_kernels.h"

namespace ojb {

namespace {

// sample type of the transform: int32 (5/3), fp32 (9/7), int64 (5/3 when the precision exceeds 32 bits: the reference's
// 64-bit line buffers, rev_vert_step / rev_horz_ana on si64, ojph_transform.cpp:316-332, :497-509)
template <bool REV, bool WIDE> struct Px;
template <> struct Px<true, false>  { typedef int T; typedef int I; };
template <> struct Px<false, false> { typedef float T; typedef int I; };
template <> struct Px<true, true>   { typedef long long T; typedef long long I; };

__device__ __forceinline__ int load_sample(const unsigned char* p, uint32_t type) {
  if (type == SRC_U8) return (int)*p;
  if (type == SRC_U16) return (int)*reinterpret_cast<const unsigned short*>(p);
  return *reinterpret_cast<const int*>(p);
}

// 9/7: dst += coeff * (a + b), separate multiply and add (no FMA), ojph_transform.cpp:703
__device__ __forceinline__ float irv_step(float d, float a, float b, float c) {
  return __fadd_rn(d, __fmul_rn(c, __fadd_rn(a, b)));
}

template <bool REV, bool WIDE>
__global__ void __launch_bounds__(DW_THREADS)
dwt_fwd_kernel(const DwtJob* __restrict__ jobs, uint32_t njobs, const ImgComp* __restrict__ img,
               uint32_t* __restrict__ coef)
{
  typedef typename Px<REV, WIDE>::T T;
  typedef typename Px<REV, WIDE>::I I;
  OJB_DYN_SMEM(T, smem);
  __shared__ DwtJob sj;
  __shared__ ImgView sv[3];
  {
    uint32_t ji = find_job(jobs, njobs, blockIdx.x);
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&jobs[ji]);
    uint32_t* d = reinterpret_cast<uint32_t*>(&sj);
    for (uint32_t i = threadIdx.x; i < sizeof(DwtJob) / 4; i += blockDim.x) d[i] = s[i];
  }
  __syncthreads();
  if (sj.first && threadIdx.x < sj.ncomp) sv[threadIdx.x] = img_view(img, sj, threadIdx.x);
  __syncthreads();
  const DwtJob& J = sj;
  const uint32_t tid = threadIdx.x;
  const uint32_t local = blockIdx.x - J.cta_base;
  const uint32_t tx = local % J.tiles_x, ty = local / J.tiles_x;
  const int x0 = (int)J.x0, y0 = (int)J.y0, x1 = x0 + (int)J.w, y1 = y0 + (int)J.h;
  const int U0 = (x0 / DW_TW) * DW_TW + (int)tx * DW_TW;      // absolute tile origin (even)
  const int V0 = (y0 / DW_TH) * DW_TH + (int)ty * DW_TH;
  const uint32_t nc = J.ncomp;

  // ---- load with mirrored coordinates, convert, colour-transform
  for (uint32_t e = tid; e < DW_ROWS * DW_COLS; e += DW_THREADS) {
    const uint32_t r = e / DW_COLS, c = e - r * DW_COLS;
    const int u = reflect_coord(U0 - DW_H + (int)c, x0, x1 - 1);
    const int v = reflect_coord(V0 - DW_H + (int)r, y0, y1 - 1);
    T val[3];
    if (J.first) {
      I iv[3];
      for (uint32_t k = 0; k < 3; ++k) if (k < nc)
        iv[k] = (I)load_sample(sv[k].org + (size_t)(v - y0) * sv[k].pitch + (size_t)(u - x0) * sv[k].step, J.src_type);
      if (J.nlt_mask) {
        const I bias = ((I)1 << (J.bit_depth - 1)) + 1;
        for (uint32_t k = 0; k < 3; ++k) if (k < nc) if ((J.nlt_mask >> k) & 1u) iv[k] = iv[k] >= 0 ? iv[k] : -iv[k] - bias;
      }
      if (REV) {
        const I shift = J.is_signed ? (I)0 : ((I)1 << (J.bit_depth - 1));
        for (uint32_t k = 0; k < 3; ++k) if (k < nc) iv[k] -= shift;
        // with the colour transform the reference converts into 32-bit temporary lines whatever the precision
        // (tile::pre_alloc / finalize_alloc, ojph_tile.cpp:181-183, :312-317): the level-shifted samples wrap to
        // si32 before the (64-bit) RCT -- byte-identical streams for 32-bit samples need the same
        if (WIDE && nc == 3)
          for (uint32_t k = 0; k < 3; ++k) if (k < nc) iv[k] = (I)(int)iv[k];
        if (nc == 3) {   // RCT
          I rr = iv[0], gg = iv[1], bb = iv[2];
          iv[0] = (rr + (gg << 1) + bb) >> 2; iv[1] = bb - gg; iv[2] = rr - gg;
        }
        for (uint32_t k = 0; k < 3; ++k) if (k < nc) val[k] = (T)iv[k];
      } else {
        const float mul = (float)(1.0 / (double)(1ull << J.bit_depth));
        const int half = J.is_signed ? 0 : (1 << (J.bit_depth - 1));
        float f[3];
        for (uint32_t k = 0; k < 3; ++k) if (k < nc) f[k] = __fmul_rn((float)((int)iv[k] - half), mul);
        if (nc == 3) {   // ICT
          float rr = f[0], gg = f[1], bb = f[2];
          float yy = __fadd_rn(__fadd_rn(__fmul_rn(ICT_ALPHA_RF, rr), __fmul_rn(ICT_ALPHA_GF, gg)),
                               __fmul_rn(ICT_ALPHA_BF, bb));
          f[0] = yy;
          f[1] = __fmul_rn(ICT_BETA_CBF, __fsub_rn(bb, yy));
          f[2] = __fmul_rn(ICT_BETA_CRF, __fsub_rn(rr, yy));
        }
        for (uint32_t k = 0; k < 3; ++k) if (k < nc) val[k] = (T)f[k];
      }
    } else {
      const T* src = reinterpret_cast<const T*>(coef) + J.full_off[0];
      val[0] = src[(size_t)(v - y0) * J.full_stride[0] + (size_t)(u - x0)];
    }
    for (uint32_t k = 0; k < 3; ++k) if (k < nc) smem[k * DW_TILE_WORDS + r * DW_PITCH + c] = val[k];
  }
  __syncthreads();

  // One lifting step of the kernel in analysis direction; steps are numbered in synthesis order (param_atk,
  // ojph_params_local.h:1103-1232): step s touches the samples of parity s & 1 and analysis runs them last to first
  // (gen_rev_vert_step / gen_irv_vert_step, ojph_transform.cpp:209-262, :691-704).  The built-in 5/3 and 9/7 are the
  // same formula with their table values (init_rev53 / init_irv97, ojph_params.cpp:2870-2895).
  auto lift = [&](T d, T a, T b, int s) -> T {
    if (REV) return (T)((I)d + (((I)J.step_b[s] + (I)J.step_a[s] * ((I)a + (I)b)) >> J.step_e[s]));
    return (T)irv_step((float)d, (float)a, (float)b, J.step_A[s]);
  };
  const int NS = (int)J.nsteps;
  // ---- vertical lifting on every column (halo columns too: they feed the horizontal pass)
  if (J.vsplit) {
    if (J.h > 1) {
      for (int i = 0; i < NS; ++i) {
        const int s = NS - 1 - i, par = s & 1;
        int rfirst = i + 1; if ((rfirst & 1) != par) ++rfirst;
        int rlast = DW_ROWS - 2 - i; if ((rlast & 1) != par) --rlast;
        const int count = ((rlast - rfirst) / 2 + 1) * DW_COLS;
        for (uint32_t k = 0; k < nc; ++k) {
          T* t = smem + k * DW_TILE_WORDS;
          for (int e = (int)tid; e < count; e += DW_THREADS) {
            const int rr = e / DW_COLS, c = e - rr * DW_COLS;
            const int r = rfirst + 2 * rr;
            t[r * DW_PITCH + c] = lift(t[r * DW_PITCH + c], t[(r - 1) * DW_PITCH + c], t[(r + 1) * DW_PITCH + c], s);
          }
        }
        __syncthreads();
      }
      if (!REV) {      // low rows * 1/K, high rows * K (ojph_resolution.cpp:662-676)
        const float K = J.K, Kinv = 1.0f / J.K;
        for (uint32_t k = 0; k < nc; ++k) {
          T* t = smem + k * DW_TILE_WORDS;
          for (uint32_t e = tid; e < DW_TH * DW_COLS; e += DW_THREADS) {
            const uint32_t rr = e / DW_COLS, c = e - rr * DW_COLS, r = DW_H + rr;
            t[r * DW_PITCH + c] = (T)__fmul_rn((float)t[r * DW_PITCH + c], (r & 1) ? K : Kinv);
          }
        }
        __syncthreads();
      }
    } else if (y0 & 1) {   // a single odd row is a high-pass sample: x2 (ojph_resolution.cpp:613-628)
      for (uint32_t k = 0; k < nc; ++k) {
        T* t = smem + k * DW_TILE_WORDS;
        for (uint32_t e = tid; e < DW_ROWS * DW_COLS; e += DW_THREADS) {
          const uint32_t r = e / DW_COLS, c = e - r * DW_COLS;
          t[r * DW_PITCH + c] = REV ? (T)((I)t[r * DW_PITCH + c] << 1) : (T)__fmul_rn((float)t[r * DW_PITCH + c], 2.0f);
        }
      }
      __syncthreads();
    }
  }
  // ---- horizontal lifting on the rows this tile outputs
  if (J.hsplit && J.w > 1) {
    for (int i = 0; i < NS; ++i) {
      const int s = NS - 1 - i, par = s & 1;
      int cfirst = i + 1; if ((cfirst & 1) != par) ++cfirst;
      int clast = DW_COLS - 2 - i; if ((clast & 1) != par) --clast;
      const int ncols = (clast - cfirst) / 2 + 1;
      const int count = DW_TH * ncols;
      for (uint32_t k = 0; k < nc; ++k) {
        T* t = smem + k * DW_TILE_WORDS;
        for (int e = (int)tid; e < count; e += DW_THREADS) {
          const int rr = e / ncols, j = e - rr * ncols;
          const int r = DW_H + rr, c = cfirst + 2 * j;
          t[r * DW_PITCH + c] = lift(t[r * DW_PITCH + c], t[r * DW_PITCH + c - 1], t[r * DW_PITCH + c + 1], s);
        }
      }
      __syncthreads();
    }
  }

  // ---- store: de-interleave into LL / HL / LH / HH (a level that splits one way only has LL and HL, or LL and LH)
  const bool hs = J.hsplit != 0, vs = J.vsplit != 0;
  const bool hscale = !REV && hs && J.w > 1;
  const bool wodd1 = hs && J.w == 1 && (x0 & 1);         // single odd column: x2
  const uint32_t nrows = vs ? DW_TH / 2 : DW_TH, ncols = hs ? DW_TW / 2 : DW_TW;
  const float Kh = J.K, Kl = 1.0f / J.K;
  for (uint32_t k = 0; k < nc; ++k) {
    const T* t = smem + k * DW_TILE_WORDS;
    for (uint32_t band = 0; band < 4; ++band) {
      const int bh = (int)(band & 1), bv = (int)(band >> 1);
      if ((bh && !hs) || (bv && !vs)) continue;
      for (uint32_t e = tid; e < nrows * ncols; e += DW_THREADS) {
        const int rr = (int)(e / ncols), cc = (int)(e - (uint32_t)rr * ncols);
        const int r = DW_H + (vs ? 2 * rr + bv : rr), c = DW_H + (hs ? 2 * cc + bh : cc);
        const int u = U0 + c - DW_H, v = V0 + r - DW_H;
        if (u < x0 || u >= x1 || v < y0 || v >= y1) continue;
        T val = t[r * DW_PITCH + c];
        // with a single row / column the lone sample keeps its parity class
        const int bx = hs ? (u >> 1) - (bh ? (x0 >> 1) : ((x0 + 1) >> 1)) : u - x0;
        const int by = vs ? (v >> 1) - (bv ? (y0 >> 1) : ((y0 + 1) >> 1)) : v - y0;
        if (hscale) val = (T)__fmul_rn((float)val, bh ? Kh : Kl);
        if (wodd1) val = REV ? (T)((I)val << 1) : (T)__fmul_rn((float)val, 2.0f);
        if (band == 0 && !J.last) {
          reinterpret_cast<T*>(coef)[J.ll_off[k] + (size_t)by * J.ll_stride[k] + (size_t)bx] = val;
        } else {
          if (WIDE) {          // 64-bit sign-magnitude words (gen_rev_tx_to_cb64, ojph_codestream_gen.cpp:81-100)
            const long long iv = (long long)val;
            const unsigned long long mag = (unsigned long long)(iv < 0 ? -iv : iv) << J.band_shift[k][band];
            reinterpret_cast<unsigned long long*>(coef)[J.band_off[k][band] + (size_t)by * J.band_stride[k][band] + (size_t)bx] =
              (iv < 0 ? 0x8000000000000000ull : 0ull) | mag;
            continue;
          }
          uint32_t sm;
          if (REV) {
            const int iv = (int)val;
            const uint32_t mag = (uint32_t)(iv < 0 ? -iv : iv) << J.band_shift[k][band];
            sm = (iv < 0 ? 0x80000000u : 0u) | mag;
          } else {
            const int q = __float2int_rn(__fmul_rn((float)val, J.band_scale[k][band]));
            sm = (q < 0 ? 0x80000000u : 0u) | (uint32_t)(q < 0 ? -q : q);
          }
          coef[J.band_off[k][band] + (size_t)by * J.band_stride[k][band] + (size_t)bx] = sm;
        }
      }
    }
  }
}

} // namespace

void dwt_tiling(uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, uint32_t& tx, uint32_t& ty) {
  if (w == 0 || h == 0) { tx = ty = 0; return; }
  tx = (x0 + w + DW_TW - 1) / DW_TW - x0 / DW_TW;
  ty = (y0 + h + DW_TH - 1) / DW_TH - y0 / DW_TH;
}

void launch_dwt_fwd(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                    uint32_t max_ncomp, const ImgComp* img, uint32_t* coef, cudaStream_t st, bool wide)
{
  if (total_ctas == 0) return;
  size_t smem = (size_t)max_ncomp * DW_TILE_WORDS * (wide ? 8 : 4);
  if (reversible && wide) {
    auto k = dwt_fwd_kernel<true, true>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    OJB_LAUNCH(k, dim3(total_ctas), dim3(DW_THREADS), smem, st, jobs, njobs, img, coef);
  } else if (reversible) {
    auto k = dwt_fwd_kernel<true, false>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    OJB_LAUNCH(k, dim3(total_ctas), dim3(DW_THREADS), smem, st, jobs, njobs, img, coef);
  } else {
    auto k = dwt_fwd_kernel<false, false>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    OJB_LAUNCH(k, dim3(total_ctas), dim3(DW_THREADS), smem, st, jobs, njobs, img, coef);
  }
}

} // namespace ojb
