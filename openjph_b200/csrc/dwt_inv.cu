// dwt_inv.cu -- one inverse DWT level (5/3 int32 / 9/7 fp32) per launch, fused with what sits
// either side of it on the reference's decode path:
//   load    : LL + HL/LH/HH coefficient planes (already de-quantised by the block decoder's
//             fused tx_from_cb32, src/core/codestream/ojph_codestream_gen.cpp:124-168)
//   lifting : HORIZONTAL synthesis first, then vertical (resolution::pull_line,
//             src/core/codestream/ojph_resolution.cpp:738-781 / :841-898; rev_horz_syn,
//             rev_vert_step(synthesis), irv_* in src/core/transform/ojph_transform.cpp:514-849)
//   top level: inverse RCT / ICT, level shift or float->int with rounding and clamping, store
//             to the image in its container type (tile::pull, ojph_tile.cpp:425-516;
//             rct_backward, ict_backward, rev_convert, irv_convert_to_integer in ojph_colour.cpp)
// Same tiling as dwt_fwd.cu: a 128x32 output tile (+4 halo) per CTA in shared memory.
#include "dwt_common.cuh"
#include "ojb_kernels.h"

namespace ojb {

namespace {

template <bool REV, bool WIDE> struct PxI;
template <> struct PxI<true, false>  { typedef int T; typedef int I; };
template <> struct PxI<false, false> { typedef float T; typedef int I; };
template <> struct PxI<true, true>   { typedef long long T; typedef long long I; };      // 64-bit lines (precision > 32 bits)

// 8 / 16-bit containers clamp to the component's range [0, smax] as the reference's file writers do
__device__ __forceinline__ void store_sample(unsigned char* p, uint32_t type, int v, int smax) {
  if (type == SRC_U8) *p = (unsigned char)min(max(v, 0), smax);
  else if (type == SRC_U16) *reinterpret_cast<unsigned short*>(p) = (unsigned short)min(max(v, 0), smax);
  else *reinterpret_cast<int*>(p) = v;
}

// float -> integer as the reference's SIMD builds do it (cvtps: round to nearest, ties to even;
// ojph_colour_avx2.cpp:303).  The generic C path rounds ties away from zero (ojph_arch.h:317-326); the two
// differ only on exact halves, which zero-decomposition 9/7 components produce systematically.
__device__ __forceinline__ int round_haz(float t) { return __float2int_rn(t); }

template <bool REV, bool WIDE>
__global__ void __launch_bounds__(DW_THREADS)
dwt_inv_kernel(const DwtJob* __restrict__ jobs, uint32_t njobs, const ImgComp* __restrict__ img,
               uint32_t* __restrict__ coef)
{
  typedef typename PxI<REV, WIDE>::T T;
  typedef typename PxI<REV, WIDE>::I I;
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
  const int U0 = (x0 / DW_TW) * DW_TW + (int)tx * DW_TW;
  const int V0 = (y0 / DW_TH) * DW_TH + (int)ty * DW_TH;
  const uint32_t nc = J.ncomp;
  const T* cf = reinterpret_cast<const T*>(coef);

  // ---- load: interleave the four bands (mirrored coordinates at the borders)
  for (uint32_t e = tid; e < DW_ROWS * DW_COLS; e += DW_THREADS) {
    const uint32_t r = e / DW_COLS, c = e - r * DW_COLS;
    const int u = reflect_coord(U0 - DW_H + (int)c, x0, x1 - 1);
    const int v = reflect_coord(V0 - DW_H + (int)r, y0, y1 - 1);
    for (uint32_t k = 0; k < nc; ++k) {
      T val;
      {
        // a level that splits one way only (DFS) interleaves LL with HL along x, or LL with LH along y
        const int bh = J.hsplit ? (u & 1) : 0, bv = J.vsplit ? (v & 1) : 0, band = bh + 2 * bv;
        const int bx = J.hsplit ? (u >> 1) - (bh ? (x0 >> 1) : ((x0 + 1) >> 1)) : u - x0;
        const int by = J.vsplit ? (v >> 1) - (bv ? (y0 >> 1) : ((y0 + 1) >> 1)) : v - y0;
        if (band == 0 && !J.last) val = cf[J.ll_off[k] + (size_t)by * J.ll_stride[k] + (size_t)bx];
        else val = cf[J.band_off[k][band] + (size_t)by * J.band_stride[k][band] + (size_t)bx];
      }
      smem[k * DW_TILE_WORDS + r * DW_PITCH + c] = val;
    }
  }
  __syncthreads();

  // One lifting step in synthesis direction, steps in the kernel's own (synthesis) order: step s acts on the samples
  // of parity s & 1 (gen_rev_horz_syn / gen_irv_horz_syn, ojph_transform.cpp:514-560, :785-849)
  auto unlift = [&](T d, T a, T b, int s) -> T {
    if (REV) return (T)((I)d - (((I)J.step_b[s] + (I)J.step_a[s] * ((I)a + (I)b)) >> J.step_e[s]));
    return (T)__fadd_rn((float)d, __fmul_rn(-J.step_A[s], __fadd_rn((float)a, (float)b)));
  };
  const int NS = (int)J.nsteps;
  // ---- horizontal synthesis on every row (halo rows feed the vertical pass)
  if (J.hsplit) {
    if (J.w > 1) {
      if (!REV) {   // low * K, high * 1/K (irv_horz_syn, ojph_transform.cpp:797-809)
        const float K = J.K, Kinv = 1.0f / J.K;
        for (uint32_t k = 0; k < nc; ++k) {
          T* t = smem + k * DW_TILE_WORDS;
          for (uint32_t e = tid; e < DW_ROWS * DW_COLS; e += DW_THREADS) {
            const uint32_t r = e / DW_COLS, c = e - r * DW_COLS;
            t[r * DW_PITCH + c] = (T)__fmul_rn((float)t[r * DW_PITCH + c], (c & 1) ? Kinv : K);
          }
        }
        __syncthreads();
      }
      for (int s = 0; s < NS; ++s) {
        const int par = s & 1;
        int cfirst = s + 1; if ((cfirst & 1) != par) ++cfirst;
        int clast = DW_COLS - 2 - s; if ((clast & 1) != par) --clast;
        const int ncols = (clast - cfirst) / 2 + 1;
        const int count = DW_ROWS * ncols;
        for (uint32_t k = 0; k < nc; ++k) {
          T* t = smem + k * DW_TILE_WORDS;
          for (int e = (int)tid; e < count; e += DW_THREADS) {
            const int r = e / ncols, j = e - r * ncols;
            const int c = cfirst + 2 * j;
            t[r * DW_PITCH + c] = unlift(t[r * DW_PITCH + c], t[r * DW_PITCH + c - 1], t[r * DW_PITCH + c + 1], s);
          }
        }
        __syncthreads();
      }
    } else if (x0 & 1) {   // single odd column: high-pass sample / 2
      for (uint32_t k = 0; k < nc; ++k) {
        T* t = smem + k * DW_TILE_WORDS;
        for (uint32_t e = tid; e < DW_ROWS * DW_COLS; e += DW_THREADS) {
          const uint32_t r = e / DW_COLS, c = e - r * DW_COLS;
          t[r * DW_PITCH + c] = REV ? (T)((I)t[r * DW_PITCH + c] >> 1) : (T)__fmul_rn((float)t[r * DW_PITCH + c], 0.5f);
        }
      }
      __syncthreads();
    }
  }
  // ---- vertical synthesis on the columns this tile outputs
  if (J.vsplit) {
    if (J.h > 1) {
      if (!REV) {   // even rows * K, odd rows * 1/K (ojph_resolution.cpp:855-872)
        const float K = J.K, Kinv = 1.0f / J.K;
        for (uint32_t k = 0; k < nc; ++k) {
          T* t = smem + k * DW_TILE_WORDS;
          for (uint32_t e = tid; e < DW_ROWS * DW_TW; e += DW_THREADS) {
            const uint32_t r = e / DW_TW, c = DW_H + (e - r * DW_TW);
            t[r * DW_PITCH + c] = (T)__fmul_rn((float)t[r * DW_PITCH + c], (r & 1) ? Kinv : K);
          }
        }
        __syncthreads();
      }
      for (int s = 0; s < NS; ++s) {
        const int par = s & 1;
        int rfirst = s + 1; if ((rfirst & 1) != par) ++rfirst;
        int rlast = DW_ROWS - 2 - s; if ((rlast & 1) != par) --rlast;
        const int count = ((rlast - rfirst) / 2 + 1) * DW_TW;
        for (uint32_t k = 0; k < nc; ++k) {
          T* t = smem + k * DW_TILE_WORDS;
          for (int e = (int)tid; e < count; e += DW_THREADS) {
            const int rr = e / DW_TW, c = DW_H + (e - rr * DW_TW);
            const int r = rfirst + 2 * rr;
            t[r * DW_PITCH + c] = unlift(t[r * DW_PITCH + c], t[(r - 1) * DW_PITCH + c], t[(r + 1) * DW_PITCH + c], s);
          }
        }
        __syncthreads();
      }
    } else if (y0 & 1) {   // single odd row: / 2 (ojph_resolution.cpp:814-827, :918-920)
      for (uint32_t k = 0; k < nc; ++k) {
        T* t = smem + k * DW_TILE_WORDS;
        for (uint32_t e = tid; e < DW_ROWS * DW_COLS; e += DW_THREADS) {
          const uint32_t r = e / DW_COLS, c = e - r * DW_COLS;
          t[r * DW_PITCH + c] = REV ? (T)((I)t[r * DW_PITCH + c] >> 1) : (T)__fmul_rn((float)t[r * DW_PITCH + c], 0.5f);
        }
      }
      __syncthreads();
    }
  }

  // ---- store
  for (uint32_t e = tid; e < DW_TH * DW_TW; e += DW_THREADS) {
    const uint32_t rr = e / DW_TW, cc = e - rr * DW_TW;
    const int r = DW_H + (int)rr, c = DW_H + (int)cc;
    const int u = U0 + (int)cc, v = V0 + (int)rr;
    if (u < x0 || u >= x1 || v < y0 || v >= y1) continue;
    if (!J.first) {
      reinterpret_cast<T*>(coef)[J.full_off[0] + (size_t)(v - y0) * J.full_stride[0] + (size_t)(u - x0)] =
        smem[r * DW_PITCH + c];
      continue;
    }
    int out[3];
    if (REV) {
      I a[3];
      for (uint32_t k = 0; k < nc; ++k) a[k] = (I)smem[k * DW_TILE_WORDS + r * DW_PITCH + c];
      if (nc == 3) {
        I yy = a[0], cb = a[1], cr = a[2];
        I gg = yy - ((cb + cr) >> 2);
        a[0] = cr + gg; a[1] = gg; a[2] = cb + gg;
      }
      if (WIDE && J.nlt_mask) {           // rev_convert_nlt_type3 on 64-bit lines: the map, then the cast to si32
        const I bias = ((I)1 << (J.bit_depth - 1)) + 1;
        for (uint32_t k = 0; k < nc; ++k) {
          if ((J.nlt_mask >> k) & 1u) out[k] = (int)(a[k] >= 0 ? a[k] : -a[k] - bias);
          else out[k] = (int)(a[k] + (J.is_signed ? (I)0 : ((I)1 << (J.bit_depth - 1))));
        }
      } else {
        const I shift = J.is_signed ? (I)0 : ((I)1 << (J.bit_depth - 1));
        for (uint32_t k = 0; k < nc; ++k) out[k] = (int)(a[k] + shift);
      }
    } else {
      float f[3];
      for (uint32_t k = 0; k < nc; ++k) f[k] = (float)smem[k * DW_TILE_WORDS + r * DW_PITCH + c];
      if (nc == 3) {
        float yy = f[0], cb = f[1], cr = f[2];
        f[1] = __fsub_rn(__fsub_rn(yy, __fmul_rn(ICT_GAMMA_CR2G, cr)), __fmul_rn(ICT_GAMMA_CB2G, cb));
        f[0] = __fadd_rn(yy, __fmul_rn(ICT_GAMMA_CR2R, cr));
        f[2] = __fadd_rn(yy, __fmul_rn(ICT_GAMMA_CB2B, cb));
      }
      // irv_convert_to_integer (ojph_colour.cpp:317-360): round, clamp to the B-bit range
      const int B = (int)J.bit_depth;
      const float mul = (float)(1ull << B);
      const int lo = -(1 << (B - 1)), hi = (1 << (B - 1)) - 1;
      const float flo = (float)lo, fhi = -(float)lo;
      const int half = J.is_signed ? 0 : (1 << (B - 1));
      for (uint32_t k = 0; k < nc; ++k) {
        float t = __fmul_rn(f[k], mul);
        int q = round_haz(t);
        q = t >= flo ? q : lo;
        q = t < fhi ? q : hi;
        out[k] = q + half;
      }
    }
    if (J.nlt_mask && !WIDE) {
      const int bias = (1 << (J.bit_depth - 1)) + 1;
      for (uint32_t k = 0; k < nc; ++k) if ((J.nlt_mask >> k) & 1u) out[k] = nlt_type3(out[k], bias);
    }
    for (uint32_t k = 0; k < nc; ++k)
      store_sample(sv[k].org + (size_t)(v - y0) * sv[k].pitch + (size_t)(u - x0) * sv[k].step, J.src_type, out[k],
                   (int)((1u << (J.bit_depth & 31u)) - 1u));
  }
}

} // namespace

void launch_dwt_inv(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                    uint32_t max_ncomp, const ImgComp* img, uint32_t* coef, cudaStream_t st, bool wide)
{
  if (total_ctas == 0) return;
  size_t smem = (size_t)max_ncomp * DW_TILE_WORDS * (wide ? 8 : 4);
  if (reversible && wide) {
    auto k = dwt_inv_kernel<true, true>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    OJB_LAUNCH(k, dim3(total_ctas), dim3(DW_THREADS), smem, st, jobs, njobs, img, coef);
  } else if (reversible) {
    auto k = dwt_inv_kernel<true, false>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    OJB_LAUNCH(k, dim3(total_ctas), dim3(DW_THREADS), smem, st, jobs, njobs, img, coef);
  } else {
    auto k = dwt_inv_kernel<false, false>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    OJB_LAUNCH(k, dim3(total_ctas), dim3(DW_THREADS), smem, st, jobs, njobs, img, coef);
  }
}

} // namespace ojb
