// dequant.cuh -- the decoder's store of one decoded sign-magnitude word (ht_decode.cu), shared with the quality
// target's reconstruction (rate_ctrl.cu), which must write exactly what the decoder writes.
#pragma once
#include "ojb_device.h"

namespace ojb {

// sm: sign in bit 31, magnitude with its bin-centre bit below the last decoded plane.  DEC_OUT_INT: the reversible
// integer (magnitude >> shift, shift = 31 - K_max); DEC_OUT_FLOAT: the irreversible coefficient magnitude * delta, sign
// carried over; DEC_OUT_SIGNMAG: the word itself
__device__ __forceinline__ uint32_t to_output(uint32_t sm, uint32_t mode, uint32_t shift, float delta) {
  if (mode == DEC_OUT_SIGNMAG) return sm;
  if (mode == DEC_OUT_INT) {
    int v = (int)((sm & 0x7FFFFFFFu) >> shift);
    return (uint32_t)((sm & 0x80000000u) ? -v : v);
  }
  float f = __fmul_rn((float)(sm & 0x7FFFFFFFu), delta);
  return __float_as_uint(f) | (sm & 0x80000000u);
}

} // namespace ojb
