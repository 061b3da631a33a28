// ojb_async.cuh -- cp.async (LDGSTS) wrappers: a thread requests global bytes into shared memory
// without holding registers while they are in flight; cp.async.wait_group orders a thread's own
// copies, so a per-thread private FIFO needs no other synchronisation.
#pragma once
#include "ojb_device.h"
#include <cstring>

namespace ojb {

#ifdef OJB_EMU_BUILD
template <int N> __device__ __forceinline__ void cp_async(void* dst, const void* src) { memcpy(dst, src, N); }
__device__ __forceinline__ void cp_commit() {}
template <int N> __device__ __forceinline__ void cp_wait() {}
__device__ __forceinline__ uint4 ld_stream16(const uint4* p) { return *p; }
#else
template <int N> __device__ __forceinline__ void cp_async(void* dst, const void* src) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" :: "r"(d), "l"(src), "n"(N) : "memory");
}
// A 16-byte load from a per-thread stream of coefficients (the block encoders for the common shape: one thread reads a code-block's
// samples, 49 152 blocks in an 8K frame, each of the two rows of a quad row 16 bytes at a time).  On an L2 miss the .L2::128B hint has L2 fetch the whole
// aligned 128 bytes that the same thread reads next, so DRAM sees 128-byte requests rather than scattered 32-byte
// sectors: the one-thread-per-block encoder of the common shape took 1.37-1.43 ms against 1.48-1.51 ms per 8K frame on an
// H100 80GB HBM3 at 400 W (the 256-byte hint measured 1.42 ms; four frames in one launch were slower, DESIGN §3).
__device__ __forceinline__ uint4 ld_stream16(const uint4* p) {
  uint4 v;
  asm("ld.global.nc.L2::128B.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }
#endif

// ---- named barriers: producer warps `arrive`, consumer warps `sync` (or the reverse); `count` = all threads that
// take part either way (a multiple of 32)
#ifdef OJB_EMU_BUILD
__device__ __forceinline__ void named_bar_sync(unsigned id, unsigned count) { ojb_emu::named_barrier(id, count, true); }
__device__ __forceinline__ void named_bar_arrive(unsigned id, unsigned count) { ojb_emu::named_barrier(id, count, false); }
#else
// (the barrier number is an immediate so that ptxas reserves only the barriers that are used: a register operand
// makes it reserve all 16, and the SM's barrier pool then caps the CTAs per SM)
template <unsigned ID> __device__ __forceinline__ void named_bar_sync_i(unsigned count) { asm volatile("bar.sync %0, %1;" :: "n"(ID), "r"(count) : "memory"); }
template <unsigned ID> __device__ __forceinline__ void named_bar_arrive_i(unsigned count) { asm volatile("bar.arrive %0, %1;" :: "n"(ID), "r"(count) : "memory"); }
__device__ __forceinline__ void named_bar_sync(unsigned id, unsigned count) {
  switch (id) { case 1: named_bar_sync_i<1>(count); break; case 2: named_bar_sync_i<2>(count); break;
                case 3: named_bar_sync_i<3>(count); break; default: named_bar_sync_i<4>(count); break; }
}
__device__ __forceinline__ void named_bar_arrive(unsigned id, unsigned count) {
  switch (id) { case 1: named_bar_arrive_i<1>(count); break; case 2: named_bar_arrive_i<2>(count); break;
                case 3: named_bar_arrive_i<3>(count); break; default: named_bar_arrive_i<4>(count); break; }
}
#endif

} // namespace ojb
