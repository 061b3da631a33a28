// assemble.cu -- codestream assembly on the device.
//
// After the block encoder has run, every code-block sits in its own slot as two pieces
// (MagSgn+MEL at the slot start, VLC at the slot end).  The host computes, from the per-block
// lengths, the packet headers (tag trees, ojb_layout.cpp) and the final byte offset of every
// block; these kernels then place block bytes and header bytes at their final positions so a
// single device->host copy delivers the finished codestream.  This replaces the reference's
// precinct::write / tile::flush memcpy chain (src/core/codestream/ojph_precinct.cpp:281-324,
// ojph_tile.cpp:584-772).
#include "ojb_device.h"
#include "ojb_kernels.h"

namespace ojb {

#define ASM_CHUNK 4096u

namespace {

// warp-cooperative byte copy: 16-byte stores once the destination is aligned, the source read as
// aligned words and funnel-shifted into place (source and destination alignments are independent)
__device__ __forceinline__ void warp_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src,
                                          uint32_t n, uint32_t lane) {
  uint32_t head = (uint32_t)((16 - ((size_t)dst & 15)) & 15);
  if (head > n) head = n;
  if (lane < head) dst[lane] = src[lane];
  dst += head; src += head; n -= head;
  const uint32_t n16 = n >> 4;
  const uint32_t sh = (uint32_t)((size_t)src & 3) * 8;
  const uint32_t* s4 = reinterpret_cast<const uint32_t*>((size_t)src & ~(size_t)3);
  uint4* d16 = reinterpret_cast<uint4*>(dst);
  #pragma unroll 2
  for (uint32_t i = lane; i < n16; i += 32) {
    const uint32_t* p = s4 + 4 * (size_t)i;
    uint32_t w0 = p[0], w1 = p[1], w2 = p[2], w3 = p[3];
    if (sh) {
      const uint32_t w4 = p[4];
      w0 = __funnelshift_r(w0, w1, sh); w1 = __funnelshift_r(w1, w2, sh);
      w2 = __funnelshift_r(w2, w3, sh); w3 = __funnelshift_r(w3, w4, sh);
    }
    d16[i] = make_uint4(w0, w1, w2, w3);
  }
  const uint32_t done = n16 << 4, tail = n - done;
  if (lane < tail) dst[done + lane] = src[done + lane];
}

__global__ void __launch_bounds__(128)
gather_blocks_kernel(const EncBlock* __restrict__ blocks, const EncResult* __restrict__ results,
                     const uint64_t* __restrict__ dst_off, uint32_t nblocks,
                     const uint8_t* __restrict__ slots, uint8_t* __restrict__ out)
{
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= nblocks) return;
  const EncResult r = results[warp];
  if (r.len_head + r.len_tail == 0) return;
  const EncBlock b = blocks[warp];
  if (dst_off[warp] == ~0ull) return;                  // the codestream does not fit its buffer (hdr_layout_kernel)
  uint8_t* d = out + dst_off[warp];
  const uint8_t* slot = slots + b.slot_off;
  warp_copy(d, slot, r.len_head, lane);
  warp_copy(d + r.len_head, slot + b.slot_cap - r.len_tail, r.len_tail, lane);
}

// ---- row regions (ojb_shard.cpp): code-block bytes change ranks between the block coder and the packet headers ----
// where each block's bytes start when the blocks are packed back to back (head piece, then tail piece) in block order:
// the exclusive prefix sum of len_head + len_tail, one CTA; total[0] = the sum.  gather_blocks_kernel with these
// offsets is the packer.
#define BO_THREADS 1024
__global__ void __launch_bounds__(BO_THREADS)
block_offsets_kernel(const EncResult* __restrict__ results, uint32_t n, uint64_t* __restrict__ off, uint64_t* __restrict__ total)
{
  __shared__ unsigned long long ssum[BO_THREADS];
  const uint32_t tid = threadIdx.x, per = (n + BO_THREADS - 1) / BO_THREADS;
  const uint32_t b0 = min(n, tid * per), b1 = min(n, b0 + per);
  unsigned long long sum = 0;
  for (uint32_t b = b0; b < b1; ++b) sum += (unsigned long long)results[b].len_head + results[b].len_tail;
  ssum[tid] = sum;
  __syncthreads();
  for (uint32_t d = 1; d < BO_THREADS; d <<= 1) {
    const unsigned long long t = tid >= d ? ssum[tid - d] : 0;
    __syncthreads();
    ssum[tid] += t;
    __syncthreads();
  }
  unsigned long long run = ssum[tid] - sum;
  for (uint32_t b = b0; b < b1; ++b) { off[b] = run; run += (unsigned long long)results[b].len_head + results[b].len_tail; }
  if (tid == BO_THREADS - 1) total[0] = ssum[tid];
}

// the writer's side: the blocks `rank` coded go from its packed bytes into their slots (as if coded here) and their
// lengths into the writer's result array; a warp per block
__global__ void __launch_bounds__(128)
scatter_blocks_kernel(const EncBlock* __restrict__ blocks, const uint8_t* __restrict__ owner, uint32_t rank,
                      const EncResult* __restrict__ results_in, const uint64_t* __restrict__ off, uint32_t nblocks,
                      const uint8_t* __restrict__ packed, uint8_t* __restrict__ slots, EncResult* __restrict__ results_out)
{
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= nblocks || owner[warp] != rank) return;
  const EncResult r = results_in[warp];
  if (lane == 0) results_out[warp] = r;
  if (r.len_head + r.len_tail == 0) return;
  const EncBlock b = blocks[warp];
  if (r.len_head + r.len_tail > b.slot_cap) return;        // cannot happen with a sane peer; never write outside the slot
  const uint8_t* src = packed + off[warp];
  uint8_t* slot = slots + b.slot_off;
  warp_copy(slot, src, r.len_head, lane);
  warp_copy(slot + b.slot_cap - r.len_tail, src + r.len_head, r.len_tail, lane);
}

__global__ void __launch_bounds__(128)
assemble_kernel(const CopyPiece* __restrict__ pieces, uint32_t npieces, const uint8_t* __restrict__ slots,
                const uint8_t* __restrict__ headers, uint8_t* __restrict__ out)
{
  // blockIdx.y walks a long piece in ASM_CHUNK-byte chunks so that a few large header runs do not
  // serialise on a handful of warps
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= npieces) return;
  const CopyPiece p = pieces[warp];
  const uint64_t c0 = (uint64_t)blockIdx.y * ASM_CHUNK;
  if (c0 >= p.len) return;
  const uint32_t n = (uint32_t)min((uint64_t)ASM_CHUNK, (uint64_t)p.len - c0);
  const uint8_t* src = (p.src_sel ? headers : slots) + p.src_off + c0;
  warp_copy(out + p.dst_off + c0, src, n, lane);
}

// small control-plane transfers (block lengths, offsets, header bytes, block descriptors) between
// pinned host memory and the device, done by the SMs over the mapped host pointer: they never queue
// on a copy engine behind another frame's image-sized transfer
__global__ void __launch_bounds__(256)
ctrl_copy_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, size_t bytes)
{
  const size_t n16 = bytes >> 4;
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (size_t i = tid; i < n16; i += nth) d[i] = s[i];
  for (size_t i = (n16 << 4) + tid; i < bytes; i += nth) dst[i] = src[i];
}

__global__ void __launch_bounds__(256)
dec_merge_kernel(DecBlock* __restrict__ blocks, const DecBlock* __restrict__ proto, const DecDyn* __restrict__ dyn, uint32_t n)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  DecBlock d = proto[b];
  const DecDyn y = dyn[b];
  d.data_off = y.data_off; d.len1 = y.len1; d.len2 = y.len2;
  d.num_passes = y.num_passes; d.missing_msbs = y.missing_msbs; d.flags = y.flags;
  if (y.skip) { d.w = 0; d.h = 0; }
  blocks[b] = d;
}

// the transcoder's block array of one frame: block b as the encoder configured it, started at the lowest plane q_b the
// input codes it down to (the decoder's gates: SigProp / MagRef passes count only with bytes and with p > 1); a block the
// input leaves out gets p = 31, which leaves it zero candidates.  map (null: the identity) names the input's block
// behind each of the encoder's when the output drops resolution levels
__global__ void __launch_bounds__(256)
transcode_blocks_kernel(const EncBlock* __restrict__ geom, const DecBlock* __restrict__ dec, const uint32_t* __restrict__ map,
                        uint32_t n, EncBlock* __restrict__ out)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  EncBlock e = geom[b];
  const DecBlock d = dec[map ? map[b] : b];
  const bool refined = d.num_passes > 1 && d.len2 != 0 && d.missing_msbs < 29;
  if (d.num_passes == 0 || d.len1 == 0) { e.p = 31; e.flags &= (uint16_t)~ENC_CHECK_NEGZERO; }
  else e.p = (uint16_t)((refined ? 29u : 30u) - d.missing_msbs);
  out[b] = e;
}

} // namespace

void launch_dec_merge(DecBlock* blocks, const DecBlock* proto, const DecDyn* dyn, uint32_t nblocks, cudaStream_t st)
{
  if (nblocks == 0) return;
  OJB_LAUNCH(dec_merge_kernel, dim3((nblocks + 255) / 256), dim3(256), 0, st, blocks, proto, dyn, nblocks);
}

void launch_transcode_blocks(const EncBlock* geom, const DecBlock* dec, const uint32_t* map, uint32_t nblocks, EncBlock* out,
                             cudaStream_t st)
{
  if (nblocks == 0) return;
  OJB_LAUNCH(transcode_blocks_kernel, dim3((nblocks + 255) / 256), dim3(256), 0, st, geom, dec, map, nblocks, out);
}

void launch_ctrl_copy(void* dst, const void* src, size_t bytes, cudaStream_t st)
{
  if (bytes == 0) return;
  size_t ctas = (bytes / 16 + 255) / 256;
  if (ctas < 1) ctas = 1;
  if (ctas > 592) ctas = 592;
  OJB_LAUNCH(ctrl_copy_kernel, dim3((unsigned)ctas), dim3(256), 0, st, (uint8_t*)dst, (const uint8_t*)src, bytes);
}

void launch_gather_blocks(const EncBlock* blocks, const EncResult* results, const uint64_t* dst_off,
                          uint32_t nblocks, const uint8_t* slots, uint8_t* out, cudaStream_t st)
{
  if (nblocks == 0) return;
  dim3 grid((nblocks + 3) / 4), block(128);
  OJB_LAUNCH(gather_blocks_kernel, grid, block, 0, st, blocks, results, dst_off, nblocks, slots, out);
}

void launch_block_offsets(const EncResult* results, uint32_t nblocks, uint64_t* off, uint64_t* total, cudaStream_t st)
{
  OJB_LAUNCH(block_offsets_kernel, dim3(1), dim3(BO_THREADS), 0, st, results, nblocks, off, total);
}

void launch_scatter_blocks(const EncBlock* blocks, const uint8_t* owner, uint32_t rank, const EncResult* results_in,
                           const uint64_t* off, uint32_t nblocks, const uint8_t* packed, uint8_t* slots,
                           EncResult* results_out, cudaStream_t st)
{
  if (nblocks == 0) return;
  dim3 grid((nblocks + 3) / 4), block(128);
  OJB_LAUNCH(scatter_blocks_kernel, grid, block, 0, st, blocks, owner, rank, results_in, off, nblocks, packed, slots, results_out);
}

void launch_assemble(const CopyPiece* pieces, uint32_t npieces, uint32_t max_len, const uint8_t* slots,
                     const uint8_t* headers, uint8_t* out, cudaStream_t st)
{
  if (npieces == 0) return;
  dim3 grid((npieces + 3) / 4, (max_len + ASM_CHUNK - 1) / ASM_CHUNK > 0 ? (max_len + ASM_CHUNK - 1) / ASM_CHUNK : 1), block(128);
  OJB_LAUNCH(assemble_kernel, grid, block, 0, st, pieces, npieces, slots, headers, out);
}

} // namespace ojb
