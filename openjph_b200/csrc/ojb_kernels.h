// ojb_kernels.h -- host-callable launchers of the CUDA kernels (one translation unit each).
#pragma once
#include "ojb_device.h"

namespace ojb {

// a second stream of the same codec object: the specialised and the general block-coder kernels of one frame work
// on disjoint blocks and each lasts as long as its longest block's serial chain, so they run side by side
// (fork after the producer of their input, join before the consumer of their output)
struct SideStream { cudaStream_t st = nullptr; cudaEvent_t fork = nullptr, join = nullptr; };

// HT cleanup encoder, one warp per code-block (ht_encode.cu)
// tables: uint16 enc_vlc[2][2048] followed by enc_uvlc[33] in device memory
void launch_ht_encode(const EncBlock* blocks, uint32_t nblocks, const uint32_t* coef, uint8_t* slots,
                      EncResult* results, const uint16_t* tables, uint32_t* status, cudaStream_t st);

// the same encoder with one THREAD per code-block (ht_encode_serial.cu); max_width = widest block; nfast of the
// blocks carry ENC_FLAG_FAST (see enc_block_is_fast) and go through the specialised kernel
void launch_ht_encode_serial(const EncBlock* blocks, uint32_t nblocks, uint32_t nfast, uint32_t max_width, const uint32_t* coef,
                             uint8_t* slots, EncResult* results, const uint16_t* tables, uint32_t* status,
                             cudaStream_t st, bool wide = false, const SideStream* side = nullptr);

// HT decoder (ht_decode.cu): one THREAD per code-block for the whole cleanup pass (+ SPP + MRP, + a zero-fill
// kernel); nfast of the blocks carry DEC_FLAG_FAST (see dec_block_is_fast) and go through the specialised kernel.
// scratch: the quad records of blocks with refinement passes, at DecBlock::scratch_off.
// tables: uint16 dec_vlc[2][1024], dec_uvlc0[320], dec_uvlc1[256]
void launch_ht_decode_serial(const DecBlock* blocks, uint32_t nblocks, uint32_t nfast, uint32_t max_width, const uint8_t* codestream,
                             uint32_t* coef, uint32_t* scratch, const uint16_t* tables, uint32_t out_mode,
                             bool cleanup_only, uint32_t* block_status, cudaStream_t st, const SideStream* side = nullptr);

// per-frame block records: blocks[b] = proto[b] with the frame's fields (dyn) applied.
// dyn may be mapped pinned host memory (read by the SMs, like launch_ctrl_copy)
void launch_dec_merge(DecBlock* blocks, const DecBlock* proto, const DecDyn* dyn, uint32_t nblocks, cudaStream_t st);
// transcoding: out[b] = geom[b] (the encoder's static block array) with p = q_b, the lowest plane the merged decoder
// record dec[map[b]] codes (31: the block is left out); map null: the identity
void launch_transcode_blocks(const EncBlock* geom, const DecBlock* dec, const uint32_t* map, uint32_t nblocks, EncBlock* out,
                             cudaStream_t st);

// 64-bit samples (precision beyond 32 bits): cleanup pass only, output int64 (or the raw sign-magnitude words)
void launch_ht_decode_wide(const DecBlock* blocks, uint32_t nblocks, uint32_t max_width, const uint8_t* codestream,
                           uint32_t* coef, const uint16_t* tables, bool signmag, uint32_t* block_status, cudaStream_t st);

// forward / inverse DWT levels (dwt_fwd.cu / dwt_inv.cu).  jobs live in device memory; the first level reaches the
// image through img (device memory, one ImgComp per component)
// wide: 64-bit samples and sign-magnitude words (reversible, precision > 32 bits); offsets and strides count elements
void launch_dwt_fwd(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                    uint32_t max_ncomp, const ImgComp* img, uint32_t* coef, cudaStream_t st, bool wide = false);
void launch_dwt_inv(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                    uint32_t max_ncomp, const ImgComp* img, uint32_t* coef, cudaStream_t st, bool wide = false);
// register-streaming fast path (dwt_stream.cu) for resolutions of at least 2x2.  interleaved: the first three
// components of the image img describes sit next to each other (3 or 4 samples per pixel: the colour-transform jobs
// take the ILV variant)
void dwt_stream_tiling(uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, bool reversible, bool forward,
                       uint32_t& strips, uint32_t& chunks, uint32_t& chunk_rows, uint32_t& ctas);
void launch_dwt_fwd_stream(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                           uint32_t ncomp, bool first, uint32_t src_type, const ImgComp* img, bool interleaved,
                           uint32_t* coef, cudaStream_t st);
void launch_dwt_inv_stream(const DwtJob* jobs, uint32_t njobs, uint32_t total_ctas, bool reversible,
                           uint32_t ncomp, bool first, uint32_t src_type, const ImgComp* img, bool interleaved, uint32_t* coef, cudaStream_t st);
// CTA tiling of a w x h resolution at origin (x0,y0): number of tiles across / down
void dwt_tiling(uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, uint32_t& tx, uint32_t& ty);

// codestream assembly (assemble.cu): copy pieces (block heads/tails, header bytes) to their
// final offsets
struct CopyPiece { uint64_t src_off; uint64_t dst_off; uint32_t len; uint32_t src_sel; };  // src_sel 0: slots, 1: headers
void launch_assemble(const CopyPiece* pieces, uint32_t npieces, uint32_t max_len, const uint8_t* slots,
                     const uint8_t* headers, uint8_t* out, cudaStream_t st);
// small host<->device control transfers done by a kernel over mapped pinned memory (both pointers
// 16-byte aligned)
void launch_ctrl_copy(void* dst, const void* src, size_t bytes, cudaStream_t st);
// interleaved big-endian pixels (.pgm / .ppm payload) <-> the component planes of the image buffer
void launch_raster_unpack(const void* src, void* image, const RasterPlanes& pl, uint32_t ncomp, uint32_t bytes_per_sample,
                          uint32_t width, uint32_t height, cudaStream_t st);
// .dpx image data: 10-bit packed RGB words or 16-bit RGB samples, either byte order
void launch_raster_unpack_dpx(const void* src, void* image, const RasterPlanes& pl, uint32_t bit_depth, bool swap,
                              uint32_t width, uint32_t height, cudaStream_t st);
void launch_raster_pack(void* dst, const void* image, const RasterPlanes& pl, uint32_t ncomp, uint32_t bytes_per_sample,
                        uint32_t width, uint32_t height, cudaStream_t st);
// packet headers, SOT / TLM / EOC and the destination of every block body, all on the device (pkt_headers.cu);
// `out` must already hold the fixed bytes (main header, TLM with blank lengths); dst[] feeds launch_gather_blocks
void launch_packet_headers(const HdrPlanDev& plan, const EncBlock* blocks, const EncResult* results, uint32_t mmsb_base,
                           uint64_t fixed_len, uint64_t cap, bool write_eoc, uint8_t* out, uint64_t* dst, cudaStream_t st);
uint32_t packet_header_launches(const HdrPlanDev& plan);
// the codestream length alone (plan.total[0]): the sizing step of rate control
void launch_packet_header_total(const HdrPlanDev& plan, const EncBlock* blocks, const EncResult* results, uint32_t mmsb_base,
                                uint64_t fixed_len, bool write_eoc, cudaStream_t st);
uint32_t packet_header_total_launches(const HdrPlanDev& plan);

// rate control (rate_ctrl.cu, and the count-only encoder of ht_encode_serial.cu)
void launch_ht_encode_lengths(const EncBlock* blocks, uint32_t nblocks, uint32_t kc, const uint8_t* ncand, uint32_t max_width,
                              const uint32_t* coef, EncResult* lengths, const uint16_t* tables, cudaStream_t st);
void launch_rc_prepare(const EncBlock* blocks, uint32_t nblocks, const uint32_t* coef, const RcTables& t, cudaStream_t st);
void launch_rc_hull(const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res, const RcTables& t, cudaStream_t st);
void launch_rc_round(const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res, const RcTables& t, cudaStream_t st);
void launch_rc_check(const RcTables& t, const uint64_t* total, uint64_t target, uint64_t min_bytes, bool first, cudaStream_t st);
double colour_weight(bool ict, uint32_t c);
// quality target (rate_ctrl.cu): the bracket; one round's selection and its reconstruction into the arena `recon`
// (the decoder's inverse DWT launches then synthesise it); the round's exact squared error and the bracket update;
// the final selection at t_pass
void launch_rq_init(const RcTables& t, uint64_t limit, uint32_t ncomp, bool lossless0, cudaStream_t st);
// (geom: the static block array, whose p = 31 - K_max is the decoder's integer shift; blocks: where each block starts)
void launch_rq_select(const EncBlock* geom, const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res,
                      const uint32_t* coef, uint32_t* recon, const RcTables& t, cudaStream_t st);
void launch_rq_measure(const ImgComp* decoded, const ImgComp* source, const RqImage& im, const RcTables& t, cudaStream_t st);
void launch_rq_final(const EncBlock* blocks, uint32_t nblocks, EncBlock* work, EncResult* res, const RcTables& t, cudaStream_t st);
// block pieces computed on the device from per-block results + destination offsets
void launch_gather_blocks(const EncBlock* blocks, const EncResult* results, const uint64_t* dst_off,
                          uint32_t nblocks, const uint8_t* slots, uint8_t* out, cudaStream_t st);

// row regions (ojb_shard.cpp).  launch_block_offsets: off[b] = where block b's bytes start when all blocks are packed
// back to back in block order (head piece, then tail piece), total[0] = their sum -- launch_gather_blocks with these
// offsets packs.  launch_scatter_blocks: on the writer, the blocks owned by `rank` go from that rank's packed bytes
// into their slots and their lengths into the writer's result array.
void launch_block_offsets(const EncResult* results, uint32_t nblocks, uint64_t* off, uint64_t* total, cudaStream_t st);
void launch_scatter_blocks(const EncBlock* blocks, const uint8_t* owner, uint32_t rank, const EncResult* results_in,
                           const uint64_t* off, uint32_t nblocks, const uint8_t* packed, uint8_t* slots,
                           EncResult* results_out, cudaStream_t st);

} // namespace ojb
