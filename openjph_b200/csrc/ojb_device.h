// ojb_device.h -- descriptors shared by host orchestration and the CUDA kernels, plus the
// launch shim that lets the same .cu sources run under tests/emu (CPU, tests only).
#pragma once
#include <cstdint>
#include <cstddef>

#ifdef OJB_EMU_BUILD
  #include "cuda_emu.h"
  #define OJB_LAUNCH(kernel, grid, block, smem, stream, ...) \
    ojb_emu::launch((grid), (block), (smem), [=]() { kernel(__VA_ARGS__); })
  #define OJB_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(ojb_emu::dyn_smem())
#else
  #include <cuda_runtime.h>
  #include <cstdlib>
  #include <mutex>
  #include <unordered_set>
  // One shared-memory carve-out for every kernel of the library: 50% of the SM's 228 KB unless OJB_SMEM_CARVEOUT
  // (a percentage; -1 = leave the driver's per-kernel choice) says otherwise.  The driver otherwise sizes the
  // carve-out per kernel from its footprint, and an SM is re-partitioned only when idle, so kernels of several
  // frames in flight whose carve-outs differ take turns on an SM instead of sharing it.  0% and 100% leave no room
  // for the coders' rings / no L1.
  namespace ojb {
  inline void prefer_carveout(const void* f) {
    static const int pct = [] { const char* e = getenv("OJB_SMEM_CARVEOUT"); return (e && *e) ? atoi(e) : 50; }();
    if (pct < 0) return;
    static std::mutex m; static std::unordered_set<const void*> done;
    std::lock_guard<std::mutex> g(m);
    if (done.insert(f).second) cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
  }
  }
  #define OJB_LAUNCH(kernel, grid, block, smem, stream, ...) \
    do { ojb::prefer_carveout(reinterpret_cast<const void*>(kernel)); kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__); } while (0)
  #define OJB_DYN_SMEM(type, name) extern __shared__ __align__(16) unsigned char name##_raw[]; \
    type* name = reinterpret_cast<type*>(name##_raw)
#endif

namespace ojb {

// ---- HT block encoder -------------------------------------------------------------------
// One record per code-block; the kernel reads sign-magnitude samples (bit 31 sign, magnitude
// MSB-aligned: |v| << (31 - K_max)), same convention as the reference's code-block buffers
// (ojph_codestream_gen.cpp:59-78, ojph_codeblock.cpp:115-139).
struct EncBlock {
  uint64_t src_off;     // word offset of sample (0,0) in the coefficient arena
  uint64_t slot_off;    // byte offset of the output slot in the slot arena (16-byte aligned)
  uint32_t stride;      // words between rows
  uint32_t slot_cap;    // slot size in bytes (multiple of 16)
  uint16_t w, h;
  uint16_t p;           // 30 - missing_msbs = 31 - K_max
  uint16_t flags;       // bit 0: look for magnitude-overflow words (0x80000000), see ENC_CHECK_NEGZERO
};
// A sample whose magnitude is exactly 2^K_max shifts out of the 31 magnitude bits and is stored as
// 0x80000000: the reference still counts it in its max_val test (ojph_codeblock.cpp:143-147,
// ojph_codestream_gen.cpp:59-78), so a block made only of such samples is coded (3 bytes, nothing
// significant) instead of being skipped.  It happens with zero decompositions and no colour transform
// (K_max = B - 1 + guard for the single band) for the most negative sample value.
#define ENC_CHECK_NEGZERO 1u
// EncBlock::flags bit 1: the block qualifies for ht_encode_split_kernel
#define ENC_FLAG_FAST 2u
inline bool enc_block_is_fast(const EncBlock& e) {
  return e.w >= 4 && e.w <= 64 && (e.w & 3) == 0 && e.h >= 2 && (e.h & 1) == 0 && ((e.src_off | e.stride) & 3u) == 0 &&
         e.p >= 16 && e.p <= 30 && !(e.flags & ENC_CHECK_NEGZERO);
}
// result per block: [0] bytes at slot start (MagSgn + MEL), [1] bytes at slot end (VLC);
// both 0 for a block with no significant sample (not included in the packet).
struct EncResult { uint32_t len_head, len_tail; };

// ---- rate control (rate_ctrl.cu) --------------------------------------------------------
// a candidate length the final encode would refuse (MEL over 192 bytes, slot overflow): never selected
#define RC_LEN_INVALID 0xFFFFFFFFu
// what the rounds that settle the body budget share on the device (one per encoder)
struct RcState {
  long long budget;          // body budget B_r of the current round
  unsigned long long total;  // codestream bytes of the last selection sized
  unsigned long long sum0;   // sum of R_b(0): the body of the unconstrained stream
  unsigned long long body;   // sum of the selected R_b(k_b)
  uint32_t thresh;           // slope key threshold of the last selection
  uint32_t done;             // the last selection sized fits the target
  uint32_t rounds;           // selections made (0: the unconstrained stream fits)
  uint32_t pad;
};
// the search of a quality target (target squared error): a bracket of slope keys, t_pass (a measured selection whose
// exact squared error is within the limit; key 0, the unconstrained selection, until one is measured) and t_fail
// (measured over it; 2^32, every block left out, until one is).  128-bit squared errors as (lo, hi) word pairs.
#define RQ_MAX_COMPS 16
#define RQ_MAX_ROUNDS 64
#define RQ_MODEL_ROUNDS 4          // rounds that may take the model's proposal
#define RQ_BODY_ROUNDS 16          // rounds that may halve the bracket's body gap; later rounds bisect the key range
struct RqRound { unsigned long long key, sse_lo, sse_hi, body; };
struct RqState {
  unsigned long long limit;                      // floor(target * N)
  unsigned long long t_pass, t_fail, body_pass, body_fail;
  unsigned long long sse_pass[2];                // of the selection at t_pass (the one returned)
  unsigned long long comp_pass[RQ_MAX_COMPS][2]; // per component, of the same selection
  unsigned long long comp_cur[RQ_MAX_COMPS][2];  // per component, of the selection this round measures
  unsigned long long key, body;                  // this round's key and body bytes
  unsigned long long body0;                      // body bytes of the unconstrained selection (key 0)
  double c;                                      // correction of the model: propose sum_b D_b <= c * limit
  double model1;                                 // the model's sum_b D_b for the selection of round 1
  uint32_t rounds, done, reached, pass_measured, fail_measured, force_zero, ncomp, pad;
  RqRound round[RQ_MAX_ROUNDS];
};
// the per-block tables of one frame; kc = 1 + the largest K_max: block b's entries are [b * kc, b * kc + K_max_b]
struct RcTables {
  uint32_t kc;
  uint8_t* ncand;            // candidates k < ncand[b] can be non-empty (the block's top magnitude plane; 1 for ENC_CHECK_NEGZERO)
  EncResult* cand;           // R_b(k) = len_head + len_tail (RC_LEN_INVALID: not a candidate)
  double* dist;              // D_b(k), k = 0 .. K_max_b
  const double* weight;      // W_b
  const uint8_t* irv;        // 1: irreversible band (h_0 = 1/2)
  uint8_t* hull_k;           // [b * (kc + 1) + j]: k of hull point j (point 0: excluded, k = K_max)
  uint32_t* hull_key;        // [b * kc + j]: ordered key of segment j (point j -> j + 1), non-increasing in j
  uint32_t* hull_len;        // [b * kc + j]: R at hull point j + 1
  uint8_t* hull_n;           // segments per block
  uint8_t* chosen;           // chosen k per block
  RcState* state;
  const float* delta;        // the decoder's step per block (DecBlock::delta; irreversible bands)
  RqState* q;                // quality target only
};
// the image planes the quality target compares: component c is comp_w[c] x comp_h[c] samples of the sample container
struct RqImage { uint32_t ncomp, sample_type, w[RQ_MAX_COMPS], h[RQ_MAX_COMPS]; };

// ---- HT block decoder -------------------------------------------------------------------
struct DecBlock {
  uint64_t data_off;    // byte offset of the coded bytes in the codestream buffer
  uint64_t dst_off;     // word offset of sample (0,0) in the coefficient arena
  uint64_t scratch_off; // word offset of this block's quad records in the scratch area (blocks with SPP / MRP)
  uint32_t len1, len2;  // cleanup bytes, SPP+MRP bytes
  uint32_t stride;      // words between rows of dst
  uint16_t w, h;
  uint8_t missing_msbs, num_passes, K_max, flags;   // flags bit0: stripe-causal, bit1: irreversible (float output)
  float delta;          // irreversible: step (already / 2^(31-K_max)); reversible: unused
};
// what changes from frame to frame for a block (the rest of DecBlock is geometry, uploaded once per parameter set):
// 16 bytes per block cross PCIe per frame instead of 48
struct DecDyn {
  uint64_t data_off;
  uint16_t len1, len2;
  uint8_t num_passes, missing_msbs, flags, skip;       // skip: the block is not needed at all (w = h = 0)
};
// DecBlock::flags bit 2, set by the host per frame: the block qualifies for ht_decode_split_kernel
#define DEC_FLAG_FAST 4u
inline bool dec_block_is_fast(const DecBlock& d) {
  return d.num_passes == 1 && d.len1 >= 2 && d.w >= 4 && d.w <= 64 && (d.w & 3) == 0 && d.h >= 2 && (d.h & 1) == 0 &&
         ((d.dst_off | d.stride) & 3u) == 0 && d.missing_msbs + 2u <= 16u && d.K_max > d.missing_msbs;
}
enum : uint32_t {       // DecBlock output modes
  DEC_OUT_SIGNMAG = 0,  // raw sign-magnitude (kernel-level parity with ojph_decode_codeblock32)
  DEC_OUT_INT = 1,      // reversible: signed integers (tx_from_cb32 fused)
  DEC_OUT_FLOAT = 2,    // irreversible: float coefficient (tx_from_cb32 fused)
  DEC_OUT_PER_BLOCK = 3,// INT or FLOAT by the block's flags (components may differ: COC)
  DEC_OUT_CODED = 4     // transcoding: the sign-magnitude word with every bit below the lowest coded plane cleared (no
                        // bin centre): the encoder's band-plane format, which the block encoder re-codes bit for bit
};

// ---- DWT --------------------------------------------------------------------------------
enum : uint32_t { SRC_U8 = 0, SRC_U16 = 1, SRC_I32 = 2, SRC_COEF = 3 };

// Where the samples of one image component are: sample (x, y) sits at base + y * pitch + x * col * (sample size).
// The first-level jobs of the DWT kernels reach the image only through an array of these, one per component (a
// per-frame control block in device memory): the codec's own image buffer (tight rows, col = 1) or the caller's
// memory (any pitch, planar or interleaved).  The streaming kernels form offsets from base in 32 bits: every
// component they address spans fewer than 2^32 bytes.
struct ImgComp {
  uint64_t base;        // device address of sample (0, 0)
  uint64_t pitch;       // bytes from one row to the next
  uint32_t col;         // samples from one column to the next
  uint32_t pad;
};

// one analysis (or synthesis) level of one tile-component (or of 3 colour components at once
// for the first level when the colour transform is used)
#define DWT_MAX_STEPS 8        // = the halo of the general kernels' tile (DW_H): one sample per lifting step
struct DwtJob {
  // geometry of the resolution being split
  uint32_t w, h;          // size
  uint32_t x0, y0;        // origin (only parity and band-origin arithmetic matter)
  // source / destination of the full-resolution samples
  uint64_t full_off[3];   // not first: word offset in the arena
  uint32_t full_stride[3];// not first: in samples
  // first: component img_comp[i] of the image (ImgComp), the resolution's origin at column img_x[i], row img_y[i]
  uint32_t img_comp[3], img_x[3], img_y[3];
  // LL output (next level input) -- arena word offsets
  uint64_t ll_off[3];
  uint32_t ll_stride[3];
  // detail bands HL, LH, HH (+ LL as band 0 when this is the last level): sign-magnitude planes
  uint64_t band_off[3][4];
  uint32_t band_stride[3][4];
  uint32_t band_shift[3][4];   // reversible: 31 - K_max
  float band_scale[3][4];      // irreversible: delta_inv (forward) / delta (inverse)
  uint32_t ncomp;         // 1, or 3 when the colour transform is fused (level 1 only)
  uint32_t first;         // 1: full-resolution side is the image (level shift / colour transform)
  uint32_t last;          // 1: LL is a final band (quantise it to band 0), else raw to ll_off
  uint32_t nodwt;         // 1: nothing to lift at this level (zero decomposition levels, or a DFS level without transform): == !(hsplit | vsplit)
  // general (shared-memory tile) kernels only -- the streaming kernels are built for the dyadic 5/3 and 9/7:
  uint32_t hsplit, vsplit;     // the level lifts along x / along y (DFS: a level may split one way only)
  uint32_t nsteps;             // lifting steps of the kernel, SYNTHESIS order: step s acts on samples of parity s & 1
  float step_A[DWT_MAX_STEPS]; // irreversible: x[n] -= A (x[n-1] + x[n+1]) on synthesis, += on analysis
  int step_a[DWT_MAX_STEPS], step_b[DWT_MAX_STEPS]; uint32_t step_e[DWT_MAX_STEPS];   // reversible: (b + a (x[n-1] + x[n+1])) >> e
  float K;                     // irreversible: low-pass / K, high-pass * K after analysis
  uint32_t src_type;      // SRC_* of the image buffer when first
  uint32_t bit_depth;     // for level shift / float conversion when first
  uint32_t is_signed;
  uint32_t nlt_mask;      // bit i: NLT type 3 on (signed) component i of the job: v < 0 -> -v - (2^(B-1) + 1)
  uint32_t tiles_x, tiles_y;   // CTA tiling of this job
  uint32_t chunk_rows;         // streaming kernels: output rows per warp chunk (even)
  uint32_t chunk0;             // streaming kernels: first row chunk of the launch (row-region sharding runs a window of
                               // tiles_y chunks starting here; 0 otherwise)
  uint32_t cta_base;      // first CTA index of this job in the launch
};

// ---- packet headers on the device (pkt_headers.cu) -----------------------------------------------------------------
// static plan, built once per configuration; every "item" is one code-block in header order (packets in stream order,
// inside a packet the bands that have blocks, inside a band the precinct's blocks in raster order)
struct HdrSeg {          // one band of one precinct with code-blocks in it (the loop body of precinct::prepare_precinct)
  uint32_t pkt;          // packet, in stream order
  uint32_t first_item;
  uint32_t w, h, nl;     // the precinct's code-block grid in this band; tag-tree levels = 1 + max(ceil log2 w, ceil log2 h)
  uint32_t block0, nbw;  // block index of item (x, y) = block0 + y * nbw + x
  uint32_t tree_off;     // first node of this segment's trees in the node arrays
};
struct HdrPkt { uint32_t first_seg, nsegs, first_item, nitems, first_group, ngroups, hdr_off /* bytes into the header scratch, x4 */, tp_first; };
struct HdrGroup { uint32_t first_item, n; };       // <= 32 consecutive items of one packet
struct HdrTp { uint32_t first_pkt, npkts, tile, tp_idx, tp_cnt, tlm_off /* byte offset of its Ptlm in the output, or ~0 */; };
struct HdrPlanDev {
  uint32_t nsegs, npkts, nitems, ngroups, ntps, max_hdr_cap;
  const HdrSeg* segs; const HdrPkt* pkts; const HdrGroup* groups; const HdrTp* tps; const uint32_t* item_seg;
  // per frame
  uint8_t *tinc, *tmm; uint32_t* tfi; uint8_t* seg_root;
  uint32_t* ibits; uint16_t* inbits; uint16_t* itab; uint32_t* ilen;
  uint32_t *gcomp, *gbits, *glen, *gstate, *gpos, *gbody;
  uint8_t* istate; uint32_t *ipos, *ibody;
  uint32_t *phdr, *pbody; uint64_t* ppos;
  uint32_t* hscr;        // packet header bytes, zeroed before every frame
  uint64_t* total;       // [0] codestream length, [1] 1 when it exceeds the output capacity (nothing is written then)
  uint64_t* tp_out;      // per tile-part: byte offset of its SOT in the output, Psot
};

// ---- raster layouts ------------------------------------------------------------------------
struct RasterPlanes {        // where the component planes of the image buffer are (bytes / samples)
  uint64_t off[3];
  uint32_t stride[3];
};

} // namespace ojb
