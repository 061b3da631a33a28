/* ojph_b200.h -- C ABI of libojph_b200.so: the H100-native HTJ2K hot path behind OpenJPH's
 * codestream interface.  Plain pointers and sizes only; every function returns 0 on success or
 * a negative status (the message is available from ojb_last_error(), formatted like the
 * reference's "ojph error 0x%08X" -- src/core/others/ojph_message.cpp:156-171).
 *
 * Each entry point names the reference interface it stands in for (paths are relative to the
 * OpenJPH tree, v0.31.0).  INTEGRATION.md shows the binding a maintainer would add on the
 * reference side.
 */
#ifndef OJPH_B200_H
#define OJPH_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* Codestream parameters: the union of what ojph_compress sets through param_siz / param_cod /
 * param_qcd (src/core/openjph/ojph_params.h; setters used at
 * src/apps/ojph_compress/ojph_compress.cpp:678-709). */
typedef struct ojb_params {
  uint32_t width, height;          /* image extent  (param_siz::set_image_extent) */
  uint32_t off_x, off_y;           /* image offset  (set_image_offset) */
  uint32_t tile_w, tile_h;         /* tile size; 0,0 = one tile (set_tile_size) */
  uint32_t tile_off_x, tile_off_y; /* tile offset   (set_tile_offset) */
  uint32_t num_comps;              /* set_num_components, <= 16 through this struct */
  uint32_t bit_depth[16];          /* set_component(c, downsampling, bit_depth, is_signed) */
  uint32_t is_signed[16];
  uint32_t dx[16], dy[16];
  uint32_t num_decomps;            /* param_cod::set_num_decomposition */
  uint32_t block_w, block_h;       /* set_block_dims */
  uint32_t num_precincts;          /* set_precinct_size; 0 = default (2^15) */
  uint32_t precinct_w[33], precinct_h[33];
  uint32_t reversible;             /* set_reversible */
  uint32_t color_transform;        /* set_color_transform */
  uint32_t prog_order;             /* 0 LRCP 1 RLCP 2 RPCL 3 PCRL 4 CPRL (set_progression_order) */
  float    qstep;                  /* param_qcd::set_irrev_quant; <= 0 = library default */
  uint32_t qfactor;                /* param_qcd::set_qfactor; 0 = unset */
  uint32_t tlm;                    /* codestream::request_tlm_marker */
  uint32_t tilepart_div;           /* codestream::set_tilepart_divisions: bit0 resolutions, bit1 components */
  int32_t  planar;                 /* codestream::set_planar; -1 = not called */
  /* per-component coding styles (COC): param_cod::set_reversible / set_num_decomposition /
   * set_block_dims with a component index (ojph_params.cpp:255-281).  As in the reference a component's
   * COC starts from the library defaults (5 levels, 64x64, irreversible), not from the COD values, so all
   * four fields are read when coc_present[c] != 0. */
  uint32_t coc_present[16];
  uint32_t coc_reversible[16];
  uint32_t coc_num_decomps[16];
  uint32_t coc_block_w[16], coc_block_h[16];
  uint32_t coc_num_precincts[16];             /* param_cod::set_precinct_size(comp_idx, n, sizes); 0 = default */
  uint32_t coc_precinct_w[16][33], coc_precinct_h[16][33];
  /* non-linearity point transform (NLT marker; param_nlt::set_nonlinear_transform(comp, type),
   * ojph_params.cpp:441, :2176): 0 = not called, else 1 + type (1: type 0 "none", 4: type 3 = two's
   * complement <-> sign-magnitude mapping of signed samples, the only one the reference implements).
   * nlt_all is the ALL_COMPS (65535) entry; nlt_seq[c] orders the per-component calls (marker order). */
  uint32_t nlt_all;
  uint32_t nlt_comp[16];
  uint32_t nlt_seq[16];
  /* codestream::set_profile (ojph_codestream_local.cpp:1124-1133): 0 none, 1 "IMF", 2 "BROADCAST".  A profile
   * checks the parameters (:292-535) and forces TLM + tile-part division by components. */
  uint32_t profile;
  /* per-component quantisation (QCC): param_qcd::set_irrev_quant(comp, delta) and set_qfactor(comp, ctype,
   * qfactor) (ojph_params.cpp:2011-2035).  qcc_calls[c] bit 0: the delta call was made, bit 1: the qfactor
   * call; *_seq give the order of ALL quantisation calls (the global qstep / qfactor above count as made
   * first): the reference's per-component delta call lands on the component's QCC only if one already exists
   * (made by an earlier per-component qfactor call) and on the global QCD otherwise, so order matters. */
  uint32_t qcc_calls[16];
  float    qcc_qstep[16];
  uint32_t qcc_qstep_seq[16];
  uint32_t qcc_qfactor[16], qcc_ctype[16];     /* ctype: 0 Y, 1 Cb, 2 Cr */
  uint32_t qcc_qfactor_seq[16];
  /* Part 2 wavelet structures.  The reference READS DFS and ATK marker segments (param_dfs::read,
   * ojph_params.cpp:2596; param_atk::read, :2770; resolution::finalize_alloc, ojph_resolution.cpp:264-396) and has
   * no writer for them; the decoder here reads what it reads, and the encoder fields below are this library's
   * own addition so that such streams can be produced (and checked against the reference's decoder):
   *   dfs_type[i], i < dfs_num_levels: how decomposition level i + 1 (1 = finest) splits -- 1 both ways,
   *     2 horizontally only, 3 vertically only; levels past the list repeat the last entry; 0 levels = dyadic.
   *   atk_*: a whole-sample symmetric lifting kernel with one tap pair per step, steps in SYNTHESIS order (step 0
   *     acts on the even samples): irreversible x[n] -= A (x[n-1] + x[n+1]) with scaling K, or reversible
   *     x[n] -= (b + a (x[n-1] + x[n+1])) >> e.  atk_num_steps = 0 keeps the COD's 5/3 or 9/7; at most 8 steps
   *     (a longer kernel in a codestream is refused, 0x000B0025). */
  uint32_t dfs_num_levels;
  uint32_t dfs_type[32];
  uint32_t atk_num_steps;
  uint32_t atk_reversible;
  float    atk_K;
  float    atk_A[8];
  int32_t  atk_a[8], atk_b[8];
  uint32_t atk_e[8];
} ojb_params;

typedef struct ojb_frame_info {
  uint32_t width, height, off_x, off_y, num_comps;
  uint32_t bit_depth[16], is_signed[16], dx[16], dy[16], comp_w[16], comp_h[16];
  uint32_t num_decomps, reversible, color_transform, num_tiles;
  uint32_t nlt_type[16];           /* param_nlt::get_nonlinear_transform: 0 none, 3 type 3 */
} ojb_frame_info;

typedef struct ojb_comment {       /* ojph::comment_exchange (ojph_params.h): one extra COM segment */
  const void* data;
  uint16_t len;
  uint16_t rcom;                   /* 0 binary, 1 Latin text */
} ojb_comment;

/* sample container of frame buffers */
enum { OJB_U8 = 0, OJB_U16 = 1, OJB_I32 = 2 };

typedef struct ojb_encoder ojb_encoder;
typedef struct ojb_decoder ojb_decoder;

const char* ojb_last_error(void);
const char* ojb_version(void);
int ojb_device_count(void);
int ojb_set_device(int device);
void ojb_params_default(ojb_params* p);      /* the reference's defaults: 5 levels, 64x64, RPCL */

/* pinned host memory for frame / codestream buffers (optional; any host pointer works) */
void* ojb_host_alloc(uint64_t bytes);
void ojb_host_free(void* p);

/* ---- encode: ojph::codestream write side (src/core/openjph/ojph_codestream.h:88-383) ---- */
ojb_encoder* ojb_enc_create(void);                       /* codestream::codestream() */
void ojb_enc_destroy(ojb_encoder* e);                    /* ~codestream / close() */
/* access_siz/cod/qcd setters + write_headers(): validates, builds geometry and device arenas */
int ojb_enc_configure(ojb_encoder* e, const ojb_params* p, uint32_t sample_type);
/* the comments argument of write_headers(file, comments, num_comments) (ojph_codestream_local.cpp:688-706):
 * extra COM segments after the library's own; copied, applies to the configure calls that follow */
int ojb_enc_set_comments(ojb_encoder* e, const ojb_comment* comments, uint32_t num_comments);
/* codestream::exchange(line_buf*, ui32& next_comp): first call with line == NULL; returns the
 * line to fill next (library owned, si32 samples), NULL after the last line */
int32_t* ojb_enc_exchange(ojb_encoder* e, int32_t* line, uint32_t* next_comp);
/* codestream::flush(): encodes the exchanged frame on the GPU into out */
int ojb_enc_flush(ojb_encoder* e, uint8_t* out, uint64_t out_cap, uint64_t* out_len);
/* frame-at-once fast path: component planes in the configured container, strides in samples
 * (NULL = tight); host pointers (pinned or pageable) */
int ojb_enc_encode_frame(ojb_encoder* e, const void* const* planes, const uint32_t* strides,
                         uint8_t* out, uint64_t out_cap, uint64_t* out_len);
/* File sample layouts of the reference's apps (src/apps/others/ojph_img_io.cpp), converted on the GPU:
 *   OJB_RASTER_PNM  .pgm / .ppm payload (after the header): interleaved components, 8-bit or 16-bit
 *                   big-endian samples (ppm_in::read :338-374, ppm_out::write :539-556); 1 or 3 components
 *   OJB_RASTER_YUV  .yuv / .raw payload: component planes one after the other, 8-bit or 16-bit
 *                   little-endian (yuv_in::read :1350-1378, yuv_out::write :1477-1516, raw_in / raw_out)
 * Samples take 1 byte when the bit depth is <= 8, else 2; the codec must be configured / opened with the
 * matching container (OJB_U8 / OJB_U16).  Decoded samples are clamped to [0, 2^depth - 1] as the
 * reference's writers do. */
/*   OJB_RASTER_DPX_BE / _LE  image data of a .dpx file (encode only, like dpx_in :1800-2150): 10-bit RGB packed one
 *                   32-bit word per pixel, or 16-bit RGB with rows padded to 32-bit words, chosen by the
 *                   configured bit depth (10 or 16); _BE / _LE = byte order of the file (magic SDPX / XPDS) */
enum { OJB_RASTER_PNM = 0, OJB_RASTER_YUV = 1, OJB_RASTER_DPX_BE = 2, OJB_RASTER_DPX_LE = 3 };
int ojb_enc_encode_raster(ojb_encoder* e, uint32_t layout, const void* payload, uint64_t payload_bytes,
                          uint8_t* out, uint64_t out_cap, uint64_t* out_len);
/* device-resident variants: the frame lives in the encoder's image buffer */
void* ojb_enc_device_plane(ojb_encoder* e, uint32_t comp);
int ojb_enc_upload_frame(ojb_encoder* e, const void* const* planes, const uint32_t* strides);
int ojb_enc_encode_resident(ojb_encoder* e, uint8_t* out, uint64_t out_cap, uint64_t* out_len,
                            int out_on_device);
/* ---- the image in the caller's device memory ---------------------------------------------
 * One descriptor per frame: sample (x, y) of component c sits at
 *   (uint8_t*)base[c] + y * row_pitch[c] + x * col_stride[c] * (sample size)
 * in the container given to configure / read_headers (OJB_U8 / OJB_U16 / OJB_I32: 1 / 2 / 4 bytes), for the
 * component sizes ojb_frame_info reports (comp_w / comp_h; on decode the reduced sizes after
 * ojb_dec_restrict_input_resolution).  col_stride 1 = planar rows, 3 = RGB interleaved (HWC), 4 = RGBA, ...; so one
 * descriptor covers CHW at any pitch, HWC, a window inside a larger canvas, a slice of a batch, and a 4-channel
 * buffer of which only three components are coded.  The DWT kernels address the memory directly: no staging copy.
 * Components must not overlap (not checked: the caller's responsibility); the decoder writes exactly the samples
 * described and no other byte.
 * Ordering: before the library reads `in` (or writes `out`) it waits on an event recorded on cuda_stream (a
 * cudaStream_t; NULL = the legacy default stream), so work queued there before the call is complete.  The calls
 * return with their output complete, like the frame calls.
 * encode: the codestream goes to out (device memory when out_on_device, else host), *out_len its length.  The
 * decode call works after ojb_dec_read_headers or ojb_dec_read_headers_device.  With the codestream in device
 * memory on both sides, the device work of a call replays as one CUDA graph from the third call on, whatever
 * image buffers the calls name.
 * Errors: 0x000B003B a null base address, or a base / row pitch that is not a multiple of the sample size;
 * 0x000B003C col_stride 0; 0x000B003D (more than one row) a row pitch smaller than one row's footprint,
 * ((comp_w - 1) * col_stride + 1) * sample size; 0x000B003E a component spanning 4 GiB or more
 * ((comp_h - 1) * row_pitch + footprint: offsets from base are formed in 32 bits); 0x000B003F the call came before
 * configure / read_headers. */
typedef struct ojb_device_image {
  void*    base[16];       /* device address of sample (0,0) of component c */
  uint64_t row_pitch[16];  /* bytes from one row of component c to the next */
  uint32_t col_stride[16]; /* samples from one column to the next: 1 = planar rows, 3 = RGB HWC, 4 = RGBA ... */
} ojb_device_image;
int ojb_enc_encode_device(ojb_encoder* e, const ojb_device_image* in, void* cuda_stream,
                          uint8_t* out, uint64_t out_cap, uint64_t* out_len, int out_on_device);
int ojb_dec_decode_device(ojb_decoder* d, const ojb_device_image* out, void* cuda_stream);
uint32_t ojb_enc_kernel_launches(ojb_encoder* e);
/* stage times of the last encode, CUDA events on the codec's stream, milliseconds:
 * [0] H2D image  [1] DWT levels  [2] HT block encoder  [3] D2H block lengths  [4] wait + host packet
 * headers (device idle)  [5] H2D headers + assembly kernels  [6] D2H codestream  [7] host ms */
void ojb_enc_timings(ojb_encoder* e, float* ms8);
/* last decode: [0] H2D codestream  [1] host packet parse (device idle)  [2] HT block decoder
 * [3] inverse DWT levels  [4] D2H image  [7] host ms */
void ojb_dec_timings(ojb_decoder* d, float* ms8);
/* diagnostics: absolute stage marks of the last call (ms since ojb_marks_reference()), for timeline tools */
int ojb_marks_reference(void);
void ojb_enc_marks(ojb_encoder* e, float* ms8);
void ojb_dec_marks(ojb_decoder* d, float* ms8);
uint32_t ojb_enc_num_blocks(ojb_encoder* e);
/* parity hook: copy one sub-band's quantised sign-magnitude plane (what the block coder reads)
 * after an encode; out has band_w * band_h words */
int ojb_enc_read_band(ojb_encoder* e, uint32_t tile, uint32_t comp, uint32_t res, uint32_t band,
                      uint32_t* out, uint32_t* band_w, uint32_t* band_h);

/* parity hook: geometry and quantisation of one sub-band as the reference derives them
 * (subband::finalize_alloc, src/core/codestream/ojph_subband.cpp:133-203): info8 = band x0, y0, w, h,
 * K_max, resolution x0, y0, number of code-blocks; delta2 = step, 1/step (irreversible) */
int ojb_enc_band_info(ojb_encoder* e, uint32_t tile, uint32_t comp, uint32_t res, uint32_t band,
                      uint32_t* info8, float* delta2);

/* ---- encode to a target codestream size ---------------------------------------------------
 * With a target of `bytes` (0 = off, the default), every frame call of the encoder returns a codestream of at
 * most `bytes`: each code-block's cleanup pass sits at the bit-plane a rate-distortion selection on the device
 * chose (dropping its k lowest magnitude planes, or the whole block), single layer, readable by any HTJ2K decoder.
 * A target at or above the unconstrained size gives the unconstrained bytes.  After configure.
 * Errors: 0x000B0038 the target is below ojb_enc_min_size (also from a frame call after a reconfigure raised it);
 * 0x000B0039 the configuration codes 64-bit coefficients, or has a tile-part without packets (both refused by
 * ojb_enc_set_target_size, and by a frame call after a reconfigure to such a configuration);
 * 0x000B003A an internal consistency check: the selection rounds did not end (each round over the target shrinks the
 * selection, so this does not happen); 0x000B0049 the encoder has a target quality (ojb_enc_set_target_mse). */
int ojb_enc_set_target_size(ojb_encoder* e, uint64_t bytes);
/* the smallest codestream of the configured geometry: every code-block left out */
int ojb_enc_min_size(ojb_encoder* e, uint64_t* bytes);
/* parity hook: the selection of the last frame with a target.  *num_blocks, *kc (entries per block: 1 + the largest
 * K_max) always; the arrays when not null: kmax[nb], k[nb] (chosen; k = K_max: left out), R[nb * kc] (cleanup bytes
 * of block b at k, 0xFFFFFFFF: not codable, 0 past the block's top plane), D[nb * kc] (weighted squared error at k,
 * k <= K_max; after a transcode kmax[b] is 31 - q_b, q_b the lowest plane the input codes block b down to, and k and
 * D count planes from q_b); info5 = final body budget B*, selection rounds, header and marker bytes, codestream bytes, slope-key
 * threshold of the final selection (segments with key >= it are taken);
 * ms4 = distortion, candidate lengths, selection rounds, final block coding */
int ojb_enc_rate_info(ojb_encoder* e, uint32_t* num_blocks, uint32_t* kc, uint8_t* kmax, uint8_t* k, uint32_t* R,
                      double* D, uint64_t* info5, float* ms4);

/* ---- encode to a target quality ------------------------------------------------------------
 * With a target mean squared error `mse` (0 = off, the default), every frame call of the encoder returns a codestream
 * whose squared error against the source is at most floor(mse * N): SSE = the sum over every component c of
 * sum (decoded - source)^2 over its comp_w x comp_h samples, decoded = what this library's decoder outputs in the
 * configured sample container (after rounding, clamping and the inverse NLT), N = sum_c comp_w * comp_h.  The stream
 * is single-layer and cleanup-only, readable by any HTJ2K decoder; each code-block's cleanup pass sits at the
 * bit-plane a search on the device chose.  Each round of that search reconstructs a selection exactly as the decoder
 * would and measures its error, so the limit is met exactly; the search stops once the passing and the failing
 * selection differ by at most max(0.25 %, 64 bytes) of code-block bytes, or their slope keys are adjacent.  A
 * reversible configuration always reaches the target (key 0 is lossless).  An irreversible one may not: its
 * quantisation sets a floor, and below it the call returns the unconstrained stream with reached = 0.
 * Needs, once set, a second coefficient arena and a scratch image of the frame in the configured sample container on
 * the device (for an 8192 x 8192 x 3 12-bit frame about 1.07 GB, and 0.40 GB in 16-bit or 0.81 GB in 32-bit samples).  After configure.  Not combined with a target size.
 * Errors: 0x000B0048 mse is negative, infinite or NaN; 0x000B0049 the encoder has a target size (ojb_enc_set_target_size
 * refuses a size while a quality target is set, with the same code); 0x000B004A the configuration codes 64-bit
 * coefficients, or has a tile-part without packets (refused here, and by a frame call after a reconfigure to such a
 * configuration). */
int ojb_enc_set_target_mse(ojb_encoder* e, double mse);
#define OJB_QUALITY_MAX_ROUNDS 64
typedef struct {
  uint64_t num_samples;          /* N */
  uint64_t limit;                /* floor(mse * N): the largest SSE accepted */
  uint64_t sse_lo, sse_hi;       /* exact SSE of the returned stream, 128 bits */
  double comp_sse[16];           /* the same per component */
  uint32_t num_comps;
  uint32_t reached;              /* 1: sse <= limit */
  uint32_t rounds;               /* measured rounds, and per round: */
  uint32_t pass_measured;        /* the passing key's selection was measured (0: key 0 of a lossless configuration) */
  uint64_t round_key[OJB_QUALITY_MAX_ROUNDS];    /* slope key tried (segments with key >= it are taken; 2^32: none) */
  uint64_t round_sse_lo[OJB_QUALITY_MAX_ROUNDS], round_sse_hi[OJB_QUALITY_MAX_ROUNDS];
  uint64_t round_body[OJB_QUALITY_MAX_ROUNDS];   /* code-block bytes of the selection */
  uint64_t pass_key, fail_key;   /* the final bracket: the returned selection, and the failing one (2^32 unmeasured) */
  uint64_t pass_body, fail_body;
  uint32_t fail_measured, pad;
  uint64_t body0;                /* code-block bytes of the unconstrained selection (key 0) */
  double model_round1;           /* the distortion model's SSE for round 1's selection */
  float ms_candidates, ms_rounds, ms_final;      /* stage times (CUDA events): distortion + candidate lengths; hull,
                                                    bracket and rounds; the final block coding */
  float pad2;
} ojb_quality_info;
/* report and parity hook: the search of the last frame encoded with a target quality (0x000B004B: none) */
int ojb_enc_quality_info(ojb_encoder* e, ojb_quality_info* out);

/* ---- transcode a codestream ----------------------------------------------------------------
 * Re-codes an existing codestream from its decoded code-blocks, never from an image: no inverse or forward transform,
 * and no second generation of rounding.  The output has the input's geometry and coding parameters and is single-layer
 * and cleanup-only; its main header is the input's byte for byte without TLM / PLM segments, plus a TLM of its own
 * when the input had one, and its tile-parts are divided as the input's.  Block b starts at q_b, the lowest plane the
 * input codes it down to: 30 - missing MSBs with a cleanup pass only, one lower with SigProp / MagRef passes; candidate
 * k = 0 re-codes exactly the bits the input carried.  So without a target every block is re-coded at k = 0: a stream
 * this library or OpenJPH wrote comes back byte for byte, and a stream with SigProp / MagRef passes comes back in
 * cleanup-only form, sample for sample, except that in a block with SigProp but no MagRef pass every sample that
 * became significant in the cleanup pass keeps its bin centre (a quarter of the cleanup plane's step) as a coded bit.
 * The encoder's targets apply as to an image: ojb_enc_set_target_size with its min_size and rules, and
 * ojb_enc_set_target_mse / PSNR, whose source is the input as this library's decoder returns it in the configured
 * sample container (for a lossless input: the original image).  ojb_enc_rate_info, ojb_enc_quality_info,
 * ojb_enc_min_size and ojb_enc_timings report on transcodes (timings: [1] the input to the device and its block
 * decode, [7] the host parse).  The device holds the coefficient arena, block slots, the input and block tables; the
 * refinement-pass scratch only when the input has such passes; with a target quality also what that target allocates.
 * Errors: 0x000B004C SOP or EPH markers (Scod bits 1-2), which the output does not write; 0x000B004D a POC, PPM or PPT
 * segment (packet headers elsewhere or in another order); 0x000B004E a tile-part header segment other than PLT;
 * 0x000B004F tile-parts that follow none of the divisions the encoder writes (none, by resolution, by component, by
 * both); 0x000B0050 a configuration on the 64-bit coefficient path (no target size or quality there); 0x000B0051 a
 * truncated or damaged codestream, or a code-block that fails to decode (there is no resilient transcode);
 * 0x000B0052 ojb_enc_transcode before ojb_enc_transcode_headers; 0x000B0053 a pixel frame call (encode, upload, raster,
 * lines) on an encoder configured by ojb_enc_transcode_headers.  A refused input leaves the encoder as it was.
 *
 * Reduced resolution (ojb_enc_transcode_headers_reduced, skipped_res = r > 0): the output is the input with its top r
 * resolution levels dropped, as ojph_expand -skip_res r would reconstruct it -- a 2K stream from a 4K master, a proxy or
 * a thumbnail stream -- from the kept code-blocks alone.  SIZ's extent, image offset and tile offset become
 * ceil(v / 2^r), and the tile size XTsiz / 2^r along a direction with more than one tile; so every kept tile, resolution,
 * band, precinct and code-block keeps its rectangle.  COD and every COC lose r levels (and their precinct sizes of the
 * dropped resolutions), QCD and every QCC keep their first 1 + 3 (D_c - r) step sizes (guard bits and Sqcd as they
 * are), CAP's MAGB is recomputed, and every other main-header segment is copied.  The tile-part division kind and the
 * TLM follow the input's.  Without a target every kept block is re-coded as the input carried it, and the reference
 * decoder's output of the result equals its decode of the input restricted to (r, r), sample for sample; a quality
 * target's source is that restricted decode.  ojb_enc_transcode, the target setters, ojb_enc_min_size,
 * ojb_enc_rate_info and ojb_enc_quality_info describe the output geometry.  r = 0 is ojb_enc_transcode_headers.
 * Errors besides the ones above: 0x000300A2 r above COD's level count, 0x000B0007 r above a component's own (COC) count
 * (both as ojb_dec_restrict_input_resolution; r equal to a count leaves that component without levels, which is
 * valid); 0x000B0054 a DFS decomposition structure (a dropped level's split would set the reduction per direction and
 * renumber the step sizes; ATK kernels alone are fine); 0x000B0055 a tile grid that does not survive the reduction
 * (several tiles along a direction whose tile size is not a multiple of 2^r, or a tile that would keep no samples:
 * tile indices, tile-parts and TLM entries stay one-to-one with the input's); 0x000B0056 the input's Rsiz names the
 * broadcast or IMF profile (bits 8-11, without the Part 2 flag) and the reduced parameters break that profile's rules
 * (e.g. broadcast needs 1 to 5 levels). */
/* the encoder counterpart of ojb_dec_read_headers: configures e from a codestream's headers and tile-parts (host
 * memory, or device memory when on_device, with >= 32 readable bytes after its end); the target setters follow it as
 * they follow ojb_enc_configure */
int ojb_enc_transcode_headers(ojb_encoder* e, const void* j2c, uint64_t len, int on_device, uint32_t sample_type);
/* the same for an output with the input's top skipped_res resolution levels dropped; info (may be null) receives the
 * output's geometry, as a decoder of the output reports it */
int ojb_enc_transcode_headers_reduced(ojb_encoder* e, const void* j2c, uint64_t len, int on_device, uint32_t sample_type,
                                      uint32_t skipped_res, ojb_frame_info* info);
/* re-codes the codestream (same main header and tile-part structure as the headers call, else it is read again) to
 * e's target; out on the device when out_on_device */
int ojb_enc_transcode(ojb_encoder* e, const void* j2c, uint64_t len, int on_device,
                      uint8_t* out, uint64_t out_cap, uint64_t* out_len, int out_on_device);

/* ---- decode: ojph::codestream read side ------------------------------------------------- */
ojb_decoder* ojb_dec_create(void);
void ojb_dec_destroy(ojb_decoder* d);
int ojb_dec_enable_resilience(ojb_decoder* d);           /* codestream::enable_resilience() */
/* codestream::read_headers(infile_base*): j2c must stay valid until the decode call returns */
int ojb_dec_read_headers(ojb_decoder* d, const uint8_t* j2c, uint64_t len, uint32_t sample_type,
                         ojb_frame_info* info);
/* codestream::restrict_input_resolution(skipped_res_for_read, skipped_res_for_recon)
 * (ojph_codestream_local.cpp:883-900), after read_headers: the top skipped_res_for_recon resolutions are
 * not reconstructed (every component comes out 2^n times smaller; *info receives the new comp_w / comp_h),
 * the top skipped_res_for_read (>= skipped_res_for_recon) are not decoded and read as zero. */
int ojb_dec_restrict_input_resolution(ojb_decoder* d, uint32_t skipped_res_for_read, uint32_t skipped_res_for_recon,
                                      ojb_frame_info* info);
/* the getters of ojph::param_cod on the read side (ojph_params.h:132-158), for one component (its COC when
 * it has one, else the COD), and of param_siz that ojb_frame_info does not carry */
typedef struct ojb_coding_style {
  uint32_t num_decomps, reversible, color_transform;
  uint32_t block_w, block_h;                 /* get_block_dims; log2 = get_log_block_dims */
  uint32_t precinct_w[33], precinct_h[33];   /* get_precinct_size(level), 0 .. num_decomps */
  uint32_t prog_order;                       /* get_progression_order: 0 LRCP 1 RLCP 2 RPCL 3 PCRL 4 CPRL */
  uint32_t num_layers;
  uint32_t may_use_sop, use_eph, vertical_causality;
  uint32_t tile_w, tile_h, tile_off_x, tile_off_y;   /* param_siz::get_tile_size / get_tile_offset */
} ojb_coding_style;
int ojb_dec_get_coding_style(ojb_decoder* d, uint32_t comp, ojb_coding_style* out);
/* codestream::create() + the pull() loop: decodes every component into planes */
int ojb_dec_decode_frame(ojb_decoder* d, void* const* planes, const uint32_t* strides);
int ojb_dec_decode_resident(ojb_decoder* d);             /* result stays in the device image buffer */
/* decode into a file payload (see ojb_enc_encode_raster); *payload_bytes receives the size */
int ojb_dec_decode_raster(ojb_decoder* d, uint32_t layout, void* payload, uint64_t payload_cap, uint64_t* payload_bytes);
/* The reference's line interface on the read side (needs the OJB_I32 container):
 *   ojb_dec_set_planar = codestream::set_planar (default after read_headers: colour transform ? 0 : 1,
 *                        ojph_codestream_local.cpp:879);
 *   ojb_dec_begin_pull = codestream::create() (:912-1115): runs the GPU decode into a library-owned frame;
 *   ojb_dec_pull       = codestream::pull(ui32& comp_num) (:1227-1272): the next line, library owned and
 *                        valid until the next call; planar => all rows of component 0 first, else row by
 *                        row, component by component; NULL (and *comp_num = 0) after the last line. */
int ojb_dec_set_planar(ojb_decoder* d, int planar);
int ojb_dec_begin_pull(ojb_decoder* d);
const int32_t* ojb_dec_pull(ojb_decoder* d, uint32_t* comp_num);
void* ojb_dec_device_plane(ojb_decoder* d, uint32_t comp);
/* after read_headers: the same codestream bytes are already in device memory (with >= 32 readable
 * bytes after the end); the next decode reads them there instead of uploading j2c */
int ojb_dec_use_device_codestream(ojb_decoder* d, const void* dev_bytes);
/* codestream::read_headers for a codestream that exists in DEVICE memory only (complete when the call is
 * made, >= 32 readable bytes after its end, valid until the decode call returns): the marker segments and
 * packet headers the host parsers read (ojph_codestream_local.cpp:734-880, ojph_precinct.cpp:328-573) are
 * fetched in 32 KB pages; code-block bodies never leave the device.  ojb_dec_mirror_bytes = bytes fetched
 * so far for the current codestream (headers + the packet headers parsed by the last decode). */
int ojb_dec_read_headers_device(ojb_decoder* d, const void* dev_j2c, uint64_t len, uint32_t sample_type,
                                ojb_frame_info* info);
uint64_t ojb_dec_mirror_bytes(ojb_decoder* d);
uint32_t ojb_dec_failed_blocks(ojb_decoder* d);
/* parity hook: parse the packet headers of the codestream given to read_headers and list every
 * code-block (precinct::parse, src/core/codestream/ojph_precinct.cpp:328-573): geometry, missing msbs,
 * passes, lengths and the byte offset of its data in j2c */
struct ojb_block_desc;
int ojb_dec_list_blocks(ojb_decoder* d, struct ojb_block_desc* out, uint32_t cap, uint32_t* n);
uint32_t ojb_dec_kernel_launches(ojb_decoder* d);
int ojb_dec_read_band(ojb_decoder* d, uint32_t tile, uint32_t comp, uint32_t res, uint32_t band,
                      uint32_t* out, uint32_t* band_w, uint32_t* band_h);

/* ---- kernel-level batch entry points (fine boundary: struct codeblock_fun,
 *      src/core/codestream/ojph_codeblock_fun.h:93-120) ----------------------------------- */
typedef struct ojb_block_desc {
  uint64_t sample_off;     /* word offset of sample (0,0) in the samples array */
  uint32_t stride, w, h;   /* stride in words */
  uint32_t missing_msbs;   /* encode: K_max - 1; decode: from the packet header */
  uint32_t num_passes;     /* decode only */
  uint32_t len1, len2;     /* decode in: cleanup / refinement bytes; encode out: len1 = bytes */
  uint64_t byte_off;       /* offset of the block's coded bytes in the bytes array */
  uint32_t status;         /* out: 0 ok, 1 failed / not coded */
  uint32_t causal;
} ojb_block_desc;
/* encode_cb32 for n blocks: samples = MSB-aligned sign-magnitude (host); coded bytes are packed
 * into bytes (cap bytes_cap) and desc[i].byte_off / len1 are filled */
int ojb_encode_blocks(const uint32_t* samples, uint64_t n_words, ojb_block_desc* desc, uint32_t n,
                      uint8_t* bytes, uint64_t bytes_cap, uint64_t* bytes_used);
/* decode_cb32 for n blocks: output sign-magnitude samples (out_mode 0) written to samples */
int ojb_decode_blocks(const uint8_t* bytes, uint64_t n_bytes, ojb_block_desc* desc, uint32_t n,
                      uint32_t* samples, uint64_t n_words);

/* ---- one image over the GPUs of a box (SURVEY 8(e)) -----------------------------------------------------
 * One process per GPU.  Tiles are independent units of the codestream (the reference builds one component /
 * resolution tree per tile, src/core/codestream/ojph_codestream_local.cpp:132-168, and concatenates the
 * tile-parts in tile-index order at flush, :1148-1164): rank r codes the tiles t with t % world == r, and the
 * only data-path exchange is the final gather to the writer rank -- tile-part bytes on encode, decoded tile
 * samples on decode -- device to device over NCCL.  The codestream on the writer is byte-identical to the one a
 * single encoder (or the reference) produces.  Every rank makes the same calls in the same order.
 * Transport: NCCL (communicator from a unique id the caller hands to every rank, e.g. through the launcher's
 * store), or caller-supplied callbacks. */
typedef struct ojb_shard ojb_shard;
typedef struct ojb_comm_callbacks {
  void* ctx;
  int (*allgather)(void* ctx, const void* send_host, void* recv_host, uint64_t bytes_per_rank);
  int (*bcast)(void* ctx, void* dev_buf, uint64_t bytes, uint32_t root);
  int (*send)(void* ctx, const void* dev_buf, uint64_t bytes, uint32_t peer);     /* blocking */
  int (*recv)(void* ctx, void* dev_buf, uint64_t bytes, uint32_t peer);           /* blocking */
} ojb_comm_callbacks;
int ojb_shard_unique_id(uint8_t out[128]);                        /* ncclGetUniqueId, on one rank */
ojb_shard* ojb_shard_create_nccl(uint32_t rank, uint32_t world, const uint8_t unique_id[128]);   /* current device */
ojb_shard* ojb_shard_create(uint32_t rank, uint32_t world, const ojb_comm_callbacks* cb);
void ojb_shard_destroy(ojb_shard* s);
const char* ojb_shard_last_error(void);
/* param setters + write_headers of the whole image; this rank prepares its tiles */
int ojb_shard_enc_configure(ojb_shard* s, const ojb_params* p, uint32_t sample_type, uint32_t writer_rank);
/* exchange() loop + flush(): planes = the whole image in host memory (a rank reads only its own tiles'
 * rectangles); the codestream arrives in out on the writer rank (*out_len = 0 elsewhere) */
int ojb_shard_enc_encode(ojb_shard* s, const void* const* planes, const uint32_t* strides,
                         uint8_t* out, uint64_t out_cap, uint64_t* out_len);
/* read_headers + create + pull loop: j2c is read on the writer rank only (broadcast device to device); the
 * decoded components arrive in planes on the writer rank */
int ojb_shard_dec_decode(ojb_shard* s, const uint8_t* j2c, uint64_t len, uint32_t sample_type, uint32_t writer_rank,
                         void* const* planes, const uint32_t* strides, ojb_frame_info* info);
/* device-resident forms: tiles uploaded once per rank, codestream left in / read from the writer's device memory, decoded
 * image left in the writer's device image buffer */
int ojb_shard_enc_upload(ojb_shard* s, const void* const* planes, const uint32_t* strides);
int ojb_shard_enc_encode_resident(ojb_shard* s, uint64_t* out_len);
const void* ojb_shard_device_codestream(ojb_shard* s);
int ojb_shard_dec_decode_resident(ojb_shard* s, const void* dev_j2c, uint64_t len, uint32_t sample_type, uint32_t writer_rank,
                                  ojb_frame_info* info);
void* ojb_shard_device_plane(ojb_shard* s, uint32_t comp);
/* frame-parallel batches: variable-length gather of device buffers (one codestream per rank) to the writer's
 * device buffer, rank order; offsets[world + 1] */
int ojb_shard_gatherv(ojb_shard* s, const void* dev, uint64_t bytes, uint32_t writer_rank, void* out_dev, uint64_t out_cap,
                      uint64_t* offsets);
/* How the image is cut (before ojb_shard_enc_configure / the decode calls; every rank the same).  0 (default): tiles.
 * 1: ROW REGIONS -- every tile-component is cut into `world` horizontal slabs; rank g codes the code-blocks that start
 * in slab g from an input halo of 2 (2^D - 1) rows (5/3) / 4 (2^D - 1) rows (9/7) per side, the footprint of one
 * lifting step reaching +-1 (src/core/transform/ojph_transform.cpp:376-390), so nothing is exchanged in mid-pipeline;
 * the one exchange is the gather of code-block bytes + lengths to the writer, which then writes packet headers and
 * markers as a single encoder does (precinct::write, src/core/codestream/ojph_precinct.cpp:281-324).  This also
 * splits a SINGLE-TILE image (SURVEY 8(e)); the codestream stays byte-identical.  Decode: each rank decodes the
 * blocks its slab depends on and delivers its rows. */
int ojb_shard_set_partition(ojb_shard* s, uint32_t kind);
/* row regions, after ojb_shard_enc_configure: rows [*lo, *hi) of component comp (first tile) this rank's encoder reads;
 * returns 0 when the partition is not row regions */
uint32_t ojb_shard_region_rows(ojb_shard* s, uint32_t comp, uint32_t* lo, uint32_t* hi);
void ojb_shard_timings(ojb_shard* s, float* ms2);                 /* last call: codec ms, gather ms (this rank) */
uint32_t ojb_shard_rank(ojb_shard* s);
uint32_t ojb_shard_world(ojb_shard* s);

#ifdef __cplusplus
}
#endif
#endif /* OJPH_B200_H */
