// ojb_codec.h -- encoder / decoder objects: the GPU counterparts of the reference's
// local::codestream (src/core/codestream/ojph_codestream_local.h:63-169).  exchange()/pull()
// only move lines in and out of a pinned frame buffer; all GPU work happens in flush() (encode)
// and create() (decode) -- SURVEY §8(b).
#pragma once
#include "ojb_layout.h"
#include "ojb_kernels.h"
#include <memory>
#include <cstdlib>

namespace ojb {

void cuda_check(cudaError_t e, const char* what);

struct DeviceBuf {
  void* p = nullptr; size_t cap = 0;
  ~DeviceBuf();
  void reserve(size_t n);
  template <typename T> T* as() { return reinterpret_cast<T*>(p); }
};
struct PinnedBuf {
  void* p = nullptr; size_t cap = 0;
  ~PinnedBuf();
  void reserve(size_t n);
  template <typename T> T* as() { return reinterpret_cast<T*>(p); }
};

struct Timings { float h2d_ms = 0, kernels_ms = 0, host_ms = 0, d2h_ms = 0; };

// sample container of the image buffers handed to / returned by the frame calls
enum SampleType : uint32_t { ST_U8 = 0, ST_U16 = 1, ST_I32 = 2 };
inline uint32_t esize_of(uint32_t st) { return st == ST_U8 ? 1u : (st == ST_U16 ? 2u : 4u); }

// the HT tables the block encoders (enc) or decoders read, packed as ojb_kernels.h describes them, into dev
void upload_ht_tables(bool enc, DeviceBuf& dev);
// a code-block's slot in the encoder's arena: its worst-case bytes, a multiple of 16
uint32_t enc_slot_cap(uint32_t w, uint32_t h, uint32_t K_max, bool wide);

class CodecBase {
public:
  CodecBase();
  virtual ~CodecBase();
  Params params;
  Layout layout;
  cudaStream_t stream = nullptr;
  SideStream side;                     // second stream + fork / join events (see ojb_kernels.h)
  uint32_t last_launches = 0;          // kernels launched by the last frame call
  uint32_t host_threads = 4;           // host threads used for packet headers
  // stage timing of the last frame call (CUDA events on `stream`, ms)
  enum { EV_MAX = 12 };
  cudaEvent_t ev[EV_MAX] = {nullptr};
  float stage_ms[EV_MAX] = {0};
  double host_ms = 0;                  // host time between the two device phases
  bool capturing = false;              // inside run_frame's stream capture: stage marks become event-record NODES
#ifdef OJB_EMU_BUILD
  void mark(int i) { cudaEventRecord(ev[i], stream); }
#else
  void mark(int i) { if (capturing) cudaEventRecordWithFlags(ev[i], stream, cudaEventRecordExternal); else cudaEventRecord(ev[i], stream); }
#endif
  // The device work of a frame call as a CUDA graph.  Small frames are bound by the launch rate of the process
  // (about 45 launches per encode + decode), not by the SMs: the resident forms, whose launches and arguments repeat
  // frame after frame, run eagerly the first time a given argument set is seen, are captured the second time and are
  // one cudaGraphLaunch from then on.  `key` holds everything the enqueued work depends on.  OJB_NO_GRAPHS=1 disables it.
  struct FrameGraph { std::vector<uint64_t> key, seen; cudaGraphExec_t exec = nullptr; uint32_t launches = 0; bool off = false; };
  FrameGraph fgraph;
  template <typename F> void run_frame(const std::vector<uint64_t>& key, F&& enqueue);
  void drop_graph();
  void collect(int n) { for (int i = 0; i + 1 < n; ++i) cudaEventElapsedTime(&stage_ms[i], ev[i], ev[i + 1]); }
  void upload_tables();
  DeviceBuf d_tables_enc, d_tables_dec;
  // image planes on the device: component c at byte offset img_off[c], tight rows
  DeviceBuf d_image;
  std::vector<uint64_t> img_off;
  std::vector<uint32_t> img_w, img_h;
  uint32_t img_type = ST_I32;
  uint32_t max_block_w = 64;            // widest nominal code-block of the current geometry
  // decoder: resolutions dropped from the top (codestream::restrict_input_resolution,
  // ojph_codestream_local.cpp:883-900): skip_recon levels are not reconstructed (smaller output),
  // skip_read >= skip_recon levels are not decoded (their bands read as zero)
  uint32_t skip_read = 0, skip_recon = 0;
  size_t img_bytes = 0;
  void plan_image(uint32_t sample_type, bool alloc = true);     // alloc = false: the planes' geometry only, no d_image
  // The image as the first-level DWT jobs reach it: one ImgComp per component in device memory.  Slot 0 describes
  // d_image (written by plan_image), slot 1 the caller's memory of a *_device call: the frame's own work copies it
  // from h_img, so a captured frame graph replays with whatever buffers the next call names.
  enum { IMG_SLOTS = 16 };
  DeviceBuf d_img;
  PinnedBuf h_img;
  cudaEvent_t ev_caller = nullptr;
  bool caller_interleaved = false;     // the first three components of the image in slot 1 sit next to each other
  const ImgComp* img_slot(bool caller) const { return reinterpret_cast<const ImgComp*>(d_img.p) + (caller ? IMG_SLOTS : 0); }
  // slot 2: the encoder's scratch image of a quality target (Encoder::plan_quality)
  const ImgComp* scratch_slot() const { return reinterpret_cast<const ImgComp*>(d_img.p) + 2 * IMG_SLOTS; }
  // the next frame call reads (encoder) or writes (decoder) the caller's memory described by comps[num_comps], after
  // the work enqueued so far on caller_stream (0: the legacy default stream)
  void use_caller_image(const ImgComp* comps, cudaStream_t caller_stream);
  void enqueue_caller_image();         // inside the frame's work: h_img -> slot 1
  DeviceBuf d_coef;                    // coefficient arena (32-bit words; 64-bit elements in wide mode)
  bool wide = false;                   // some component needs more than 32 bits: every plane holds 64-bit elements, general kernels only
  // DWT jobs per level (index 0: full resolution level D, ...), uploaded once
  // jobs of one level are grouped by the kernel variant that runs them
  struct JobGroup { std::vector<DwtJob> jobs; uint32_t ctas = 0, ncomp = 1; bool first = false, stream = false, reversible = true; size_t dev_off = 0; };
  std::vector<std::vector<JobGroup>> jobs;
  DeviceBuf d_jobs;
  // the analysis (forward) or synthesis jobs of the geometry into out, uploaded to dev (the codec's own: jobs, d_jobs)
  void build_dwt_jobs(bool forward, std::vector<std::vector<JobGroup>>& out, DeviceBuf& dev);
  // every level of groups (uploaded to dev) between the image img and the arena coef: analysis from the finest level
  // down, synthesis from the coarsest up
  void enqueue_dwt(bool forward, const std::vector<std::vector<JobGroup>>& groups, DeviceBuf& dev, const ImgComp* img,
                   bool interleaved, uint32_t* coef);
  // one image over several GPUs (ojb_shard.cpp): this object works on the tiles whose mask byte is set (empty =
  // all tiles).  The geometry, arenas and block tables stay those of the whole image, so Isot, canvas coordinates
  // and byte offsets are the single-encoder ones; DWT jobs, code-blocks and packets of the other tiles are skipped.
  std::vector<uint8_t> tile_mask;
  bool tile_wanted(uint32_t t) const { return tile_mask.empty() || (t < tile_mask.size() && tile_mask[t] != 0); }
  // one image over several GPUs by ROW REGIONS (ojb_shard.cpp, partition "regions"; SURVEY 8(e)): a tile-component is
  // cut into `world` horizontal slabs.  Encoder: rank g codes the code-blocks whose first row falls into slab g and runs,
  // at every decomposition level, only the row chunks of the streaming DWT kernels those blocks depend on -- the input
  // rows it needs are its slab plus a halo of about 2 (2^D - 1) rows (5/3) or 4 (2^D - 1) rows (9/7) each side, the
  // exact footprint of one lifting step reaching +-1 (ojph_transform.cpp:376-390), so no coefficient crosses a rank
  // boundary in mid-pipeline.  Decoder: rank g delivers the image rows of slab g, runs the synthesis chunks that
  // produce them and decodes every code-block those chunks read (its own and a halo of its neighbours').  The
  // geometry, arenas and block tables stay those of the whole image, as with a tile mask.  A tile-component whose
  // levels do not all run on the streaming kernels (degenerate sizes, DFS / ATK, 64-bit path) keeps whole-plane
  // transforms on every rank; only its block coding is shared.
  struct RegionSpec { uint32_t rank = 0, world = 0; bool on() const { return world > 1; } } region;
  struct RegionWin { uint32_t chunk0 = 0, nchunks = 0; bool full = true; };   // row chunks of one level's job; full: all of them
  std::vector<std::vector<std::vector<RegionWin>>> region_win;   // [tile][comp][resolution being split / rebuilt]
  std::vector<uint8_t> region_owner;   // encoder: the rank that codes block b
  std::vector<uint8_t> region_blocks;  // the blocks this object works on (encoder: the ones it owns; decoder: all its rows depend on)
  struct RowSpan { uint32_t lo = 0, hi = 0; };       // rows [lo, hi) in absolute tile-component coordinates
  std::vector<std::vector<RowSpan>> region_rows;     // [tile][comp]: encoder: image rows this rank reads; decoder: rows it delivers
  static RowSpan region_slab(const Rect& tc, uint32_t g, uint32_t world);
  void plan_region(bool forward);
  bool no_stream_dwt = getenv("OJB_NO_STREAM_DWT") != nullptr;     // force the general shared-memory DWT kernels (tests)
  bool no_fast_blocks = getenv("OJB_NO_FAST_BLOCKS") != nullptr;   // force the general block-coder kernels (tests, A/B)
};

class Decoder;
// one frame's block decode (Decoder::frame_records): the output mode, blocks through the specialised kernel, whether
// no block has refinement passes
struct BlockFrame { uint32_t nfast = 0, dec_out = 0; bool cleanup_only = true; };

class Encoder : public CodecBase {
public:
  ~Encoder();
  // finalises parameters, builds geometry and device arenas, produces the main header
  void configure(const Params& p, uint32_t sample_type);
  // configure's part after the main header: geometry, arenas, block tables, header plan (params and main_header set)
  void setup(uint32_t sample_type);
  // encode one frame whose component planes are on the host (pinned or pageable; planes[c] points at sample (0,0) of
  // component c, stride in samples), already in d_image (planes == nullptr), or in the caller's device memory
  // (caller_image: described by use_caller_image)
  size_t encode(const void* const* planes, const uint32_t* strides, bool caller_image,
                uint8_t* out, size_t out_cap, bool out_on_device);
  // row regions (ojb_shard.cpp): the frame call split at the point where code-block bytes change hands.  encode_front:
  // this rank's transform and block coding of the image in d_image; encode_back, on the writer once every rank's blocks
  // sit in its slots: packet headers, markers and layout into out (device memory)
  void encode_front();
  size_t encode_back(uint8_t* out, size_t out_cap);
  uint32_t status_flags = 0;
  // The stages of a frame call.  Frame holds what the entry point chose for this frame: where the coefficients come
  // from (front: the forward DWT, a transcode's block decoders, or nothing -- encode_back's blocks are coded already),
  // whether a target selects the coded planes, and the block arrays the stages read.
  struct Frame {
    enum Front : uint8_t { DWT, TRANSCODE, CODED } front = DWT;
    bool caller_image = false;
    bool graph = false;                  // the device work may be captured and replayed as a graph (resident form)
    bool rc = false, rq = false;         // a size or a quality target selects each block's plane
    uint32_t nb = 0;
    const EncBlock* blocks = nullptr;    // where each block starts (a transcode: at the input's plane)
    const EncBlock* code_blocks = nullptr;   // what the block coder codes: blocks, or with a target the selection in work
    EncBlock* work = nullptr;
  };
  Frame begin_frame(Frame::Front front, bool targets, bool caller_image = false, const void* const* planes = nullptr,
                    const uint32_t* strides = nullptr);
  void upload_planes(const void* const* planes, const uint32_t* strides);   // host planes -> d_image, on stream
  void enqueue_front(const Frame& f);
  void enqueue_code(const Frame& f);
  void enqueue_rc(const Frame& f);     // a target's candidates and the selection rounds inside the frame's graph
  void rc_size(const Frame& f, bool first);
  void rc_state_out(const Frame& f);
  void rq_round(const Frame& f);
  void rq_final(const Frame& f);
  bool rc_settle(const Frame& f);
  void check_coder_status();
  size_t finish_device(const Frame& f, uint8_t* out, size_t out_cap, bool out_on_device);
  void enqueue_device_layout(const Frame& f, uint8_t* dev_out, uint64_t cap);
  size_t finish_host(const Frame& f, uint8_t* out, size_t out_cap, bool out_on_device);
  struct HostLayout;
  void host_packets(const Frame& f, HostLayout& hl);
  size_t host_markers(HostLayout& hl);
  size_t end_frame(const Frame& f, uint8_t* out, const uint8_t* dev_out, size_t total, bool out_on_device);
  void rc_times(const Frame& f);
  // line-based front end (ojph::codestream::exchange): lines go to a pinned frame
  PinnedBuf h_frame;
  std::vector<uint32_t> line_cur;
  uint32_t cur_comp = 0;
  bool lines_done = false;
  int32_t* exchange(const int32_t* line_written, uint32_t& next_comp);
  std::vector<int32_t> line_buf;
  std::vector<uint8_t> main_header;
  std::vector<EncBlock> h_blocks;
  DeviceBuf d_blocks, d_results, d_status, d_slots, d_dst, d_hdr, d_pieces, d_out;
  PinnedBuf h_results, h_dst, h_hdr, h_pieces, h_status;
  std::vector<CodedBlock> coded;
  // with a tile mask the output is this object's tile-parts only (no main header, no EOC); where each one sits:
  struct TilePartOut { uint32_t tile; uint64_t offset; uint32_t bytes; };
  std::vector<TilePartOut> last_tileparts;
  size_t slot_bytes = 0;
  uint32_t num_fast_blocks = 0;        // blocks flagged ENC_FLAG_FAST
  bool few_blocks_warp = false;        // sharded image, few blocks on this rank: the warp-per-block encoder (see configure)
  // packet headers, tile-part markers and the byte layout on the device (pkt_headers.cu): no host round trip between
  // the block coder and the finished codestream.  OJB_HOST_HEADERS=1 keeps the host writer (ojb_layout.cpp), which also
  // serves the odd configuration with an empty tile-part.  With a tile mask (ojb_shard.cpp) the output is this rank's
  // tile-parts only and their positions come back in a few bytes
  bool device_headers = false;
  HdrPlanDev hplan;
  std::vector<uint8_t> fixed_blob;     // main header [+ TLM with blank lengths]
  DeviceBuf d_fixed, d_hplan[32];
  PinnedBuf h_total, h_tpout;
  std::vector<uint32_t> h_tp_tile;
  size_t hscr_bytes = 0;
  void build_header_plan();
  size_t out_cap_dev = 0;
  // rate control (rate_ctrl.cu): with a target, every frame call returns a codestream of at most target_bytes, each
  // code-block coded at the bit-plane a rate-distortion selection on the device chose.  0 = off.  The selection works
  // on a per-frame copy of the block array (d_work); the header plan sizes each selection (rc_sizing: it exists)
  uint64_t target_bytes = 0;
  uint64_t min_bytes = 0;              // every block left out: depends on the geometry only
  bool rc_sizing = false;
  enum { RC_ROUNDS = 3 };              // selection rounds inside the frame's graph; more run eagerly when needed
  RcTables rc;
  DeviceBuf d_rc, d_work;
  PinnedBuf h_rc;                      // RcState, then the chosen k per block
  uint32_t rc_kc = 0;
  float rc_ms[4] = {0, 0, 0, 0};       // last frame: distortion, candidate lengths, selection, final encode
  void set_target(uint64_t bytes);
  void check_target_size(uint64_t bytes) const;
  uint64_t min_size_of_geometry() const;
  void plan_rate_control();
  bool rc_on() const { return target_bytes != 0; }
  // quality target (rate_ctrl.cu): with a target mean squared error (0 = off), every frame call returns the smallest
  // stream the search finds whose exact squared error against the source, summed over every sample of every
  // component, is at most rq_limit = floor(target_mse * N); N = the number of samples.  Each round of the search
  // reconstructs a selection as the decoder would -- into a second coefficient arena (d_rcoef), through the decoder's
  // synthesis jobs (rq_jobs) into a scratch image (d_rimg, slot 2 of d_img) -- and measures it.  The buffers exist
  // only once a target is set (plan_quality)
  double target_mse = 0;
  uint64_t rq_limit = 0, rq_samples = 0;
  bool rq_planned = false, rq_lossless0 = false, rq_valid = false;
  // rounds inside the frame's graph; a search that needs more goes on eagerly, one synchronisation per round.  Their
  // inverse DWT launches run even after the search is done.  On the 8K 12-bit frame (H100, tools/quality_probe.py)
  // searches took 2-13 rounds: four hold the 45 dB 5/3 search and every 9/7 one there
  enum { RQ_GRAPH_ROUNDS = 4 };
  std::vector<std::vector<JobGroup>> rq_jobs;
  DeviceBuf d_rq, d_rcoef, d_rimg, d_rq_jobs;
  PinnedBuf h_rq;                      // RqState of the last frame
  RqImage rq_image;
  cudaEvent_t rq_ev[3] = {nullptr, nullptr, nullptr};
  float rq_ms[3] = {0, 0, 0};          // last frame: candidates, rounds, final block coding
  void set_target_mse(double mse);
  void check_target_mse() const;
  void plan_quality();
  bool rq_on() const { return target_mse > 0; }
  // Transcoding: the encoder configured from a codestream's headers and tile-parts (transcode_headers), and every
  // frame re-coded from that codestream's code-blocks (transcode), single-layer and cleanup-only, to the encoder's
  // target.  A parse-only decoder (no arena, image or synthesis jobs of its own) reads the input; its block decoders
  // write the coded sign-magnitude words (DEC_OUT_CODED) into d_coef, whose band planes sit where the decoder's do
  // when the output keeps the input's geometry (one Layout of one parameter set).  d_xblocks is the frame's block
  // array: block b at p = q_b, the lowest plane the input codes it down to (31: left out), so candidate k = 0 re-codes
  // exactly the input's bits; rate control and the block coder read it in place of d_blocks.  With a quality target the
  // source is the input decoded as the decoder would, into d_rcoef and through rq_jobs into d_image, which exists only
  // then.
  //
  // With xc_skip = r > 0 the output is the input with its top r resolution levels dropped (reduce_main_header derives
  // its main header and parameters).  The parse-only decoder then reads the input restricted to (r, r): the dropped
  // resolutions' blocks are marked skip and neither uploaded nor decoded.  The two sides number their blocks and lay out
  // their arenas differently (see plan_block_map): d_xmap gives the input's block behind each of the encoder's, and
  // d_xproto holds the input's block prototypes with each kept block's words sent to the encoder's band planes.
  std::unique_ptr<Decoder> src;
  bool transcoding = false;
  bool xc_two_pass = false;            // the frame has SigProp-without-MagRef blocks: k = 0 is not the source
  DeviceBuf d_xblocks;
  PinnedBuf h_xdyn;                    // the source decode's block records (the coded decode's sit in src->h_dyn)
  const uint8_t* xc_cs = nullptr;      // the input on the device
  BlockFrame xc_coded, xc_source;      // the frame's two block decodes (the source: with a quality target only)
  uint32_t xc_skip = 0;                // resolution levels the output drops
  std::vector<uint8_t> xc_in_header;   // the input's main header (less TLM / PLM) this configuration was derived from
  DeviceBuf d_xmap, d_xproto;          // xc_skip > 0 only
  void transcode_headers(const uint8_t* j2c, size_t len, bool on_device, uint32_t sample_type, uint32_t skipped_res = 0);
  size_t transcode(const uint8_t* j2c, size_t len, bool on_device, uint8_t* out, size_t out_cap, bool out_on_device);
  void transcode_parse(const uint8_t* j2c, size_t len, bool on_device, uint32_t sample_type, uint32_t skipped_res);
  void plan_block_map();
  void enqueue_transcode_front();
};

struct FrameInfo {
  uint32_t width, height, off_x, off_y, num_comps;
  uint32_t bit_depth[16], is_signed[16], dx[16], dy[16], comp_w[16], comp_h[16];
  uint32_t num_decomps, reversible, color_transform, num_tiles;
  uint32_t nlt_type[16];
};

// block-encoder variants, identical results: the thread-per-block family by default (blocks of the common shape
// split over two threads), OJB_BLOCK_ENCODER=warp selects one warp per block.
bool serial_block_encoder();

class Decoder : public CodecBase {
public:
  bool resilient = false;
  // parse main header; (re)builds geometry when parameters changed
  void read_headers(const uint8_t* j2c, size_t len, uint32_t sample_type);
  // the same for a codestream that is in DEVICE memory only (complete, with >= 32 readable bytes after its end):
  // the marker segments and packet headers the host parsers touch are fetched page by page into a pinned mirror
  void read_headers_device(const uint8_t* dev_j2c, size_t len, uint32_t sample_type);
  struct Mirror : HostMirror {
    Decoder* owner = nullptr; const uint8_t* dev = nullptr; PinnedBuf host; size_t fetched_bytes = 0;
    std::vector<size_t> last_pages;     // pages the previous frame's parse needed
    void fetch(size_t first_page, size_t npages) override;
  } mirror;
  bool mirrored = false;                // j2c points into mirror.host
  // after read_headers, before decode: rebuilds the output planes and the synthesis schedule
  void restrict_resolution(uint32_t skipped_res_for_read, uint32_t skipped_res_for_recon);
  void setup_geometry(uint32_t sample_type);
  std::vector<uint8_t> block_res;       // per block: how many resolutions lie above its own (D_c - r)
  std::vector<uint8_t> block_wanted;    // with a tile mask: the block belongs to one of this object's tiles
  void info(FrameInfo& fi) const;
  // decode into host planes, into d_image (planes == nullptr) or into the caller's device memory (caller_image:
  // described by use_caller_image); returns number of code-blocks that failed to decode
  uint32_t decode(void* const* planes, const uint32_t* strides, bool caller_image);
  uint32_t failed_blocks = 0;
  const uint8_t* j2c = nullptr; size_t j2c_len = 0; size_t first_sot = 0;
  const uint8_t* dev_cs = nullptr;     // optional: the same bytes already resident in HBM (+32 bytes slack)
  std::vector<uint8_t> header_sig;     // bytes of the main header the geometry was built for
  std::vector<CodedBlock> coded;
  std::vector<DecBlock> h_dec_proto;   // geometry part of DecBlock, per block
  // what the per-frame record loop of decode() needs of it: static flags, K_max, and whether the block's shape
  // qualifies for ht_decode_split_kernel (dec_block_is_fast minus the frame's fields)
  struct DecStatic { uint8_t flags = 0, K_max = 0, fast_shape = 0, pad = 0; };
  std::vector<DecStatic> block_static;
  DeviceBuf d_cs, d_dec, d_proto, d_scratch, d_bstatus;
  PinnedBuf h_dyn, h_bstatus;
  bool any_rev_blocks = false, any_irv_blocks = false;
  uint32_t native_out() const {
    return (any_rev_blocks && any_irv_blocks) ? (uint32_t)DEC_OUT_PER_BLOCK : any_irv_blocks ? (uint32_t)DEC_OUT_FLOAT : (uint32_t)DEC_OUT_INT;
  }
  void parse_tiles();
  // what parse_tiles saw of the tile-parts: per tile, the packet each tile-part starts with; tile-part header segments
  // (bit 0: other than PLT, bit 1: PPT or POC)
  std::vector<std::vector<uint32_t>> tp_starts;
  std::vector<uint32_t> pkts_read;     // per tile: packets parsed
  uint32_t tp_segments = 0;
  // the transcoder's parse (Encoder::transcode_headers): read_headers allocates no coefficient arena, image, synthesis
  // jobs or refinement scratch (enqueue_blocks reserves the scratch when a frame has refinement passes)
  bool parse_only = false;
  size_t scratch_words = 0;
  // the transcoder's block prototypes when its output lays out the kept blocks elsewhere (null: d_proto)
  const DecBlock* out_proto = nullptr;
  // the block records of the parsed frame into hy, for the output mode dec_out; the block decoders of those records
  // into the arena coef on stream st (launches counted)
  BlockFrame frame_records(uint32_t dec_out, DecDyn* hy);
  void enqueue_blocks(const BlockFrame& f, const DecDyn* hy, const uint8_t* cs, uint32_t* coef, cudaStream_t st,
                      const SideStream* sd, uint32_t& launches);
};


template <typename F> void CodecBase::run_frame(const std::vector<uint64_t>& key, F&& enqueue) {
#ifdef OJB_EMU_BUILD
  (void)key; enqueue();
#else
  static const bool disabled = [] { const char* e = getenv("OJB_NO_GRAPHS"); return e && *e && *e != '0'; }();
  FrameGraph& g = fgraph;
  if (disabled || g.off) { enqueue(); return; }
  if (g.exec && g.key == key) {
    if (cudaGraphLaunch(g.exec, stream) == cudaSuccess) { last_launches += g.launches; return; }
    cudaGetLastError(); drop_graph(); g.off = true; enqueue(); return;
  }
  if (g.seen != key) { g.seen = key; enqueue(); return; }       // first sight of this argument set: eager
  drop_graph();
  if (cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); g.off = true; enqueue(); return; }
  const uint32_t l0 = last_launches;
  cudaGraph_t graph = nullptr;
  capturing = true;
  try { enqueue(); } catch (...) { capturing = false; cudaStreamEndCapture(stream, &graph); if (graph) cudaGraphDestroy(graph); cudaGetLastError(); g.off = true; throw; }
  capturing = false;
  g.launches = last_launches - l0;
  cudaError_t rc = cudaStreamEndCapture(stream, &graph);
  if (rc == cudaSuccess) rc = cudaGraphInstantiate(&g.exec, graph, 0);
  if (graph) cudaGraphDestroy(graph);
  if (rc == cudaSuccess) rc = cudaGraphLaunch(g.exec, stream);
  if (rc != cudaSuccess) {          // whatever the capture could not take: this object stays eager
    cudaGetLastError(); drop_graph(); g.off = true; last_launches = l0; enqueue(); return;
  }
  g.key = key;
#endif
}

} // namespace ojb
