// ojb_codec.cpp -- host orchestration of the GPU HTJ2K path (see ojb_codec.h).
#include "ojb_codec.h"
#include "ht_tables.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <chrono>
#include <atomic>
#include <thread>

namespace ojb {

void cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) fail(0x000B00C0, "CUDA failure in %s: %s", what, cudaGetErrorString(e));
}
#define CK(x) cuda_check((x), #x)

DeviceBuf::~DeviceBuf() { if (p) cudaFree(p); }
void DeviceBuf::reserve(size_t n) {
  if (n <= cap) return;
  if (p) { cudaFree(p); p = nullptr; cap = 0; }
  size_t want = (n + 255) & ~(size_t)255;
  CK(cudaMalloc(&p, want));
  cap = want;
}
PinnedBuf::~PinnedBuf() { if (p) cudaFreeHost(p); }
void PinnedBuf::reserve(size_t n) {
  if (n <= cap) return;
  if (p) { cudaFreeHost(p); p = nullptr; cap = 0; }
  size_t want = (n + 4095) & ~(size_t)4095;
  CK(cudaMallocHost(&p, want));
  cap = want;
}

bool serial_block_encoder() {
  static const bool v = [] { const char* e = getenv("OJB_BLOCK_ENCODER"); return !(e && strcmp(e, "warp") == 0); }();
  return v;
}

CodecBase::CodecBase() {
  CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&side.st, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&side.fork, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&side.join, cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ev_caller, cudaEventDisableTiming));
  unsigned hc = std::thread::hardware_concurrency();
  host_threads = hc == 0 ? 4u : std::min(8u, hc);
  for (int i = 0; i < EV_MAX; ++i) CK(cudaEventCreate(&ev[i]));
}
void CodecBase::drop_graph() {
#ifndef OJB_EMU_BUILD
  if (fgraph.exec) { cudaGraphExecDestroy(fgraph.exec); fgraph.exec = nullptr; }
#endif
  fgraph.key.clear();
}
CodecBase::~CodecBase() {
  drop_graph();
  for (int i = 0; i < EV_MAX; ++i) if (ev[i]) cudaEventDestroy(ev[i]);
  if (side.fork) cudaEventDestroy(side.fork);
  if (side.join) cudaEventDestroy(side.join);
  if (ev_caller) cudaEventDestroy(ev_caller);
  if (side.st) cudaStreamDestroy(side.st);
  if (stream) cudaStreamDestroy(stream);
}

void upload_ht_tables(bool enc, DeviceBuf& dev) {
  const HtTables& t = ht_tables();
  std::vector<uint16_t> w(enc ? 2 * 2048 + 36 : 1024 * 2 + 320 + 256, 0);
  if (enc) {
    memcpy(w.data(), t.enc_vlc, sizeof(t.enc_vlc));
    memcpy(w.data() + 2 * 2048, t.enc_uvlc, sizeof(t.enc_uvlc));
  } else {
    memcpy(w.data(), t.dec_vlc, sizeof(t.dec_vlc));
    memcpy(w.data() + 2048, t.dec_uvlc0, sizeof(t.dec_uvlc0));
    memcpy(w.data() + 2048 + 320, t.dec_uvlc1, sizeof(t.dec_uvlc1));
  }
  dev.reserve(w.size() * 2);
  CK(cudaMemcpy(dev.p, w.data(), w.size() * 2, cudaMemcpyHostToDevice));
}

void CodecBase::upload_tables() {
  upload_ht_tables(true, d_tables_enc);
  upload_ht_tables(false, d_tables_dec);
}

void CodecBase::plan_image(uint32_t sample_type, bool alloc) {
  img_type = sample_type;
  uint32_t nc = params.num_comps();
  img_off.assign(nc, 0); img_w.assign(nc, 0); img_h.assign(nc, 0);
  size_t off = 0;
  for (uint32_t c = 0; c < nc; ++c) {
    if (sample_type == ST_U8 && params.comps[c].bit_depth > 8)
      fail(0x000B0010, "8-bit sample container with %d-bit component", params.comps[c].bit_depth);
    if (sample_type == ST_U16 && params.comps[c].bit_depth > 16)
      fail(0x000B0010, "16-bit sample container with %d-bit component", params.comps[c].bit_depth);
    if (sample_type != ST_I32 && params.comps[c].is_signed)
      fail(0x000B0011, "signed components need the 32-bit sample container");
    // reconstruction size: sub-sampling times 2^skip_recon (param_siz::get_recon_width, ojph_params.cpp)
    uint32_t fx, fy; params.res_downsamp(c, skip_recon, fx, fy);   // 2^skip_recon both ways unless a DFS says otherwise (get_recon_downsampling, :931-944)
    const uint32_t rdx = params.comps[c].dx * fx, rdy = params.comps[c].dy * fy;
    img_w[c] = div_ceil(params.Xsiz, rdx) - div_ceil(params.XOsiz, rdx);
    img_h[c] = div_ceil(params.Ysiz, rdy) - div_ceil(params.YOsiz, rdy);
    img_off[c] = off;
    off += (size_t)img_w[c] * img_h[c] * esize_of(sample_type);
    off = (off + 255) & ~(size_t)255;
  }
  img_bytes = off + 256;
  if (alloc) d_image.reserve(img_bytes);
  if (nc > IMG_SLOTS) fail(0x000B0008, "%u components: the frame interface carries at most %u", nc, (uint32_t)IMG_SLOTS);
  std::vector<ImgComp> own(IMG_SLOTS);
  for (uint32_t c = 0; c < nc; ++c) {
    own[c].base = alloc ? (uint64_t)(size_t)(d_image.as<uint8_t>() + img_off[c]) : 0;
    own[c].pitch = (uint64_t)img_w[c] * esize_of(sample_type); own[c].col = 1; own[c].pad = 0;
  }
  d_img.reserve(3 * IMG_SLOTS * sizeof(ImgComp));
  h_img.reserve(IMG_SLOTS * sizeof(ImgComp));
  CK(cudaMemcpy(d_img.p, own.data(), IMG_SLOTS * sizeof(ImgComp), cudaMemcpyHostToDevice));
}

void CodecBase::use_caller_image(const ImgComp* comps, cudaStream_t caller_stream) {
  const uint32_t nc = params.num_comps(), es = esize_of(img_type);
  memcpy(h_img.p, comps, (size_t)nc * sizeof(ImgComp));
  caller_interleaved = false;
  if (nc >= 3 && (comps[0].col == 3 || comps[0].col == 4)) {
    bool adj = true;
    for (uint32_t k = 1; k < 3; ++k)
      adj = adj && comps[k].base == comps[0].base + k * es && comps[k].pitch == comps[0].pitch && comps[k].col == comps[0].col;
    caller_interleaved = adj;
  }
  CK(cudaEventRecord(ev_caller, caller_stream));
  CK(cudaStreamWaitEvent(stream, ev_caller, 0));
}
void CodecBase::enqueue_caller_image() {
  launch_ctrl_copy(const_cast<ImgComp*>(img_slot(true)), h_img.p, (size_t)params.num_comps() * sizeof(ImgComp), stream);
  ++last_launches;
}

// the register-streaming kernels take a level when it splits both ways with the built-in 5/3 or 9/7, the resolution is
// at least 2 x 2 and byte / word offsets fit 32 bits (dwt_stream.cu)
static bool level_streams(const CodecBase& C, const Params& P, uint32_t c, const ResGeom& rg) {
  return !C.wide && rg.hsplit && rg.vsplit && P.wavelet_of(c) <= 1 && rg.rect.w >= 2 && rg.rect.h >= 2 && !C.no_stream_dwt &&
         C.layout.coef_words < (1ull << 30) && C.img_bytes < (1ull << 32);
}

// slab g of `world` of a tile-component: rows [lo, hi) in absolute component coordinates; inner boundaries on multiples
// of 128 rows (two code-block rows of the first level, whole row chunks of the kernels)
CodecBase::RowSpan CodecBase::region_slab(const Rect& tc, uint32_t g, uint32_t world) {
  // OJB_REGION_ALIGN (a power of two; tests): finer slab boundaries, so that small images are cut as well
  static const uint64_t align = [] {
    const char* e = getenv("OJB_REGION_ALIGN");
    uint64_t a = e ? strtoull(e, nullptr, 10) : 128;
    return (a >= 2 && (a & (a - 1)) == 0) ? a : (uint64_t)128;
  }();
  auto bound = [&](uint32_t i) -> uint32_t {
    if (i == 0) return tc.y0;
    if (i >= world) return tc.y1();
    const uint64_t y = (uint64_t)tc.y0 + (uint64_t)tc.h * i / world;
    return std::min(std::max((uint32_t)(y & ~(align - 1)), tc.y0), tc.y1());
  };
  RowSpan s; s.lo = bound(g); s.hi = bound(g + 1);
  return s;
}

// Row-region sharding (see ojb_codec.h): block ownership, the window of row chunks every level's job runs, the
// blocks a decoder has to decode and the image rows read / delivered -- all from the geometry, identically on
// every rank.  What a chunk [R0, R1) of the streaming kernels reads (dwt_stream.cu): analysis, source rows
// [R0 - m, R1 + m); synthesis, interleaved band rows [R0 - m, R1 + m + 1) (even: a low-pass row, odd: a
// high-pass row, index >> 1); m = 2 for 5/3, 4 for 9/7, mirrored at the resolution's own borders only.
void CodecBase::plan_region(bool forward) {
  const Params& P = params;
  const uint32_t nc = P.num_comps(), W = region.world, me = region.rank;
  region_win.assign(layout.tiles.size(), std::vector<std::vector<RegionWin>>());
  region_rows.assign(layout.tiles.size(), std::vector<RowSpan>());
  region_owner.assign(layout.num_blocks, 0);
  region_blocks.assign(layout.num_blocks, 0);
  struct Span { int64_t lo = INT64_MAX, hi = INT64_MIN; bool empty() const { return lo >= hi; }
                void add(int64_t a, int64_t b) { if (a < b) { lo = std::min(lo, a); hi = std::max(hi, b); } } };
  for (const TileGeom& t : layout.tiles) {
    region_win[t.idx].assign(nc, std::vector<RegionWin>());
    region_rows[t.idx].assign(nc, RowSpan());
    for (uint32_t c = 0; c < nc; ++c) {
      const TileCompGeom& tc = t.comps[c];
      const uint32_t D = (uint32_t)tc.res.size() - 1;
      region_win[t.idx][c].assign(D + 1, RegionWin());
      bool streams = D >= 1;
      for (uint32_t r = 1; r <= D && streams; ++r) streams = level_streams(*this, P, c, tc.res[r]);
      // block ownership: by the slab the block's first row falls into, scaled up to the component's resolution
      for (uint32_t r = 0; r <= D; ++r)
        for (uint32_t b = 0; b < 4; ++b) {
          const BandGeom& bg = tc.res[r].bands[b];
          if (bg.empty) continue;
          const uint32_t depth = r ? D - r + 1 : D;
          for (uint32_t by = 0; by < bg.nbh; ++by) {
            const Rect br = bg.block_rect(0, by);
            const uint64_t yf = std::min<uint64_t>(std::max<uint64_t>((uint64_t)br.y0 << depth, tc.rect.y0), tc.rect.y1() ? tc.rect.y1() - 1 : 0);
            uint32_t g = 0;
            while (g + 1 < W && yf >= region_slab(tc.rect, g, W).hi) ++g;
            for (uint32_t bx = 0; bx < bg.nbw; ++bx) {
              region_owner[bg.block_base + by * bg.nbw + bx] = (uint8_t)g;
              if (forward) region_blocks[bg.block_base + by * bg.nbw + bx] = g == me ? 1 : 0;
            }
          }
        }
      // rows of band b of resolution r spanned by the blocks this rank owns (encoder)
      auto owned_rows = [&](uint32_t r, uint32_t b) {
        Span s; const BandGeom& bg = tc.res[r].bands[b];
        if (bg.empty) return s;
        for (uint32_t by = 0; by < bg.nbh; ++by)
          if (region_owner[bg.block_base + by * bg.nbw] == me) { const Rect br = bg.block_rect(0, by); s.add(br.y0, br.y1()); }
        return s;
      };
      auto want_rows = [&](uint32_t r, uint32_t b, const Span& rows) {      // decoder: blocks of the band that meet the rows
        const BandGeom& bg = tc.res[r].bands[b];
        if (bg.empty || rows.empty()) return;
        for (uint32_t by = 0; by < bg.nbh; ++by) {
          const Rect br = bg.block_rect(0, by);
          if ((int64_t)br.y0 < rows.hi && (int64_t)br.y1() > rows.lo)
            for (uint32_t bx = 0; bx < bg.nbw; ++bx) region_blocks[bg.block_base + by * bg.nbw + bx] = 1;
        }
      };
      const RowSpan slab = region_slab(tc.rect, me, W);
      if (!streams) {
        // whole-plane transforms on every rank; the decoder then needs every block of the component
        if (forward) { region_rows[t.idx][c].lo = tc.rect.y0; region_rows[t.idx][c].hi = tc.rect.y1(); }
        else {
          region_rows[t.idx][c] = slab;
          for (uint32_t r = 0; r <= D; ++r) for (uint32_t b = 0; b < 4; ++b) { Span all; all.add(0, INT64_MAX); want_rows(r, b, all); }
        }
        continue;
      }
      const uint32_t m = P.reversible(c) ? 2u : 4u;
      // rows [lo, hi) of resolution r that have to be produced -> the chunks that do it and what they read
      auto chunks_for = [&](uint32_t r, Span out, RegionWin& w, Span& read) {
        const ResGeom& rg = tc.res[r];
        const int64_t y0 = rg.rect.y0, y1 = rg.rect.y1(), ye = y0 & ~(int64_t)1;
        out.lo = std::max(out.lo, y0); out.hi = std::min(out.hi, y1);
        w.full = false; w.chunk0 = 0; w.nchunks = 0; read = Span();
        if (out.empty()) return;
        uint32_t strips, chunks, cr, ctas;
        dwt_stream_tiling(rg.rect.x0, rg.rect.y0, rg.rect.w, rg.rect.h, P.reversible(c), forward, strips, chunks, cr, ctas);
        const int64_t c_lo = (out.lo - ye) / cr, c_hi = (out.hi - 1 - ye) / cr;
        w.chunk0 = (uint32_t)c_lo; w.nchunks = (uint32_t)(c_hi - c_lo + 1);
        const int64_t R0 = ye + c_lo * cr, R1 = std::min<int64_t>(ye + (c_hi + 1) * cr, y1);
        read.add(std::max(y0, R0 - (int64_t)m), std::min(y1, R1 + (int64_t)m + (forward ? 0 : 1)));
      };
      if (forward) {
        Span low = owned_rows(0, 0);                          // rows of resolution r - 1 this rank needs
        for (uint32_t r = 1; r <= D; ++r) {
          Span out;
          if (!low.empty()) out.add(2 * low.lo, 2 * (low.hi - 1) + 1);
          { const Span s = owned_rows(r, 1); if (!s.empty()) out.add(2 * s.lo, 2 * (s.hi - 1) + 1); }
          for (uint32_t b = 2; b < 4; ++b) { const Span s = owned_rows(r, b); if (!s.empty()) out.add(2 * s.lo + 1, 2 * (s.hi - 1) + 2); }
          Span read;
          chunks_for(r, out, region_win[t.idx][c][r], read);
          low = read;
        }
        if (!low.empty()) { region_rows[t.idx][c].lo = (uint32_t)low.lo; region_rows[t.idx][c].hi = (uint32_t)low.hi; }
      } else {
        region_rows[t.idx][c] = slab;
        Span out; out.add(slab.lo, slab.hi);
        for (uint32_t r = D; r >= 1; --r) {
          Span read;
          chunks_for(r, out, region_win[t.idx][c][r], read);
          Span bandrows;
          if (!read.empty()) bandrows.add(read.lo >> 1, ((read.hi - 1) >> 1) + 1);
          for (uint32_t b = 1; b < 4; ++b) want_rows(r, b, bandrows);
          out = bandrows;
        }
        want_rows(0, 0, out);
      }
    }
    // the colour transform fuses the first three components into one job at the top level: one window for the three
    if (P.color_transform() && nc >= 3) {
      const uint32_t D = (uint32_t)t.comps[0].res.size() - 1;
      RegionWin& a = region_win[t.idx][0][D];
      if (D >= 1 && !a.full) {
        uint32_t lo = UINT32_MAX, hi = 0;
        for (uint32_t c = 0; c < 3; ++c) {
          const RegionWin& w = region_win[t.idx][c][D];
          if (w.nchunks) { lo = std::min(lo, w.chunk0); hi = std::max(hi, w.chunk0 + w.nchunks); }
        }
        for (uint32_t c = 0; c < 3; ++c) { RegionWin& w = region_win[t.idx][c][D]; w.chunk0 = lo < hi ? lo : 0; w.nchunks = lo < hi ? hi - lo : 0; }
        if (forward) {
          uint32_t rl = UINT32_MAX, rh = 0;
          for (uint32_t c = 0; c < 3; ++c) if (region_rows[t.idx][c].hi > region_rows[t.idx][c].lo) { rl = std::min(rl, region_rows[t.idx][c].lo); rh = std::max(rh, region_rows[t.idx][c].hi); }
          for (uint32_t c = 0; c < 3; ++c) { region_rows[t.idx][c].lo = rl < rh ? rl : 0; region_rows[t.idx][c].hi = rl < rh ? rh : 0; }
        }
      }
    }
  }
}

void CodecBase::build_dwt_jobs(bool forward, std::vector<std::vector<JobGroup>>& jobs, DeviceBuf& d_jobs) {
  const Params& P = params;
  drop_graph(); fgraph.seen.clear();       // a new geometry: whatever was captured launched the old job lists
  if (region.on()) {
    if (!tile_mask.empty()) fail(0x000B0045, "a tile mask and row regions cannot be combined");
    if (skip_read || skip_recon) fail(0x000B0046, "reduced-resolution decoding is not available with row regions");
    plan_region(forward);
  } else { region_win.clear(); region_rows.clear(); region_owner.clear(); region_blocks.clear(); }
  const uint32_t nc = P.num_comps();
  // level li counts decompositions from the full resolution down; every component follows its own
  // coding style (COC): component c takes part in levels li < max(1, D_c) with resolution D_c - li
  uint32_t nlev = forward ? 1u : skip_recon + 1;
  for (uint32_t c = 0; c < nc; ++c) nlev = std::max(nlev, P.decomps(c));
  if (P.color_transform())
    for (uint32_t c = 1; c < 3; ++c)
      if (P.decomps(c) != P.decomps(0) || P.wavelet_of(c) != P.wavelet_of(0) || P.dfs_of(c) != P.dfs_of(0))
        fail(0x000B0006, "the colour transform needs one coding style for the first three components");
  jobs.assign(nlev, std::vector<JobGroup>());
  for (uint32_t li = 0; li < nlev; ++li) {
    // groups per wavelet w (0: 5/3, 1: 9/7): [4w+0] streaming 3-comp first, [4w+1] streaming 1-comp first,
    // [4w+2] streaming inner levels, [4w+3] general
    std::vector<JobGroup> grp(8);
    for (uint32_t w = 0; w < 2; ++w) {
      grp[4 * w].stream = grp[4 * w + 1].stream = grp[4 * w + 2].stream = true;
      grp[4 * w].ncomp = 3; grp[4 * w].first = grp[4 * w + 1].first = true;
      for (uint32_t i = 0; i < 4; ++i) grp[4 * w + i].reversible = (w == 0);
    }
    for (const TileGeom& t : layout.tiles) {
      if (!tile_wanted(t.idx)) continue;
      for (uint32_t c = 0; c < nc; ) {
        const uint32_t D = P.decomps(c);
        // levels above `top` are not run (decoder with restrict_resolution: reduced output); a component
        // with nothing to split / rebuild (D == 0, or its whole pyramid skipped) is a plain conversion of LL
        const uint32_t top = forward ? 0u : skip_recon;
        const bool conv_only = D <= top;
        const bool here = conv_only ? (li == top) : (li >= top && li < D);
        const bool is_top = li == top;
        bool fused = P.color_transform() && c == 0 && is_top;
        uint32_t k = fused ? 3 : 1;
        if (!here) { ++c; continue; }
        const uint32_t r = conv_only ? 0 : D - li;               // resolution being split (or rebuilt)
        const bool rev = P.reversible(c);
        const uint32_t gw = rev ? 0u : 4u;
        DwtJob j; memset(&j, 0, sizeof(j));
        const ResGeom& rg = t.comps[c].res[r];
        j.w = rg.rect.w; j.h = rg.rect.h; j.x0 = rg.rect.x0; j.y0 = rg.rect.y0;
        j.ncomp = k; j.first = is_top ? 1u : 0u; j.last = (r <= 1) ? 1u : 0u;
        // which way this level lifts (one way only, or not at all, under a DFS marker segment) and with which kernel
        j.hsplit = conv_only ? 0u : rg.hsplit; j.vsplit = conv_only ? 0u : rg.vsplit;
        j.nodwt = (j.hsplit | j.vsplit) ? 0u : 1u;
        {
          const AtkSpec& kern = P.atk_of(c);
          if (kern.steps.size() > DWT_MAX_STEPS)
            fail(0x000B0025, "transformation kernels with more than %d lifting steps are not built (this one has %d)",
                 DWT_MAX_STEPS, (int)kern.steps.size());
          j.nsteps = (uint32_t)kern.steps.size(); j.K = kern.K;
          for (uint32_t i = 0; i < j.nsteps; ++i) {
            j.step_A[i] = kern.steps[i].A; j.step_a[i] = kern.steps[i].a; j.step_b[i] = kern.steps[i].b; j.step_e[i] = kern.steps[i].e;
          }
        }
        j.src_type = img_type; j.bit_depth = P.comps[c].bit_depth; j.is_signed = P.comps[c].is_signed ? 1u : 0u;
        if (is_top && P.nlt_any())             // the type-3 map only touches signed samples (ojph_tile.cpp:352, 446)
          for (uint32_t i = 0; i < k; ++i)
            if (P.comps[c + i].is_signed && P.nlt_type(c + i) == 3) j.nlt_mask |= 1u << i;
        for (uint32_t i = 0; i < k; ++i) {
          const TileCompGeom& tc = t.comps[c + i];
          const ResGeom& rr = tc.res[r];
          if (is_top) {
            // the resolution's rectangle sits at (ceil(x0 / 2^s) - ceil(XO / (dx 2^s))) in the output plane
            uint32_t fx, fy; P.res_downsamp(c + i, top, fx, fy);
            uint32_t cx0 = div_ceil(P.XOsiz, P.comps[c + i].dx * fx), cy0 = div_ceil(P.YOsiz, P.comps[c + i].dy * fy);
            j.img_comp[i] = c + i; j.img_x[i] = rr.rect.x0 - cx0; j.img_y[i] = rr.rect.y0 - cy0;
          } else { j.full_off[i] = rr.plane_off; j.full_stride[i] = rr.plane_stride; }
          if (r > 0) {
            const ResGeom& lo = tc.res[r - 1];
            j.ll_off[i] = lo.plane_off; j.ll_stride[i] = lo.plane_stride;
            for (uint32_t b = 1; b < 4; ++b) {
              const BandGeom& bg = rr.bands[b];
              if (((b & 1) && !rr.hsplit) || ((b >> 1) && !rr.vsplit)) continue;       // no such band at this level
              j.band_off[i][b] = bg.plane_off + bg.plane_pad_x; j.band_stride[i][b] = bg.plane_stride;
              j.band_shift[i][b] = (wide ? 63u : 31u) - bg.K_max;
              j.band_scale[i][b] = forward ? bg.delta_inv : bg.delta;
            }
            if (r == 1) {
              const BandGeom& bg = lo.bands[0];
              j.band_off[i][0] = bg.plane_off + bg.plane_pad_x; j.band_stride[i][0] = bg.plane_stride;
              j.band_shift[i][0] = (wide ? 63u : 31u) - bg.K_max;
              j.band_scale[i][0] = forward ? bg.delta_inv : bg.delta;
            }
          } else {   // zero decomposition levels
            const BandGeom& bg = rr.bands[0];
            j.band_off[i][0] = bg.plane_off + bg.plane_pad_x; j.band_stride[i][0] = bg.plane_stride;
            j.band_shift[i][0] = (wide ? 63u : 31u) - bg.K_max;
            j.band_scale[i][0] = forward ? bg.delta_inv : bg.delta;
          }
        }
        const bool stream = !j.nodwt && level_streams(*this, P, c, rg);   // 32-bit byte offsets in the stream kernels
        uint32_t gi, n;
        if (stream) {
          gi = gw + (j.first ? (k == 3 ? 0u : 1u) : 2u);
          dwt_stream_tiling(j.x0, j.y0, j.w, j.h, rev, forward, j.tiles_x, j.tiles_y, j.chunk_rows, n);
          if (region.on() && !conv_only && !region_win[t.idx][c][r].full) {      // this rank's window of row chunks
            const RegionWin& rw = region_win[t.idx][c][r];
            const uint32_t per_row = j.tiles_y ? n / j.tiles_y : 0;
            j.chunk0 = rw.chunk0; j.tiles_y = rw.nchunks; n = per_row * rw.nchunks;
          }
        } else {
          gi = gw + 3;
          dwt_tiling(j.x0, j.y0, j.w, j.h, j.tiles_x, j.tiles_y);
          n = j.tiles_x * j.tiles_y;
          grp[gi].ncomp = std::max(grp[gi].ncomp, k);
        }
        j.cta_base = grp[gi].ctas;
        if (n) { grp[gi].ctas += n; grp[gi].jobs.push_back(j); }
        c += k;
      }
    }
    for (JobGroup& g : grp) if (!g.jobs.empty()) jobs[li].push_back(g);
  }
  size_t total = 0;
  for (auto& lv : jobs) for (JobGroup& g : lv) { g.dev_off = total; total += g.jobs.size(); }
  d_jobs.reserve(std::max<size_t>(1, total) * sizeof(DwtJob));
  for (auto& lv : jobs) for (JobGroup& g : lv)
    CK(cudaMemcpy(d_jobs.as<DwtJob>() + g.dev_off, g.jobs.data(), g.jobs.size() * sizeof(DwtJob), cudaMemcpyHostToDevice));
}

void CodecBase::enqueue_dwt(bool forward, const std::vector<std::vector<JobGroup>>& groups, DeviceBuf& dev,
                            const ImgComp* img, bool interleaved, uint32_t* coef) {
  for (size_t i = 0; i < groups.size(); ++i)
    for (const JobGroup& g : groups[forward ? i : groups.size() - 1 - i]) {
      const DwtJob* j = dev.as<DwtJob>() + g.dev_off;
      const uint32_t n = (uint32_t)g.jobs.size();
      if (forward && g.stream)
        launch_dwt_fwd_stream(j, n, g.ctas, g.reversible, g.ncomp, g.first, img_type, img, interleaved, coef, stream);
      else if (forward)
        launch_dwt_fwd(j, n, g.ctas, g.reversible, g.ncomp, img, coef, stream, wide);
      else if (g.stream)
        launch_dwt_inv_stream(j, n, g.ctas, g.reversible, g.ncomp, g.first, img_type, img, interleaved, coef, stream);
      else
        launch_dwt_inv(j, n, g.ctas, g.reversible, g.ncomp, img, coef, stream, wide);
      ++last_launches;
    }
}

// widest nominal code-block; blocks wider than 64 samples go through the thread-per-block kernels
// (the warp-per-block kernels keep one quad column per lane)
static uint32_t widest_block(const Layout& L) {
  uint32_t w = 4;
  for (const TileGeom& t : L.tiles)
    for (const TileCompGeom& tc : t.comps)
      for (const ResGeom& rg : tc.res)
        for (uint32_t b = 0; b < 4; ++b)
          if (!rg.bands[b].empty) w = std::max(w, 1u << rg.bands[b].xcb);
  return w;
}

//------------------------------------------------------------------------------------------
// Encoder
//------------------------------------------------------------------------------------------
uint32_t enc_slot_cap(uint32_t w, uint32_t h, uint32_t K_max, bool wide) {
  // worst case: (K_max+1) MagSgn bits / sample (+1/15 stuffing), 30 VLC bits / quad pair
  // (+1/7), 192 MEL bytes, working margin of the kernel
  uint64_t ms = ((uint64_t)w * h * (K_max + 1) + 7) / 8; ms += ms / 15 + 8;
  uint64_t nq = (uint64_t)((w + 1) / 2) * ((h + 1) / 2);
  uint64_t vl = ((nq + 1) / 2 * (wide ? 38 : 30) + 12 + 7) / 8; vl += vl / 7 + 8;      // (+ two 4-bit U-VLC extensions per pair)
  return (uint32_t)((ms + vl + 192 + 160 + 15) & ~(uint64_t)15);
}

void Encoder::configure(const Params& p, uint32_t sample_type) {
  params = p;
  params.finalize_for_encode();
  transcoding = false;
  main_header.clear();
  params.write_main_header(main_header, nullptr, nullptr, 0);
  setup(sample_type);
}

void Encoder::setup(uint32_t sample_type) {
  wide = params.needs_wide();
  if (wide && sample_type != ST_I32) fail(0x000B0010, "samples beyond 16 bits need the 32-bit sample container");
  layout.build(params);
  max_block_w = widest_block(layout);
  plan_image(sample_type, !transcoding);            // a transcoder needs an image only for a quality target (plan_quality)
  upload_tables();
  d_coef.reserve((layout.coef_words + 64) * (wide ? 8 : 4));
  CK(cudaMemset(d_coef.p, 0, d_coef.cap));
  build_dwt_jobs(true, jobs, d_jobs);
  // block descriptors and slots
  h_blocks.assign(layout.num_blocks, EncBlock());
  num_fast_blocks = 0;
  size_t slot = 0;
  for (const TileGeom& t : layout.tiles)
    for (const TileCompGeom& tc : t.comps)
      for (const ResGeom& rg : tc.res)
        for (uint32_t b = 0; b < 4; ++b) {
          const BandGeom& bg = rg.bands[b];
          if (bg.empty) continue;
          for (uint32_t by = 0; by < bg.nbh; ++by)
            for (uint32_t bx = 0; bx < bg.nbw; ++bx) {
              Rect r = bg.block_rect(bx, by);
              EncBlock& e = h_blocks[bg.block_base + by * bg.nbw + bx];
              e.src_off = bg.plane_off + bg.plane_pad_x + (uint64_t)(r.y0 - bg.rect.y0) * bg.plane_stride + (r.x0 - bg.rect.x0);
              e.stride = bg.plane_stride; e.w = (uint16_t)r.w; e.h = (uint16_t)r.h;
              e.p = (uint16_t)((wide ? 63u : 31u) - bg.K_max);
              e.flags = (tc.res.size() == 1 && params.reversible(tc.comp)) ? (uint16_t)ENC_CHECK_NEGZERO : (uint16_t)0;
              e.slot_off = slot; e.slot_cap = enc_slot_cap(r.w, r.h, bg.K_max, wide);
              slot += e.slot_cap;
              if (!tile_wanted(t.idx)) { e.w = e.h = 0; }                  // another rank's tile: nothing to code
              if (region.on() && !region_blocks[bg.block_base + by * bg.nbw + bx]) { e.w = e.h = 0; }   // another rank's rows
              if (!no_fast_blocks && !wide && enc_block_is_fast(e)) { e.flags |= ENC_FLAG_FAST; ++num_fast_blocks; }
            }
        }
  slot_bytes = slot + 64;
  // One rank's share of a sharded image may be a few thousand blocks: one thread per block then leaves most of the
  // device idle for as long as one block's serial chain lasts, and the warp-per-block kernel -- more instructions,
  // a ten times shorter chain -- is faster; with many blocks the thread-per-block kernel wins again.
  // OJB_ENC_WARP_BELOW moves the limit.
  {
    uint32_t coded_blocks = 0;
    for (const EncBlock& e : h_blocks) if (e.w && e.h) ++coded_blocks;
    uint32_t limit = 8192;
    if (const char* e = getenv("OJB_ENC_WARP_BELOW")) limit = (uint32_t)strtoul(e, nullptr, 10);
    few_blocks_warp = (region.on() || !tile_mask.empty()) && coded_blocks > 0 && coded_blocks <= limit && max_block_w <= 64 && !wide;
  }
  d_slots.reserve(slot_bytes);
  d_blocks.reserve(std::max<size_t>(1, h_blocks.size()) * sizeof(EncBlock));
  if (!h_blocks.empty())
    CK(cudaMemcpy(d_blocks.p, h_blocks.data(), h_blocks.size() * sizeof(EncBlock), cudaMemcpyHostToDevice));
  d_results.reserve(std::max<size_t>(1, h_blocks.size()) * sizeof(EncResult));
  h_results.reserve(std::max<size_t>(1, h_blocks.size()) * sizeof(EncResult));
  d_dst.reserve(std::max<size_t>(1, h_blocks.size()) * 8);
  h_dst.reserve(std::max<size_t>(1, h_blocks.size()) * 8);
  d_status.reserve(256); h_status.reserve(256);
  coded.assign(layout.num_blocks, CodedBlock());
  if (transcoding) d_xblocks.reserve(std::max<size_t>(1, h_blocks.size()) * sizeof(EncBlock));
  build_header_plan();
  min_bytes = min_size_of_geometry();
  rc_kc = 0;                           // rate-control tables follow the geometry: planned again on first use
  rq_planned = false;
  // line-based front end state
  line_cur.assign(params.num_comps(), 0); cur_comp = 0; lines_done = false;
}

// The static side of pkt_headers.cu: packets in stream order, their bands with blocks (segments), blocks in header
// order (items), groups of 32 items, tile-parts -- everything that depends on the geometry only.
void Encoder::build_header_plan() {
  device_headers = false; rc_sizing = false;
  memset(&hplan, 0, sizeof(hplan));
  // OJB_HOST_HEADERS=1 keeps the host writer; the plan is still built for rate control, which sizes its selections with it
  const bool host_writer = [] { const char* e = getenv("OJB_HOST_HEADERS"); return e && *e && *e != '0'; }();
  const bool partial = !tile_mask.empty();        // this rank's tile-parts only: no main header, TLM or EOC (ojb_shard.cpp)
  std::vector<HdrSeg> segs; std::vector<HdrPkt> pkts; std::vector<HdrGroup> groups; std::vector<HdrTp> tps; std::vector<uint32_t> item_seg;
  uint64_t nodes = 0, hoff = 0; uint32_t max_cap = 0;
  auto log2ceil = [](uint32_t x) { uint32_t t = 31u - (uint32_t)__builtin_clz(x); return t + ((x & (x - 1)) ? 1u : 0u); };
  fixed_blob.clear();
  if (!partial) fixed_blob = main_header;
  std::vector<PacketRef> seq; std::vector<uint32_t> tp_first, tp_index; uint32_t tp_total = 0;
  struct TpTmp { uint32_t tile, first, count, idx, cnt; };
  std::vector<TpTmp> tpt;
  for (uint32_t t = 0; t < (uint32_t)layout.tiles.size(); ++t) {
    if (!tile_wanted(t)) continue;
    layout.packet_sequence(t, seq, tp_first, &tp_index, &tp_total);
    const uint32_t base = (uint32_t)pkts.size();
    for (const PacketRef& pr : seq) {
      const ResGeom& rg = layout.res_of(pr); const PrecinctGeom& pc = rg.precincts[pr.precinct];
      HdrPkt pk; memset(&pk, 0, sizeof(pk));
      pk.first_seg = (uint32_t)segs.size(); pk.first_item = (uint32_t)item_seg.size(); pk.first_group = (uint32_t)groups.size();
      for (uint32_t sb = 0; sb < 4; ++sb) {
        const BandGeom& bg = rg.bands[sb];
        if (bg.empty) continue;
        const Rect& ci = pc.cb_idx[sb];
        if (ci.w == 0 || ci.h == 0) continue;
        HdrSeg sg; sg.pkt = (uint32_t)pkts.size(); sg.first_item = (uint32_t)item_seg.size();
        sg.w = ci.w; sg.h = ci.h; sg.nl = 1 + std::max(log2ceil(ci.w), log2ceil(ci.h));
        sg.block0 = bg.block_base + ci.y0 * bg.nbw + ci.x0; sg.nbw = bg.nbw; sg.tree_off = (uint32_t)nodes;
        for (uint32_t l = 0, pw = ci.w, ph = ci.h; l < sg.nl; ++l) { nodes += (uint64_t)pw * ph; pw = (pw + 1) >> 1; ph = (ph + 1) >> 1; }
        item_seg.insert(item_seg.end(), (size_t)ci.w * ci.h, (uint32_t)segs.size());
        segs.push_back(sg);
      }
      pk.nsegs = (uint32_t)segs.size() - pk.first_seg; pk.nitems = (uint32_t)item_seg.size() - pk.first_item;
      for (uint32_t i = 0; i < pk.nitems; i += 32) groups.push_back(HdrGroup{ pk.first_item + i, std::min(32u, pk.nitems - i) });
      pk.ngroups = (uint32_t)groups.size() - pk.first_group;
      // <= 160 bits per block, one stuffed bit per eight at worst
      const uint64_t cap = (((uint64_t)pk.nitems * 23 + 16) + 3) & ~(uint64_t)3;
      pk.hdr_off = (uint32_t)hoff; hoff += cap; max_cap = (uint32_t)std::max<uint64_t>(max_cap, cap);
      pkts.push_back(pk);
    }
    for (size_t i = 0; i < tp_first.size(); ++i) {
      const uint32_t end = (i + 1 < tp_first.size()) ? tp_first[i + 1] : (uint32_t)seq.size();
      if (end == tp_first[i]) return;                 // a tile-part without packets: the host writer handles it (no rate control)
      tpt.push_back(TpTmp{ t, base + tp_first[i], end - tp_first[i], tp_index[i], tp_total });
      pkts[base + tp_first[i]].tp_first = 1;
    }
  }
  if (nodes >= (1ull << 32) || hoff >= (1ull << 32) || item_seg.size() >= (1ull << 31)) return;
  const bool tlm = params.need_tlm && !partial;
  if (tlm) {
    if (4 + 6 * tpt.size() > 65535) fail(0x000500B1, "too many tile-parts for one TLM marker segment");
    put_u16(fixed_blob, M_TLM); put_u16(fixed_blob, (uint32_t)(4 + 6 * tpt.size())); put_u8(fixed_blob, 0); put_u8(fixed_blob, 0x60);
    for (const TpTmp& tp : tpt) { put_u16(fixed_blob, tp.tile); put_u32(fixed_blob, 0); }
  }
  h_tp_tile.clear();
  for (const TpTmp& tp : tpt) h_tp_tile.push_back(tp.tile);
  for (size_t i = 0; i < tpt.size(); ++i)
    tps.push_back(HdrTp{ tpt[i].first, tpt[i].count, tpt[i].tile, tpt[i].idx, tpt[i].cnt,
                         tlm ? (uint32_t)(main_header.size() + 6 + 6 * i + 2) : 0xFFFFFFFFu });
  int nb = 0;
  auto up = [&](const void* src, size_t bytes) -> void* {
    DeviceBuf& b = d_hplan[nb++]; b.reserve(std::max<size_t>(16, bytes));
    if (bytes) CK(cudaMemcpy(b.p, src, bytes, cudaMemcpyHostToDevice));
    return b.p;
  };
  auto scratch = [&](size_t bytes) -> void* { DeviceBuf& b = d_hplan[nb++]; b.reserve(std::max<size_t>(16, bytes)); return b.p; };
  hplan.nsegs = (uint32_t)segs.size(); hplan.npkts = (uint32_t)pkts.size(); hplan.nitems = (uint32_t)item_seg.size();
  hplan.ngroups = (uint32_t)groups.size(); hplan.ntps = (uint32_t)tps.size(); hplan.max_hdr_cap = max_cap;
  hplan.segs = (const HdrSeg*)up(segs.data(), segs.size() * sizeof(HdrSeg));
  hplan.pkts = (const HdrPkt*)up(pkts.data(), pkts.size() * sizeof(HdrPkt));
  hplan.groups = (const HdrGroup*)up(groups.data(), groups.size() * sizeof(HdrGroup));
  hplan.tps = (const HdrTp*)up(tps.data(), tps.size() * sizeof(HdrTp));
  hplan.item_seg = (const uint32_t*)up(item_seg.data(), item_seg.size() * 4);
  const size_t ni = item_seg.size(), ng = groups.size(), np = pkts.size();
  hplan.tinc = (uint8_t*)scratch(nodes); hplan.tmm = (uint8_t*)scratch(nodes); hplan.tfi = (uint32_t*)scratch(nodes * 4);
  hplan.seg_root = (uint8_t*)scratch(segs.size());
  hplan.ibits = (uint32_t*)scratch(ni * 20); hplan.inbits = (uint16_t*)scratch(ni * 2); hplan.itab = (uint16_t*)scratch(ni * 32);
  hplan.ilen = (uint32_t*)scratch(ni * 4);
  hplan.gcomp = (uint32_t*)scratch(ng * 64); hplan.gbits = (uint32_t*)scratch(ng * 4); hplan.glen = (uint32_t*)scratch(ng * 4);
  hplan.gstate = (uint32_t*)scratch(ng * 4); hplan.gpos = (uint32_t*)scratch(ng * 4); hplan.gbody = (uint32_t*)scratch(ng * 4);
  hplan.istate = (uint8_t*)scratch(ni); hplan.ipos = (uint32_t*)scratch(ni * 4); hplan.ibody = (uint32_t*)scratch(ni * 4);
  hplan.phdr = (uint32_t*)scratch(np * 4); hplan.pbody = (uint32_t*)scratch(np * 4); hplan.ppos = (uint64_t*)scratch(np * 8);
  hscr_bytes = (size_t)hoff + 16;
  hplan.hscr = (uint32_t*)scratch(hscr_bytes);
  hplan.total = (uint64_t*)scratch(16);
  hplan.tp_out = (uint64_t*)scratch(tps.size() * 16);
  h_tpout.reserve(std::max<size_t>(16, tps.size() * 16));
  d_fixed.reserve(fixed_blob.size() + 16);
  CK(cudaMemcpy(d_fixed.p, fixed_blob.data(), fixed_blob.size(), cudaMemcpyHostToDevice));
  h_total.reserve(64);
  rc_sizing = true;
  device_headers = !host_writer;
}

// the codestream with every code-block left out: main header [+ TLM], SOT + SOD per tile-part, empty packets, EOC
uint64_t Encoder::min_size_of_geometry() const {
  uint64_t n = main_header.size() + 2;
  const std::vector<CodedBlock> empty(layout.num_blocks);
  std::vector<PacketRef> seq; std::vector<uint32_t> tp_first; std::vector<uint8_t> hdr;
  uint64_t ntp = 0;
  for (uint32_t t = 0; t < (uint32_t)layout.tiles.size(); ++t) {
    layout.packet_sequence(t, seq, tp_first);
    ntp += tp_first.size();
    for (const PacketRef& pr : seq) {
      const ResGeom& rg = layout.res_of(pr);
      hdr.clear(); write_packet_header(rg, rg.precincts[pr.precinct], empty.data(), hdr);
      n += hdr.size();
    }
  }
  n += 14 * ntp;
  if (params.need_tlm) n += 6 + 6 * ntp;
  return n;
}

void Encoder::set_target(uint64_t bytes) {
  if (bytes && rq_on()) fail(0x000B0049, "a target size and a target quality cannot be combined on one encoder");
  if (bytes) check_target_size(bytes);
  target_bytes = bytes;
}

// what a size target needs of the configuration and of the geometry (a reconfigure may raise min_bytes past it)
void Encoder::check_target_size(uint64_t bytes) const {
  if (wide)
    fail(0x000B0039, "a target size needs the 32-bit coefficient path: this configuration codes 64-bit coefficients");
  if (!rc_sizing)
    fail(0x000B0039, "a target size needs every tile-part to hold a packet: the device header plan that sizes each "
         "selection cannot describe an empty tile-part");
  if (bytes < min_bytes)
    fail(0x000B0038, "target of %llu bytes is below the smallest codestream of this geometry (%llu bytes)",
         (unsigned long long)bytes, (unsigned long long)min_bytes);
}

// what a quality target needs of the configuration: the size target's conditions (the selection and the final layout
// are the same)
void Encoder::check_target_mse() const {
  if (wide)
    fail(0x000B004A, "a target quality needs the 32-bit coefficient path: this configuration codes 64-bit coefficients");
  if (!rc_sizing)
    fail(0x000B004A, "a target quality needs every tile-part to hold a packet: the device header plan cannot describe an "
         "empty tile-part");
}

void Encoder::set_target_mse(double mse) {
  if (!(std::isfinite(mse) && mse >= 0.0)) fail(0x000B0048, "the target mean squared error must be a finite number >= 0 (got %g)", mse);
  if (mse > 0.0 && rc_on()) fail(0x000B0049, "a target size and a target quality cannot be combined on one encoder");
  if (mse > 0.0) check_target_mse();
  target_mse = mse;
  rq_valid = false;
}

Encoder::~Encoder() {
  for (cudaEvent_t& e : rq_ev) if (e) { cudaEventDestroy(e); e = nullptr; }
}

// the buffers of a quality target, after plan_rate_control: the synthesis jobs of the geometry, a second coefficient
// arena, the scratch image and its descriptors (slot 2), the limit floor(target * N) -- exactly: target = m 2^e with an
// integer m of at most 53 bits
void Encoder::plan_quality() {
  const uint32_t nc = params.num_comps();
  if (transcoding) plan_image(img_type, true);     // the source: the input as the decoder returns it
  build_dwt_jobs(false, rq_jobs, d_rq_jobs);
  d_rcoef.reserve((layout.coef_words + 64) * 4);
  CK(cudaMemset(d_rcoef.p, 0, d_rcoef.cap));
  d_rimg.reserve(img_bytes);
  std::vector<ImgComp> sc(IMG_SLOTS);
  memset(&rq_image, 0, sizeof(rq_image));
  rq_image.ncomp = nc; rq_image.sample_type = img_type;
  rq_samples = 0;
  for (uint32_t c = 0; c < nc; ++c) {
    sc[c].base = (uint64_t)(size_t)(d_rimg.as<uint8_t>() + img_off[c]);
    sc[c].pitch = (uint64_t)img_w[c] * esize_of(img_type); sc[c].col = 1; sc[c].pad = 0;
    rq_image.w[c] = img_w[c]; rq_image.h[c] = img_h[c];
    rq_samples += (uint64_t)img_w[c] * img_h[c];
  }
  CK(cudaMemcpy(const_cast<ImgComp*>(scratch_slot()), sc.data(), IMG_SLOTS * sizeof(ImgComp), cudaMemcpyHostToDevice));
  d_rq.reserve(sizeof(RqState));
  h_rq.reserve(sizeof(RqState));
  memset(h_rq.p, 0, sizeof(RqState));
  rc.q = d_rq.as<RqState>();
  rq_lossless0 = true;
  for (uint32_t c = 0; c < nc; ++c) rq_lossless0 = rq_lossless0 && params.reversible(c);
  for (const EncBlock& e : h_blocks) rq_lossless0 = rq_lossless0 && !(e.flags & ENC_CHECK_NEGZERO);
  for (cudaEvent_t& e : rq_ev) if (!e) CK(cudaEventCreate(&e));
  rq_planned = true;
}

// floor(mse * n), exactly (mse = m 2^(e - 53) with an integer m < 2^53), saturated at 2^64 - 1
static uint64_t sse_limit(double mse, uint64_t n) {
  int e = 0;
  const uint64_t m = (uint64_t)std::ldexp(std::frexp(mse, &e), 53);
  const unsigned __int128 prod = (unsigned __int128)m * n;
  const int sh = e - 53;
  if (sh < 0) { const unsigned __int128 v = -sh >= 128 ? 0 : prod >> -sh; return (v >> 64) ? ~0ull : (uint64_t)v; }
  if (sh >= 64 || (prod && (prod >> (127 - sh)))) return ~0ull;
  const unsigned __int128 v = prod << sh;
  return (v >> 64) ? ~0ull : (uint64_t)v;
}

// per-block weights W_b = G_b C_c s_c^2 and the device tables of the selection (see RcTables)
void Encoder::plan_rate_control() {
  const uint32_t nb = (uint32_t)h_blocks.size();
  uint32_t kmax = 0;
  for (const EncBlock& e : h_blocks) kmax = std::max<uint32_t>(kmax, 31u - e.p);
  const uint32_t kc = kmax + 1;
  std::vector<double> wgt(nb, 0.0);
  std::vector<uint8_t> irv(nb, 0);
  std::vector<float> dlt(nb, 0.f);
  const Params& P = params;
  const bool ct = P.color_transform();
  std::vector<std::vector<double>> gains(P.num_comps());
  for (uint32_t c = 0; c < P.num_comps(); ++c) gains[c] = P.band_energy_gains(c);
  for (const TileGeom& t : layout.tiles)
    for (const TileCompGeom& tc : t.comps)
      for (const ResGeom& rg : tc.res)
        for (uint32_t b = 0; b < 4; ++b) {
          const BandGeom& bg = rg.bands[b];
          if (bg.empty) continue;
          const uint32_t c = tc.comp;
          const bool rev = P.reversible(c);
          const double G = gains[c][P.subband_index(c, rg.res_num, b)];
          const double C = (ct && c < 3) ? colour_weight(!P.reversible(0), c) : 1.0;
          const double s = rev ? 1.0 : (double)P.band_delta(c, rg.res_num, b) * std::ldexp(1.0, (int)P.comps[c].bit_depth);
          for (uint32_t i = 0; i < bg.nbw * bg.nbh; ++i) {
            wgt[bg.block_base + i] = G * C * s * s; irv[bg.block_base + i] = rev ? 0 : 1; dlt[bg.block_base + i] = bg.delta;
          }
        }
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 63) & ~(size_t)63; return o; };
  const size_t o_cand = take((size_t)nb * kc * sizeof(EncResult)), o_dist = take((size_t)nb * kc * 8), o_w = take((size_t)nb * 8);
  const size_t o_irv = take(nb), o_nc = take(nb), o_hk = take((size_t)nb * (kc + 1)), o_key = take((size_t)nb * kc * 4);
  const size_t o_len = take((size_t)nb * kc * 4), o_hn = take(nb), o_ch = take(nb), o_st = take(sizeof(RcState));
  const size_t o_dl = take((size_t)nb * 4);
  d_rc.reserve(off);
  uint8_t* base = d_rc.as<uint8_t>();
  rc.kc = kc;
  rc.cand = (EncResult*)(base + o_cand); rc.dist = (double*)(base + o_dist); rc.weight = (const double*)(base + o_w);
  rc.irv = base + o_irv; rc.ncand = base + o_nc; rc.hull_k = base + o_hk; rc.hull_key = (uint32_t*)(base + o_key);
  rc.hull_len = (uint32_t*)(base + o_len); rc.hull_n = base + o_hn; rc.chosen = base + o_ch; rc.state = (RcState*)(base + o_st);
  CK(cudaMemcpy(base + o_w, wgt.data(), (size_t)nb * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(base + o_irv, irv.data(), nb, cudaMemcpyHostToDevice));
  rc.delta = (const float*)(base + o_dl); rc.q = nullptr;
  CK(cudaMemcpy(base + o_dl, dlt.data(), (size_t)nb * 4, cudaMemcpyHostToDevice));
  d_work.reserve(std::max<size_t>(1, nb) * sizeof(EncBlock));
  h_rc.reserve(64 + nb);
  rc_kc = kc;
}

int32_t* Encoder::exchange(const int32_t* line_written, uint32_t& next_comp) {
  // ojph::codestream::exchange (ojph_codestream_local.cpp:1176-1224): the caller fills the
  // returned line; planar => all rows of comp 0 first, else row by row, comp by comp
  uint32_t nc = params.num_comps();
  if (h_frame.p == nullptr) {
    size_t tot = 0; for (uint32_t c = 0; c < nc; ++c) tot += (size_t)img_w[c] * img_h[c];
    h_frame.reserve(tot * 4);
    uint32_t mw = 0; for (uint32_t c = 0; c < nc; ++c) mw = std::max(mw, img_w[c]);
    line_buf.assign(mw, 0);
  }
  auto plane = [&](uint32_t c) { size_t o = 0; for (uint32_t i = 0; i < c; ++i) o += (size_t)img_w[i] * img_h[i]; return h_frame.as<int32_t>() + o; };
  if (line_written) {
    if (lines_done) { next_comp = 0; return nullptr; }
    memcpy(plane(cur_comp) + (size_t)line_cur[cur_comp] * img_w[cur_comp], line_written, (size_t)img_w[cur_comp] * 4);
    line_cur[cur_comp]++;
    if (params.planar == 1) {
      if (line_cur[cur_comp] >= img_h[cur_comp]) { if (++cur_comp >= nc) { lines_done = true; next_comp = 0; return nullptr; } }
    } else {
      // next component that still has rows, in round-robin order
      uint32_t tries = 0;
      do { cur_comp = (cur_comp + 1) % nc; ++tries; } while (line_cur[cur_comp] >= img_h[cur_comp] && tries <= nc);
      if (tries > nc) { lines_done = true; next_comp = 0; return nullptr; }
    }
  }
  next_comp = cur_comp;
  return line_buf.data();
}

size_t Encoder::encode(const void* const* planes, const uint32_t* strides, bool caller_image,
                       uint8_t* out, size_t out_cap, bool out_on_device)
{
  if (transcoding)
    fail(0x000B0053, "this encoder was configured from a codestream (ojb_enc_transcode_headers): it transcodes, it has no image");
  Frame f = begin_frame(Frame::DWT, true, caller_image, planes, strides);
  f.graph = planes == nullptr && out_on_device;
  return device_headers ? finish_device(f, out, out_cap, out_on_device) : finish_host(f, out, out_cap, out_on_device);
}

void Encoder::encode_front() {
  const Frame f = begin_frame(Frame::DWT, false);
  enqueue_front(f);
  launch_ctrl_copy(h_status.p, d_status.p, 16, stream); ++last_launches;
  mark(4);
  CK(cudaStreamSynchronize(stream));
  CK(cudaGetLastError());
  collect(5);
  check_coder_status();
}

size_t Encoder::encode_back(uint8_t* out, size_t out_cap) {
  const Frame f = begin_frame(Frame::CODED, false);
  return device_headers ? finish_device(f, out, out_cap, true) : finish_host(f, out, out_cap, true);
}

// stage marks 0 and 1 around the planes' upload; with a target (targets: a whole frame), its conditions and buffers
Encoder::Frame Encoder::begin_frame(Frame::Front front, bool targets, bool caller_image, const void* const* planes,
                                    const uint32_t* strides) {
  last_launches = 0;
  mark(0);
  if (planes) upload_planes(planes, strides);
  mark(1);
  Frame f;
  f.front = front; f.caller_image = caller_image;
  f.nb = (uint32_t)h_blocks.size();
  f.rq = targets && rq_on() && f.nb > 0;
  f.rc = (targets && rc_on() && f.nb > 0) || f.rq;
  if (f.rq) {
    check_target_mse();
    if (rc_kc == 0) plan_rate_control();
    if (!rq_planned) plan_quality();
    rq_limit = sse_limit(target_mse, rq_samples);
    rq_valid = false;
  } else if (f.rc) {
    check_target_size(target_bytes);
    if (rc_kc == 0) plan_rate_control();
  }
  f.work = d_work.as<EncBlock>();
  f.blocks = front == Frame::TRANSCODE ? d_xblocks.as<EncBlock>() : d_blocks.as<EncBlock>();
  f.code_blocks = f.rc ? f.work : f.blocks;
  return f;
}

void Encoder::upload_planes(const void* const* planes, const uint32_t* strides) {
  const uint32_t es = esize_of(img_type);
  for (uint32_t c = 0; c < params.num_comps(); ++c) {
    uint8_t* d = d_image.as<uint8_t>() + img_off[c];
    const uint32_t st = strides ? strides[c] : img_w[c];
    if (st == img_w[c])
      cuda_check(cudaMemcpyAsync(d, planes[c], (size_t)img_w[c] * img_h[c] * es, cudaMemcpyHostToDevice, stream), "upload");
    else
      for (uint32_t y = 0; y < img_h[c]; ++y)
        cuda_check(cudaMemcpyAsync(d + (size_t)y * img_w[c] * es, (const uint8_t*)planes[c] + (size_t)y * st * es,
                                   (size_t)img_w[c] * es, cudaMemcpyHostToDevice, stream), "upload");
  }
}

// the transform (forward DWT or a transcode's block decoders), a target's selection and the block coding
void Encoder::enqueue_front(const Frame& f) {
  CK(cudaMemsetAsync(d_status.p, 0, 16, stream));
  if (f.caller_image) enqueue_caller_image();
  if (f.front == Frame::TRANSCODE) enqueue_transcode_front();
  else if (f.front == Frame::DWT)
    enqueue_dwt(true, jobs, d_jobs, img_slot(f.caller_image), f.caller_image && caller_interleaved, d_coef.as<uint32_t>());
  mark(2);
  if (f.front == Frame::CODED) { mark(3); return; }
  if (f.rc) enqueue_rc(f);
  enqueue_code(f);
  mark(3);
}

void Encoder::enqueue_code(const Frame& f) {
  const bool thread_per_block = (serial_block_encoder() && !few_blocks_warp) || max_block_w > 64 || wide;
  if (thread_per_block)
    launch_ht_encode_serial(f.code_blocks, f.nb, num_fast_blocks, max_block_w, d_coef.as<uint32_t>(), d_slots.as<uint8_t>(),
                            d_results.as<EncResult>(), d_tables_enc.as<uint16_t>(), d_status.as<uint32_t>(), stream, wide, &side);
  else
    launch_ht_encode(f.code_blocks, f.nb, d_coef.as<uint32_t>(), d_slots.as<uint8_t>(),
                     d_results.as<EncResult>(), d_tables_enc.as<uint16_t>(), d_status.as<uint32_t>(), stream);
  last_launches += thread_per_block ? (num_fast_blocks ? 1 : 0) + (num_fast_blocks < f.nb ? 1 : 0) : 1;
}

void Encoder::check_coder_status() {
  status_flags = h_status.as<uint32_t>()[0];
  if (status_flags & 2u) fail(0x00020001, "mel encoder's buffer is full");
  if (status_flags & 1u) fail(0x00020005, "block encoder's output slot is full");
}

// rate control: the candidates and the rounds of the selection (rate_ctrl.cu); each round sizes its selection with the
// packet header kernels, so the block coder's final pass and the headers see the chosen planes in work
void Encoder::enqueue_rc(const Frame& f) {
  CK(cudaMemsetAsync(rc.state, 0, sizeof(RcState), stream));
  launch_rc_prepare(f.blocks, f.nb, d_coef.as<uint32_t>(), rc, stream);
  mark(8);
  launch_ht_encode_lengths(f.blocks, f.nb, rc.kc, rc.ncand, max_block_w, d_coef.as<uint32_t>(), rc.cand,
                           d_tables_enc.as<uint16_t>(), stream);
  mark(9);
  launch_rc_hull(f.blocks, f.nb, f.work, d_results.as<EncResult>(), rc, stream);
  last_launches += 4;
  if (f.rq) {
    CK(cudaMemsetAsync(rc.q, 0, sizeof(RqState), stream));
    launch_rq_init(rc, rq_limit, params.num_comps(), rq_lossless0 && !(f.front == Frame::TRANSCODE && xc_two_pass), stream);
    ++last_launches;
    for (int r = 0; r < RQ_GRAPH_ROUNDS; ++r) rq_round(f);
    rq_final(f);
    mark(10);
    return;
  }
  rc_size(f, true);
  for (int r = 0; r < RC_ROUNDS; ++r) {
    launch_rc_round(f.blocks, f.nb, f.work, d_results.as<EncResult>(), rc, stream);
    last_launches += 2;
    rc_size(f, false);
  }
  rc_state_out(f);
  mark(10);
}

void Encoder::rc_size(const Frame& f, bool first) {
  launch_packet_header_total(hplan, f.work, d_results.as<EncResult>(), 30u, fixed_blob.size(), true, stream);
  launch_rc_check(rc, hplan.total, target_bytes, min_bytes, first, stream);
  last_launches += packet_header_total_launches(hplan) + 1;
}

void Encoder::rc_state_out(const Frame& f) {
  launch_ctrl_copy(h_rc.p, rc.state, sizeof(RcState), stream);
  launch_ctrl_copy(h_rc.as<uint8_t>() + 64, rc.chosen, f.nb, stream);
  last_launches += 2;
}

// a round of the quality target: select, reconstruct as the decoder would, synthesise, measure (rate_ctrl.cu).  The
// synthesis is on 32-bit coefficients: check_target_mse refuses the 64-bit path
void Encoder::rq_round(const Frame& f) {
  launch_rq_select(d_blocks.as<EncBlock>(), f.blocks, f.nb, f.work, d_results.as<EncResult>(), d_coef.as<uint32_t>(),
                   d_rcoef.as<uint32_t>(), rc, stream);
  last_launches += 3;
  enqueue_dwt(false, rq_jobs, d_rq_jobs, scratch_slot(), false, d_rcoef.as<uint32_t>());
  launch_rq_measure(scratch_slot(), img_slot(f.caller_image), rq_image, rc, stream);
  last_launches += 2;
}

void Encoder::rq_final(const Frame& f) {
  launch_rq_final(f.blocks, f.nb, f.work, d_results.as<EncResult>(), rc, stream);
  launch_ctrl_copy(h_rq.p, rc.q, sizeof(RqState), stream);
  launch_ctrl_copy(h_rc.as<uint8_t>() + 64, rc.chosen, f.nb, stream);
  last_launches += 3;
}

// after the frame's rounds: the rare selection that still does not fit goes on eagerly; true = it changed
bool Encoder::rc_settle(const Frame& f) {
  if (f.rq) {
    if (h_rq.as<RqState>()->done) return false;
    CK(cudaEventRecord(rq_ev[0], stream));
    // the bracket closes within RQ_BODY_ROUNDS + 34 rounds (rq_update_kernel); one synchronisation per round
    while (!h_rq.as<RqState>()->done) {
      rq_round(f);
      launch_ctrl_copy(h_rq.p, rc.q, sizeof(RqState), stream); ++last_launches;
      CK(cudaStreamSynchronize(stream));
    }
    rq_final(f);
    CK(cudaEventRecord(rq_ev[1], stream));
    return true;
  }
  if (!f.rc || h_rc.as<RcState>()->done) return false;
  for (int i = 0; !h_rc.as<RcState>()->done; ++i) {
    // every round over the target strictly lowers the selected body (rc_check_kernel), so there are at most as many
    // rounds as distinct selections: one more hull segment per block and round at the very worst
    if ((uint64_t)i > (uint64_t)f.nb * rc.kc + 2)
      fail(0x000B003A, "rate control did not settle on a selection that fits the target (internal error)");
    launch_rc_round(f.blocks, f.nb, f.work, d_results.as<EncResult>(), rc, stream);
    last_launches += 2;
    rc_size(f, false);
    rc_state_out(f);
    CK(cudaStreamSynchronize(stream));
  }
  return true;
}

// packet headers, markers and layout by kernels; the host only learns the length (and, for a host buffer, waits for it
// before asking for the copy)
size_t Encoder::finish_device(const Frame& f, uint8_t* out, size_t out_cap, bool out_on_device) {
  uint8_t* dev_out;
  uint64_t cap = out_cap;
  if (out_on_device) dev_out = out;
  else {
    if (d_out.cap < 1024) d_out.reserve(std::max<size_t>(1 << 20, fixed_blob.size() + 64));
    dev_out = d_out.as<uint8_t>(); cap = std::min<uint64_t>(out_cap, d_out.cap);
  }
  auto sync = [&] {
    CK(cudaStreamSynchronize(stream));
    CK(cudaGetLastError());
    check_coder_status();
  };
  auto enqueue = [&] {
    enqueue_front(f);
    launch_ctrl_copy(h_status.p, d_status.p, 16, stream); ++last_launches;
    mark(4); mark(5);
    enqueue_device_layout(f, dev_out, cap);
  };
  // resident form (frame already in HBM, codestream stays there): nothing in the call depends on host data, so the
  // whole thing replays as a graph (a caller's image is named by the control block the graph copies in, so its
  // addresses are not part of the key)
  if (f.graph)
    run_frame({ (uint64_t)(size_t)dev_out, cap, (uint64_t)f.nb, (uint64_t)num_fast_blocks, (uint64_t)(size_t)d_slots.p, (uint64_t)(size_t)d_coef.p,
                f.rc ? target_bytes : 0, (uint64_t)(size_t)d_rc.p, (uint64_t)(size_t)d_work.p,
                f.rq ? rq_limit : 0, (uint64_t)f.rq, (uint64_t)(size_t)d_rq.p, (uint64_t)(size_t)d_rcoef.p,
                (uint64_t)(size_t)d_rimg.p, (uint64_t)(size_t)d_rq_jobs.p,
                (uint64_t)(size_t)img_slot(f.caller_image), (uint64_t)(f.caller_image && caller_interleaved) }, enqueue);
  else enqueue();
  sync();
  if (rc_settle(f)) {                  // code and lay out the settled selection
    enqueue_code(f); launch_ctrl_copy(h_status.p, d_status.p, 16, stream); ++last_launches;
    if (f.rq) CK(cudaEventRecord(rq_ev[2], stream));
    enqueue_device_layout(f, dev_out, cap);
    sync();
  }
  // did not fit: the caller's buffer is too small, or (host output) the staging buffer has to grow once
  for (bool grown = false; h_total.as<uint64_t>()[1] != 0; grown = true) {
    const size_t need = (size_t)h_total.as<uint64_t>()[0];
    if (need > out_cap || out_on_device || grown)
      fail(0x000B0030, "output buffer too small: need %zu bytes, have %zu", need, out_cap);
    d_out.reserve(need + 64); dev_out = d_out.as<uint8_t>(); cap = std::min<uint64_t>(out_cap, d_out.cap);
    enqueue_device_layout(f, dev_out, cap);
    sync();
  }
  host_ms = 0;
  last_tileparts.clear();
  if (!tile_mask.empty())
    for (uint32_t i = 0; i < hplan.ntps; ++i)
      last_tileparts.push_back(TilePartOut{ h_tp_tile[i], h_tpout.as<uint64_t>()[2 * i], (uint32_t)h_tpout.as<uint64_t>()[2 * i + 1] });
  return end_frame(f, out, dev_out, (size_t)h_total.as<uint64_t>()[0], out_on_device);
}

void Encoder::enqueue_device_layout(const Frame& f, uint8_t* dev_out, uint64_t cap) {
  if (fixed_blob.size() <= cap) CK(cudaMemcpyAsync(dev_out, d_fixed.p, fixed_blob.size(), cudaMemcpyDeviceToDevice, stream));
  CK(cudaMemsetAsync(hplan.hscr, 0, hscr_bytes, stream));
  launch_packet_headers(hplan, f.code_blocks, d_results.as<EncResult>(), wide ? 62u : 30u, fixed_blob.size(), cap,
                        tile_mask.empty(), dev_out, d_dst.as<uint64_t>(), stream);
  if (!tile_mask.empty() && hplan.ntps) { launch_ctrl_copy(h_tpout.p, hplan.tp_out, (size_t)hplan.ntps * 16, stream); ++last_launches; }
  launch_gather_blocks(d_blocks.as<EncBlock>(), d_results.as<EncResult>(), d_dst.as<uint64_t>(), f.nb, d_slots.as<uint8_t>(), dev_out, stream);
  launch_ctrl_copy(h_total.p, hplan.total, 16, stream);
  last_launches += packet_header_launches(hplan) + 2;
  mark(6);
}

// the host writer's frame: packets with their headers, tile-parts, and everything that is not code-block data (blob)
// with the pieces that place it in the codestream
struct Encoder::HostLayout {
  struct Pkt { PacketRef ref; std::vector<uint8_t> hdr; uint32_t hdr_len, body; };
  struct TilePart { uint32_t tile, first, count, tp_idx, tp_cnt; uint64_t bytes; };
  struct Piece { size_t src, dst; uint32_t len; };
  std::vector<Pkt> pkts;
  std::vector<TilePart> tps;
  std::vector<uint8_t> blob;
  std::vector<Piece> pieces;
};

// packet headers and the final layout on the host (with a target: at the planes the selection chose), assembled on
// the device with one copy out
size_t Encoder::finish_host(const Frame& f, uint8_t* out, size_t out_cap, bool out_on_device) {
  const uint32_t nb = f.nb;
  enqueue_front(f);
  if (nb) launch_ctrl_copy(h_results.p, d_results.p, (size_t)nb * sizeof(EncResult), stream);
  launch_ctrl_copy(h_status.p, d_status.p, 16, stream);
  last_launches += nb ? 2 : 1;
  mark(4);
  CK(cudaStreamSynchronize(stream));
  auto host_t0 = std::chrono::steady_clock::now();
  CK(cudaGetLastError());
  check_coder_status();
  if (rc_settle(f)) {
    enqueue_code(f);
    if (f.rq) CK(cudaEventRecord(rq_ev[2], stream));
    launch_ctrl_copy(h_results.p, d_results.p, (size_t)nb * sizeof(EncResult), stream); ++last_launches;
    CK(cudaStreamSynchronize(stream));
    CK(cudaGetLastError());
  }
  HostLayout hl;
  host_packets(f, hl);
  const size_t total = host_markers(hl);
  if (total > out_cap) fail(0x000B0030, "output buffer too small: need %zu bytes, have %zu", total, out_cap);
  const std::vector<uint8_t>& blob = hl.blob;
  const std::vector<HostLayout::Piece>& pieces = hl.pieces;
  uint8_t* dev_out;
  if (out_on_device) dev_out = out; else { d_out.reserve(total + 64); dev_out = d_out.as<uint8_t>(); }
  h_hdr.reserve(blob.size() + 64); memcpy(h_hdr.p, blob.data(), blob.size());
  host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count();
  mark(5);
  d_hdr.reserve(blob.size() + 64);
  launch_ctrl_copy(d_hdr.p, h_hdr.p, blob.size(), stream);
  h_pieces.reserve(pieces.size() * sizeof(CopyPiece)); d_pieces.reserve(pieces.size() * sizeof(CopyPiece));
  CopyPiece* cp = h_pieces.as<CopyPiece>();
  uint32_t max_piece = 0;
  for (size_t i = 0; i < pieces.size(); ++i) {
    cp[i].src_off = pieces[i].src; cp[i].dst_off = pieces[i].dst; cp[i].len = pieces[i].len; cp[i].src_sel = 1;
    max_piece = std::max(max_piece, cp[i].len);
  }
  launch_ctrl_copy(d_pieces.p, h_pieces.p, pieces.size() * sizeof(CopyPiece), stream);
  if (nb) launch_ctrl_copy(d_dst.p, h_dst.p, (size_t)nb * 8, stream);
  last_launches += (blob.size() ? 1 : 0) + (pieces.empty() ? 0 : 1) + (nb ? 1 : 0);
  launch_gather_blocks(f.code_blocks, d_results.as<EncResult>(), d_dst.as<uint64_t>(), nb,
                       d_slots.as<uint8_t>(), dev_out, stream);
  launch_assemble(d_pieces.as<CopyPiece>(), (uint32_t)pieces.size(), max_piece, d_slots.as<uint8_t>(), d_hdr.as<uint8_t>(), dev_out, stream);
  last_launches += 2;
  mark(6);
  return end_frame(f, out, dev_out, total, out_on_device);
}

// the blocks' records from the coder's results, the packet sequence of every tile-part and the packet headers
void Encoder::host_packets(const Frame& f, HostLayout& hl) {
  const uint32_t nb = f.nb;
  const EncResult* res = h_results.as<EncResult>();
  const uint8_t* chosen = f.rc ? h_rc.as<uint8_t>() + 64 : nullptr;
  std::vector<EncBlock> xb;                // a transcode's per-frame start planes
  if (f.front == Frame::TRANSCODE && nb) {
    xb.resize(nb);
    CK(cudaMemcpy(xb.data(), d_xblocks.p, (size_t)nb * sizeof(EncBlock), cudaMemcpyDeviceToHost));
  }
  const EncBlock* hb = xb.empty() ? h_blocks.data() : xb.data();
  for (uint32_t b = 0; b < nb; ++b) {
    CodedBlock& cb = coded[b];
    uint32_t len = res[b].len_head + res[b].len_tail;
    cb.pass_len[0] = len; cb.pass_len[1] = 0;
    cb.num_passes = len ? 1 : 0;
    cb.missing_msbs = len ? (uint8_t)((wide ? 62u : 30u) - hb[b].p - (chosen ? chosen[b] : 0u)) : 0;
  }
  std::vector<HostLayout::Pkt>& pkts = hl.pkts;
  std::vector<PacketRef> seq; std::vector<uint32_t> tp_first, tp_index;
  uint32_t tp_total = 0;
  for (uint32_t t = 0; t < (uint32_t)layout.tiles.size(); ++t) {
    if (!tile_wanted(t)) continue;
    layout.packet_sequence(t, seq, tp_first, &tp_index, &tp_total);
    size_t base = pkts.size();
    for (const PacketRef& pr : seq) { pkts.emplace_back(); pkts.back().ref = pr; pkts.back().hdr_len = pkts.back().body = 0; }
    for (size_t i = 0; i < tp_first.size(); ++i) {
      HostLayout::TilePart tp; tp.tile = t; tp.first = (uint32_t)(base + tp_first[i]);
      uint32_t end = (i + 1 < tp_first.size()) ? tp_first[i + 1] : (uint32_t)seq.size();
      tp.count = end - tp_first[i]; tp.tp_idx = tp_index[i]; tp.tp_cnt = tp_total;
      tp.bytes = 0;
      hl.tps.push_back(tp);
    }
  }
  // packet headers are independent of each other: a few host threads share them (largest first)
  std::vector<uint32_t> order(pkts.size());
  for (uint32_t i = 0; i < order.size(); ++i) order[i] = i;
  auto weight = [&](uint32_t i) {
    const ResGeom& rg = layout.res_of(pkts[i].ref); const PrecinctGeom& pc = rg.precincts[pkts[i].ref.precinct];
    uint32_t n = 0; for (int b = 0; b < 4; ++b) n += pc.cb_idx[b].w * pc.cb_idx[b].h; return n;
  };
  std::vector<uint32_t> wt(pkts.size());
  for (uint32_t i = 0; i < wt.size(); ++i) wt[i] = weight(i);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return wt[a] > wt[b]; });
  std::atomic<uint32_t> next(0);
  auto work = [&]() {
    for (;;) {
      uint32_t k = next.fetch_add(1);
      if (k >= order.size()) break;
      HostLayout::Pkt& pk = pkts[order[k]];
      const ResGeom& rg = layout.res_of(pk.ref);
      pk.hdr.reserve(64 + wt[order[k]] * 4);
      pk.body = write_packet_header(rg, rg.precincts[pk.ref.precinct], coded.data(), pk.hdr);
      pk.hdr_len = (uint32_t)pk.hdr.size();
    }
  };
  uint32_t nthreads = (uint32_t)std::min<size_t>(std::min<size_t>(host_threads, pkts.size()), 16);
  if (nb < 2048 || nthreads <= 1) work();
  else {
    std::vector<std::thread> th;
    for (uint32_t i = 1; i < nthreads; ++i) th.emplace_back(work);
    work();
    for (auto& t : th) t.join();
  }
  for (HostLayout::TilePart& tp : hl.tps)
    for (uint32_t q = 0; q < tp.count; ++q) tp.bytes += pkts[tp.first + q].hdr_len + pkts[tp.first + q].body;
}

// marker bytes (main header [+ TLM], SOT+SOD per tile-part, EOC) and packet headers into the blob, the pieces that
// place it and each block's offset (h_dst); returns the codestream's length
size_t Encoder::host_markers(HostLayout& hl) {
  std::vector<uint8_t>& blob = hl.blob;
  std::vector<HostLayout::Piece>& pieces = hl.pieces;
  uint64_t pos = 0;
  auto add_piece = [&](size_t src, uint32_t len) {
    if (!pieces.empty() && pieces.back().src + pieces.back().len == src && pieces.back().dst + pieces.back().len == pos)
      pieces.back().len += len;
    else pieces.push_back(HostLayout::Piece{ src, (size_t)pos, len });
    pos += len;
  };
  const bool partial = !tile_mask.empty();       // tile-parts only: the writer rank adds main header, TLM and EOC
  if (!partial) blob = main_header;
  last_tileparts.clear();
  if (params.need_tlm && !partial) {
    if (4 + 6 * hl.tps.size() > 65535) fail(0x000500B1, "too many tile-parts for one TLM marker segment");
    put_u16(blob, M_TLM); put_u16(blob, (uint32_t)(4 + 6 * hl.tps.size())); put_u8(blob, 0); put_u8(blob, 0x60);
    for (const HostLayout::TilePart& tp : hl.tps) { put_u16(blob, tp.tile); put_u32(blob, (uint32_t)(tp.bytes + 14)); }
  }
  if (!blob.empty()) add_piece(0, (uint32_t)blob.size());
  uint64_t* dst = h_dst.as<uint64_t>();
  for (const HostLayout::TilePart& tp : hl.tps) {
    size_t s = blob.size();
    last_tileparts.push_back(TilePartOut{ tp.tile, pos, (uint32_t)(tp.bytes + 14) });
    put_u16(blob, M_SOT); put_u16(blob, 10); put_u16(blob, tp.tile); put_u32(blob, (uint32_t)(tp.bytes + 14));
    put_u8(blob, tp.tp_idx); put_u8(blob, tp.tp_cnt);
    put_u16(blob, M_SOD);
    add_piece(s, 14);
    for (uint32_t q = 0; q < tp.count; ++q) {
      const HostLayout::Pkt& k = hl.pkts[tp.first + q];
      size_t hs = blob.size();
      blob.insert(blob.end(), k.hdr.begin(), k.hdr.end());
      add_piece(hs, k.hdr_len);
      if (k.body == 0) continue;
      const ResGeom& rg = layout.res_of(k.ref);
      const PrecinctGeom& pc = rg.precincts[k.ref.precinct];
      for (uint32_t sb = 0; sb < 4; ++sb) {
        const BandGeom& bg = rg.bands[sb];
        if (bg.empty) continue;
        const Rect& ci = pc.cb_idx[sb];
        for (uint32_t y = 0; y < ci.h; ++y)
          for (uint32_t x = 0; x < ci.w; ++x) {
            uint32_t bi = bg.block_base + (ci.y0 + y) * bg.nbw + ci.x0 + x;
            dst[bi] = pos; pos += coded[bi].pass_len[0];
          }
      }
    }
  }
  if (!partial) { size_t s = blob.size(); put_u16(blob, M_EOC); add_piece(s, 2); }
  return (size_t)pos;
}

// the end of both finishing paths: the codestream to a host buffer, the stage times, the line front end reset
size_t Encoder::end_frame(const Frame& f, uint8_t* out, const uint8_t* dev_out, size_t total, bool out_on_device) {
  if (!out_on_device) CK(cudaMemcpyAsync(out, dev_out, total, cudaMemcpyDeviceToHost, stream));
  mark(7);
  CK(cudaStreamSynchronize(stream));
  collect(8);
  rc_times(f);
  CK(cudaGetLastError());
  std::fill(line_cur.begin(), line_cur.end(), 0u); cur_comp = 0; lines_done = false;
  return total;
}

void Encoder::rc_times(const Frame& f) {
  if (f.rq) {
    const bool eager = h_rq.as<RqState>()->rounds > (uint32_t)RQ_GRAPH_ROUNDS;
    cudaEventElapsedTime(&rq_ms[0], ev[2], ev[9]); cudaEventElapsedTime(&rq_ms[1], ev[9], ev[10]);
    if (eager) {
      float t = 0; cudaEventElapsedTime(&t, rq_ev[0], rq_ev[1]); rq_ms[1] += t;
      cudaEventElapsedTime(&rq_ms[2], rq_ev[1], rq_ev[2]);
    } else cudaEventElapsedTime(&rq_ms[2], ev[10], ev[3]);
    rq_valid = true;
    return;
  }
  if (!f.rc) return;
  cudaEventElapsedTime(&rc_ms[0], ev[2], ev[8]); cudaEventElapsedTime(&rc_ms[1], ev[8], ev[9]);
  cudaEventElapsedTime(&rc_ms[2], ev[9], ev[10]); cudaEventElapsedTime(&rc_ms[3], ev[10], ev[3]);
}

//------------------------------------------------------------------------------------------
// Decoder
//------------------------------------------------------------------------------------------
void Decoder::Mirror::fetch(size_t first_page, size_t npages) {
  // one copy for the missing page and, when the request is a single page, the one after it (headers of large
  // packets run on for tens of kilobytes; the round trip, not the bytes, is the cost)
  const size_t total = (len + (1u << PAGE_SHIFT) - 1) >> PAGE_SHIFT;
  size_t last = std::min(total, first_page + std::max<size_t>(npages, 1));
  while (last > first_page + 1 && present[last - 1]) --last;
  const size_t a = first_page << PAGE_SHIFT, b = std::min(len, last << PAGE_SHIFT);
  cuda_check(cudaMemcpyAsync(host.as<uint8_t>() + a, dev + a, b - a, cudaMemcpyDeviceToHost, owner->stream), "codestream page fetch");
  cuda_check(cudaStreamSynchronize(owner->stream), "codestream page fetch");
  for (size_t pg = first_page; pg < last; ++pg) present[pg] = 1;
  fetched_bytes += b - a;
}

void Decoder::read_headers_device(const uint8_t* dev, size_t len, uint32_t sample_type) {
  mirror.owner = this; mirror.dev = dev; mirror.len = len; mirror.fetched_bytes = 0;
  mirror.host.reserve(len + 64);
  mirror.present.assign((len + (1u << HostMirror::PAGE_SHIFT) - 1) >> HostMirror::PAGE_SHIFT, 0);
  // a stream of frames of one geometry keeps its packet headers in about the same places: the pages the previous
  // frame's parse touched are requested up front, back to back, and awaited once (a miss is fetched on demand)
  if (len <= (8u << 20)) {
    // a small codestream: one copy of everything instead of the driver calls of a page-wise fetch (tens of page
    // copies per frame, from every stream in flight)
    CK(cudaMemcpyAsync(mirror.host.p, dev, len, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    std::fill(mirror.present.begin(), mirror.present.end(), (uint8_t)1);
    mirror.fetched_bytes += len;
  } else if (!mirror.last_pages.empty()) {
    // runs of adjacent pages go out as one copy each
    size_t got = 0;
    const size_t np = mirror.present.size();
    for (size_t i = 0; i < mirror.last_pages.size(); ) {
      const size_t first = mirror.last_pages[i];
      size_t last = first;
      while (i + 1 < mirror.last_pages.size() && mirror.last_pages[i + 1] <= last + 2) last = mirror.last_pages[++i];   // bridge single-page gaps
      ++i;
      if (first >= np) continue;
      last = std::min(last, np - 1);
      const size_t a = first << HostMirror::PAGE_SHIFT, b = std::min(len, (last + 1) << HostMirror::PAGE_SHIFT);
      CK(cudaMemcpyAsync(mirror.host.as<uint8_t>() + a, dev + a, b - a, cudaMemcpyDeviceToHost, stream));
      for (size_t pg = first; pg <= last; ++pg) mirror.present[pg] = 1;
      got += b - a;
    }
    CK(cudaStreamSynchronize(stream));
    mirror.fetched_bytes += got;
  }
  mirror.last_pages.clear();
  // the main header: normally well inside the first page; a parse that runs out of fetched bytes is repeated
  // with everything fetched
  size_t have = std::min<size_t>(len, 1u << HostMirror::PAGE_SHIFT);
  if (len) mirror.need(0, have);
  for (;;) {
    try { read_headers(mirror.host.as<uint8_t>(), have, sample_type); break; }
    catch (const Error&) {
      if (have == len) throw;
      have = len; mirror.need(0, len);
    }
  }
  j2c_len = len; dev_cs = dev; mirrored = true;
}

void Decoder::read_headers(const uint8_t* data, size_t len, uint32_t sample_type) {
  Params np;
  size_t sot = np.read_main_header(data, len);
  j2c = data; j2c_len = len; first_sot = sot; dev_cs = nullptr; mirrored = false;
  // geometry depends on SIZ/COD/QCD/QCC only; rebuild when any of those bytes changed
  std::vector<uint8_t> sig;
  {
    // strip COM/TLM-like segments is unnecessary: compare everything up to the first SOT
    sig.assign(data, data + sot);
    sig.push_back((uint8_t)sample_type);
    sig.insert(sig.end(), tile_mask.begin(), tile_mask.end());
    if (region.on()) { sig.push_back(0xA5); sig.push_back((uint8_t)region.rank); sig.push_back((uint8_t)region.world); }
  }
  if (sig == header_sig && !layout.tiles.empty()) return;
  // everything below can throw (precision check, geometry, cudaMalloc, container check): the signature
  // that lets the next call skip this rebuild is committed last, so a failed setup is redone
  header_sig.clear();
  if (np.num_comps() > 16)
    fail(0x000B0008, "%u components: the frame interface carries at most 16", np.num_comps());
  params = np;
  // the decoder side derives the same planar default as the reference (read_headers :879)
  params.planar = params.color_transform() ? 0 : 1;
  wide = params.needs_wide();
  if (wide && sample_type != ST_I32) fail(0x000B0010, "samples beyond 16 bits need the 32-bit sample container");
  skip_read = skip_recon = 0;
  layout.build(params);
  max_block_w = widest_block(layout);
  upload_tables();
  if (!parse_only) {
    d_coef.reserve((layout.coef_words + 64) * (wide ? 8 : 4));
    setup_geometry(sample_type);
  }
  // geometry part of the block records
  h_dec_proto.assign(layout.num_blocks, DecBlock());
  block_res.assign(layout.num_blocks, 0);
  block_wanted.clear();
  if (!tile_mask.empty()) block_wanted.assign(layout.num_blocks, 0);
  if (region.on()) block_wanted = region_blocks;           // row regions: the blocks this rank's rows depend on (plan_region)
  size_t scratch = 0;
  for (const TileGeom& t : layout.tiles)
    for (const TileCompGeom& tc : t.comps)
      for (const ResGeom& rg : tc.res)
        for (uint32_t b = 0; b < 4; ++b) {
          const BandGeom& bg = rg.bands[b];
          if (bg.empty) continue;
          for (uint32_t by = 0; by < bg.nbh; ++by)
            for (uint32_t bx = 0; bx < bg.nbw; ++bx) {
              Rect r = bg.block_rect(bx, by);
              DecBlock& d = h_dec_proto[bg.block_base + by * bg.nbw + bx];
              block_res[bg.block_base + by * bg.nbw + bx] = (uint8_t)(tc.res.size() - 1 - rg.res_num);
              if (!tile_mask.empty()) block_wanted[bg.block_base + by * bg.nbw + bx] = tile_wanted(t.idx) ? 1 : 0;
              memset(&d, 0, sizeof(d));
              d.dst_off = bg.plane_off + bg.plane_pad_x + (uint64_t)(r.y0 - bg.rect.y0) * bg.plane_stride + (r.x0 - bg.rect.x0);
              d.stride = bg.plane_stride; d.w = (uint16_t)r.w; d.h = (uint16_t)r.h;
              d.K_max = (uint8_t)bg.K_max; d.delta = bg.delta;
              d.flags = (params.stripe_causal(tc.comp) ? 1u : 0u) | (params.reversible(tc.comp) ? 0u : 2u);
              // quad records of the refinement passes (an even number of words: 8-byte aligned)
              uint32_t nq = (r.w + 1) / 2, qs = (nq + 1) & ~1u, nqr = (r.h + 1) / 2;
              d.scratch_off = scratch;
              scratch += (size_t)qs * nqr;
            }
        }
  scratch_words = scratch;
  if (!parse_only) d_scratch.reserve((scratch + 64) * 4);
  coded.assign(layout.num_blocks, CodedBlock());
  block_static.assign(layout.num_blocks, DecStatic());
  for (size_t b = 0; b < h_dec_proto.size(); ++b) {
    const DecBlock& d = h_dec_proto[b];
    DecStatic& g = block_static[b];
    g.flags = d.flags; g.K_max = d.K_max;
    DecBlock t = d; t.num_passes = 1; t.len1 = 2; t.missing_msbs = 0; t.K_max = 1;       // the frame's part of the test set to "yes"
    g.fast_shape = dec_block_is_fast(t) ? 1 : 0;
  }
  d_dec.reserve(std::max<size_t>(1, h_dec_proto.size()) * sizeof(DecBlock));
  d_proto.reserve(std::max<size_t>(1, h_dec_proto.size()) * sizeof(DecBlock));
  if (!h_dec_proto.empty())
    CK(cudaMemcpy(d_proto.p, h_dec_proto.data(), h_dec_proto.size() * sizeof(DecBlock), cudaMemcpyHostToDevice));
  h_dyn.reserve(std::max<size_t>(1, h_dec_proto.size()) * sizeof(DecDyn));
  any_rev_blocks = any_irv_blocks = false;
  for (const DecBlock& d : h_dec_proto) { if (d.flags & 2) any_irv_blocks = true; else any_rev_blocks = true; }
  d_bstatus.reserve(std::max<size_t>(1, h_dec_proto.size()) * 4);
  h_bstatus.reserve(std::max<size_t>(1, h_dec_proto.size()) * 4);
  header_sig = sig;
}

void Decoder::setup_geometry(uint32_t sample_type) {
  plan_image(sample_type);
  build_dwt_jobs(false, jobs, d_jobs);
}

void Decoder::restrict_resolution(uint32_t skipped_res_for_read, uint32_t skipped_res_for_recon) {
  // codestream::restrict_input_resolution (ojph_codestream_local.cpp:883-900)
  if (skipped_res_for_read < skipped_res_for_recon)
    fail(0x000300A1, "skipped_resolution for data %d must be equal or smaller than  skipped_resolution for "
         "reconstruction %d", skipped_res_for_read, skipped_res_for_recon);
  if (skipped_res_for_read > params.num_decomps)
    fail(0x000300A2, "skipped_resolution for data %d must be smaller than  the number of decomposition levels %d",
         skipped_res_for_read, params.num_decomps);
  // a component with its own (COC) decomposition count below the request: the reference's arithmetic wraps
  // (ojph_resolution.cpp:252-255) and what it then reads depends on the progression order; refused here
  for (uint32_t c = 0; c < params.num_comps(); ++c)
    if (skipped_res_for_read > params.decomps(c))
      fail(0x000B0007, "component %u has %u decomposition levels; %u cannot be skipped", c, params.decomps(c),
           skipped_res_for_read);
  if (skipped_res_for_read == skip_read && skipped_res_for_recon == skip_recon) return;
  skip_read = skipped_res_for_read; skip_recon = skipped_res_for_recon;
  setup_geometry(img_type);
}

void Decoder::info(FrameInfo& fi) const {
  memset(&fi, 0, sizeof(fi));
  fi.width = params.Xsiz; fi.height = params.Ysiz; fi.off_x = params.XOsiz; fi.off_y = params.YOsiz;
  fi.num_comps = params.num_comps();
  for (uint32_t c = 0; c < fi.num_comps && c < 16; ++c) {
    fi.bit_depth[c] = params.comps[c].bit_depth; fi.is_signed[c] = params.comps[c].is_signed;
    fi.dx[c] = params.comps[c].dx; fi.dy[c] = params.comps[c].dy;
    fi.comp_w[c] = img_w[c]; fi.comp_h[c] = img_h[c];            // reconstruction size (restrict_resolution)
    fi.nlt_type[c] = params.nlt_type(c);
  }
  // COD values (components may differ: COC)
  fi.num_decomps = params.num_decomps; fi.reversible = params.reversible();
  fi.color_transform = params.color_transform();
  fi.num_tiles = (uint32_t)layout.tiles.size();
}

void Decoder::parse_tiles() {
  // tile-part loop of codestream::read (ojph_codestream_local.cpp:912-1115) and
  // tile::parse_tile_header (ojph_tile.cpp:777-936)
  for (CodedBlock& cb : coded) cb = CodedBlock();
  size_t ntiles = layout.tiles.size();
  std::vector<std::vector<PacketRef>> seqs(ntiles);
  std::vector<uint32_t> next_pkt(ntiles, 0), next_tp(ntiles, 0);
  std::vector<bool> have_seq(ntiles, false);
  tp_starts.assign(ntiles, std::vector<uint32_t>());
  tp_segments = 0;
  size_t pos = first_sot;
  const uint8_t* d = j2c;
  HostMirror* hm = mirrored ? &mirror : nullptr;
  while (pos + 2 <= j2c_len) {
    // find SOT or EOC
    if (hm) hm->need(pos, 12);
    if (!(d[pos] == 0xFF && (d[pos + 1] == 0x90 || d[pos + 1] == 0xD9))) { ++pos; continue; }
    if (d[pos + 1] == 0xD9) break;
    if (pos + 12 > j2c_len) {
      if (resilient) break;
      fail(0x00050091, "error reading SOT marker");
    }
    uint32_t Lsot = ((uint32_t)d[pos + 2] << 8) | d[pos + 3];
    uint32_t Isot = ((uint32_t)d[pos + 4] << 8) | d[pos + 5];
    uint32_t Psot = ((uint32_t)d[pos + 6] << 24) | ((uint32_t)d[pos + 7] << 16) | ((uint32_t)d[pos + 8] << 8) | d[pos + 9];
    uint32_t TPsot = d[pos + 10], TNsot = d[pos + 11];
    (void)TNsot;
    if (Lsot != 10) { if (resilient) { pos += 2; continue; } fail(0x00050092, "error in SOT length"); }
    size_t tile_start = pos + 12;          // file position after the SOT segment
    size_t tp_end = Psot ? pos + Psot : j2c_len;
    if (tp_end > j2c_len) tp_end = j2c_len;
    if (Isot >= ntiles) {
      if (!resilient) fail(0x00030061, "wrong tile index");
      pos = tp_end; continue;
    }
    if (!tile_wanted(Isot)) { pos = tp_end; continue; }          // another rank's tile
    // skip tile-part header segments up to SOD
    size_t q = tile_start; bool sod = false;
    while (q + 2 <= tp_end) {
      if (hm) hm->need(q, 4);
      if (d[q] != 0xFF) { ++q; continue; }
      uint8_t m = d[q + 1];
      if (m == 0x93) { sod = true; q += 2; break; }
      bool seg = (m == 0x52 || m == 0x53 || m == 0x5C || m == 0x5D || m == 0x5E || m == 0x5F || m == 0x61 ||
                  m == 0x58 || m == 0x64 || m == 0x76);
      if (!seg) { ++q; continue; }
      tp_segments |= (m == 0x61 || m == 0x5F) ? 2u : (m != 0x58 ? 1u : 0u);
      if (q + 4 > tp_end) break;
      uint32_t L = ((uint32_t)d[q + 2] << 8) | d[q + 3];
      q += 2 + L;
    }
    if (!sod) {
      if (!resilient) fail(0x00030063, "File terminated early before start of data is found for tile "
                           "indexed %d and tile part %d", Isot, TPsot);
      pos = tp_end; continue;
    }
    if (TPsot != next_tp[Isot]) {
      if (!resilient) fail(0x00030091, "wrong tile part index");
    }
    ++next_tp[Isot];
    uint32_t payload = Psot ? Psot - 12 : (uint32_t)(j2c_len - tile_start);
    uint32_t data_left = payload - (uint32_t)(q - tile_start);     // what Psot promises, not what the buffer holds
    if (!have_seq[Isot]) { std::vector<uint32_t> tpf; layout.packet_sequence(Isot, seqs[Isot], tpf); have_seq[Isot] = true; }
    tp_starts[Isot].push_back(next_pkt[Isot]);
    try {
      std::vector<PacketRef>& seq = seqs[Isot];
      while (data_left > 0 && next_pkt[Isot] < seq.size()) {
        const PacketRef& pr = seq[next_pkt[Isot]++];
        const ResGeom& rg = layout.res_of(pr);
        parse_packet(params, rg, rg.precincts[pr.precinct], coded.data(), d, q, data_left, j2c_len, hm);
      }
    } catch (const Error& e) {
      if (!resilient) throw;
    }
    pos = tp_end;
  }
  pkts_read = next_pkt;
}

// the frame's part of every block record (the geometry part sits in d_proto): lengths, passes, missing msbs, where
// the bytes are, and whether the block goes through the specialised kernel (one output type per launch).
// (the geometry a block's record needs here -- static flags, whether its shape suits the specialised kernel --
// sits in 4 bytes per block, block_static, instead of the 48-byte DecBlock prototype)
BlockFrame Decoder::frame_records(uint32_t dec_out, DecDyn* hy) {
  BlockFrame f; f.dec_out = dec_out;
  const uint32_t nb = (uint32_t)h_dec_proto.size();
  const bool fast_ok = dec_out != DEC_OUT_PER_BLOCK && !no_fast_blocks && !wide;
  const bool masked = !block_wanted.empty(), restricted = skip_read > 0;
  const DecStatic* bst = block_static.data();
  for (uint32_t b = 0; b < nb; ++b) {
    const CodedBlock& cb = coded[b];
    const DecStatic g = bst[b];
    uint32_t len1 = cb.pass_len[0], len2 = cb.pass_len[1], np = cb.num_passes;
    const uint32_t mm = cb.missing_msbs;
    bool skip = false;
    if (masked && !block_wanted[b]) { np = 0; len1 = len2 = 0; skip = true; }   // another rank's tile / rows
    if (restricted && block_res[b] < skip_read) {            // resolution not read: its bands are zero ...
      np = 0; len1 = len2 = 0;
      if (block_res[b] < skip_recon) skip = true;            // ... and not even needed: nothing to fill
    }
    if (np > 1) f.cleanup_only = false;
    uint32_t flags = g.flags;
    // dec_block_is_fast(): the shape part is g.fast_shape, the frame's part is checked here
    if (fast_ok && g.fast_shape && !skip && np == 1 && len1 >= 2 && mm + 2u <= 16u && g.K_max > mm) { flags |= DEC_FLAG_FAST; ++f.nfast; }
    DecDyn y; y.data_off = cb.data_off; y.len1 = (uint16_t)len1; y.len2 = (uint16_t)len2;
    y.num_passes = (uint8_t)np; y.missing_msbs = (uint8_t)mm; y.flags = (uint8_t)flags; y.skip = skip ? 1 : 0;
    hy[b] = y;
  }
  return f;
}

// the block decoders of one frame into the arena coef: records merged from hy, then the kernels (launches counted)
void Decoder::enqueue_blocks(const BlockFrame& f, const DecDyn* hy, const uint8_t* cs, uint32_t* coef, cudaStream_t st,
                             const SideStream* sd, uint32_t& launches) {
  const uint32_t nb = (uint32_t)h_dec_proto.size();
  if (nb) { launch_dec_merge(d_dec.as<DecBlock>(), out_proto ? out_proto : d_proto.as<DecBlock>(), hy, nb, st); ++launches; }
  if (wide) {
    if (!f.cleanup_only) fail(0x000B0009, "SigProp / MagRef passes are not implemented on the 64-bit coefficient path");
    launch_ht_decode_wide(d_dec.as<DecBlock>(), nb, max_block_w, cs, coef, d_tables_dec.as<uint16_t>(), false,
                          d_bstatus.as<uint32_t>(), st);
  } else {
    if (!f.cleanup_only) d_scratch.reserve((scratch_words + 64) * 4);
    launch_ht_decode_serial(d_dec.as<DecBlock>(), nb, f.nfast, max_block_w, cs, coef, d_scratch.as<uint32_t>(),
                            d_tables_dec.as<uint16_t>(), f.dec_out, f.cleanup_only,
                            d_bstatus.as<uint32_t>(), st, sd);
  }
  launches += 1 + (f.nfast ? 1 : 0) + (f.nfast < nb ? 1 : 0);
}

uint32_t Decoder::decode(void* const* planes, const uint32_t* strides, bool caller_image) {
  const Params& P = params;
  uint32_t nc = P.num_comps(), es = esize_of(img_type);
  last_launches = 0;
  // codestream to the device while the host parses packet headers
  mark(0);
  const uint8_t* cs_dev = dev_cs;
  if (cs_dev == nullptr) {
    d_cs.reserve(j2c_len + 64);
    if (tile_mask.empty())
      CK(cudaMemcpyAsync(d_cs.p, j2c, j2c_len, cudaMemcpyHostToDevice, stream));
    else {
      // only the tile-parts of this object's tiles, at their own offsets (walk the SOT chain by Psot)
      size_t pos = first_sot;
      while (pos + 12 <= j2c_len && j2c[pos] == 0xFF && j2c[pos + 1] == 0x90) {
        const uint32_t Isot = ((uint32_t)j2c[pos + 4] << 8) | j2c[pos + 5];
        const uint32_t Psot = ((uint32_t)j2c[pos + 6] << 24) | ((uint32_t)j2c[pos + 7] << 16) | ((uint32_t)j2c[pos + 8] << 8) | j2c[pos + 9];
        const size_t end = (Psot && pos + Psot <= j2c_len) ? pos + Psot : j2c_len;
        if (tile_wanted(Isot))
          CK(cudaMemcpyAsync(d_cs.as<uint8_t>() + pos, j2c + pos, end - pos, cudaMemcpyHostToDevice, stream));
        if (!Psot) break;
        pos = end;
      }
    }
    CK(cudaMemsetAsync(d_cs.as<uint8_t>() + j2c_len, 0, 32, stream));
    cs_dev = d_cs.as<uint8_t>();
  }
  mark(1);
  auto host_t0 = std::chrono::steady_clock::now();
  parse_tiles();
  auto host_t1 = std::chrono::steady_clock::now();
  if (mirrored) {
    mirror.last_pages.clear();
    for (size_t pg = 0; pg < mirror.present.size(); ++pg) if (mirror.present[pg]) mirror.last_pages.push_back(pg);
  }
  uint32_t nb = (uint32_t)h_dec_proto.size();
  DecDyn* hy = h_dyn.as<DecDyn>();
  const BlockFrame bf = frame_records(native_out(), hy);
  const uint32_t nfast = bf.nfast, dec_out = bf.dec_out;
  const bool cleanup_only = bf.cleanup_only;
  host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count();
  if (getenv("OJB_PARSE_PROF")) fprintf(stderr, "decode host: parse %.3f ms, records %.3f ms\n", std::chrono::duration<double, std::milli>(host_t1 - host_t0).count(), host_ms - std::chrono::duration<double, std::milli>(host_t1 - host_t0).count());
  auto enqueue = [&] {
  mark(2);
  enqueue_blocks(bf, hy, cs_dev, d_coef.as<uint32_t>(), stream, &side, last_launches);
  mark(3);
  if (nb) { launch_ctrl_copy(h_bstatus.p, d_bstatus.p, (size_t)nb * 4, stream); ++last_launches; }
  if (caller_image) enqueue_caller_image();
  enqueue_dwt(false, jobs, d_jobs, img_slot(caller_image), caller_image && caller_interleaved, d_coef.as<uint32_t>());
  mark(4);
  if (planes) {
    for (uint32_t c = 0; c < nc; ++c) {
      const uint8_t* s = d_image.as<uint8_t>() + img_off[c];
      uint32_t st = strides ? strides[c] : img_w[c];
      if (st == img_w[c])
        CK(cudaMemcpyAsync(planes[c], s, (size_t)img_w[c] * img_h[c] * es, cudaMemcpyDeviceToHost, stream));
      else
        for (uint32_t y = 0; y < img_h[c]; ++y)
          CK(cudaMemcpyAsync((uint8_t*)planes[c] + (size_t)y * st * es, s + (size_t)y * img_w[c] * es,
                             (size_t)img_w[c] * es, cudaMemcpyDeviceToHost, stream));
    }
  }
  mark(5);
  };
  // resident form (codestream in HBM, image stays there or goes to the caller's memory): what follows the host parse
  // replays as a graph -- the frame's own data (block records, lengths, offsets, where the caller's image is) reaches
  // the kernels through pinned buffers the graph copies in
  if (planes == nullptr && dev_cs != nullptr)
    run_frame({ (uint64_t)(size_t)cs_dev, (uint64_t)nb, (uint64_t)(nfast != 0), (uint64_t)(nfast < nb), (uint64_t)cleanup_only, (uint64_t)dec_out,
                (uint64_t)(size_t)d_scratch.p, (uint64_t)skip_recon, (uint64_t)(size_t)hy, (uint64_t)(size_t)d_coef.p, (uint64_t)(size_t)d_image.p,
                (uint64_t)(size_t)img_slot(caller_image), (uint64_t)(caller_image && caller_interleaved) }, enqueue);
  else enqueue();
  CK(cudaStreamSynchronize(stream));
  CK(cudaGetLastError());
  collect(6);
  failed_blocks = 0;
  const uint32_t* bs = h_bstatus.as<uint32_t>();
  for (uint32_t b = 0; b < nb; ++b) if (bs[b] & 1u) ++failed_blocks;
  if (failed_blocks && !resilient) fail(0x000300A1, "Error decoding a codeblock.");
  return failed_blocks;
}

} // namespace ojb

namespace ojb {

//------------------------------------------------------------------------------------------
// Transcoder (see ojb_codec.h)
//------------------------------------------------------------------------------------------
// The input's parse, what it refuses and the configuration it implies: the input's coding parameters, its main header
// without TLM / PLM, its tile-part division and whether it had a TLM -- or, with skipped_res = r > 0, the parameters and
// main header of the input with its top r resolution levels dropped (reduce_main_header), with the same tile-part
// division kind and TLM.  The encoder is configured again only when that changed, and only after every check passed,
// so a refused input leaves the encoder as it was.
void Encoder::transcode_parse(const uint8_t* j2c, size_t len, bool on_device, uint32_t sample_type, uint32_t skipped_res) {
  if (!src) { src.reset(new Decoder()); src->parse_only = true; }
  Decoder& D = *src;
  if (on_device) D.read_headers_device(j2c, len, sample_type); else D.read_headers(j2c, len, sample_type);
  // the dropped resolutions' blocks are skipped (Decoder::frame_records); restrict_resolution would also plan an image
  D.skip_read = D.skip_recon = skipped_res;
  if (D.params.uses_sop() || D.params.uses_eph())
    fail(0x000B004C, "the codestream uses SOP or EPH markers (Scod bits 1-2), which a transcode does not write");
  if (D.wide)
    fail(0x000B0050, "a transcode needs the 32-bit coefficient path: this configuration codes 64-bit coefficients");
  const uint8_t* d = D.j2c;
  std::vector<uint8_t> hdr(d, d + 2);              // SOC
  bool tlm = false;
  for (size_t q = 2; q < D.first_sot; ) {
    if (q + 4 > D.first_sot) fail(0x000B0051, "the codestream's main header is damaged");
    const uint32_t m = ((uint32_t)d[q] << 8) | d[q + 1], L = ((uint32_t)d[q + 2] << 8) | d[q + 3];
    if (q + 2 + L > D.first_sot) fail(0x000B0051, "the codestream's main header is damaged");
    if (m == M_POC || m == M_PPM)
      fail(0x000B004D, "the codestream has a %s segment, which changes where packet headers are or their order",
           m == M_POC ? "POC" : "PPM");
    if (m == M_TLM) tlm = true;
    else if (m != M_PLM) hdr.insert(hdr.end(), d + q, d + q + 2 + L);
    q += 2 + L;
  }
  try { D.parse_tiles(); }
  catch (const Error& e) { fail(0x000B0051, "the codestream is truncated or damaged: %s", e.what()); }
  if (D.tp_segments & 2u)
    fail(0x000B004D, "a tile-part header has a PPT or POC segment, which changes where packet headers are or their order");
  if (D.tp_segments & 1u)
    fail(0x000B004E, "a tile-part header carries a marker segment other than PLT; a transcode writes none");
  // the tile-part division: where the input's tile-parts start in each tile's packet sequence, against the four
  // divisions the header plan writes (none, resolutions, components, both)
  const uint32_t ntiles = (uint32_t)D.layout.tiles.size();
  std::vector<PacketRef> seq; std::vector<uint32_t> tpf;
  const uint32_t div0 = D.params.tilepart_div;
  int div = -1;
  for (uint32_t v = 0; v < 4 && div < 0; ++v) {
    D.params.tilepart_div = v;
    bool ok = true;
    for (uint32_t t = 0; t < ntiles && ok; ++t) {
      D.layout.packet_sequence(t, seq, tpf);
      if (D.pkts_read[t] < seq.size()) { D.params.tilepart_div = div0; fail(0x000B0051, "the codestream is truncated: tile %u lacks packets", t); }
      ok = tpf == D.tp_starts[t];
    }
    if (ok) div = (int)v;
  }
  D.params.tilepart_div = div0;
  if (div < 0)
    fail(0x000B004F, "the codestream's tile-parts follow none of the divisions a transcode writes (none, by resolution, by "
         "component, by both)");
  if (transcoding && hdr == xc_in_header && xc_skip == skipped_res && params.tilepart_div == (uint32_t)div &&
      params.need_tlm == tlm && img_type == sample_type)
    return;
  Params np;
  std::vector<uint8_t> out_hdr;
  if (skipped_res) {
    reduce_main_header(hdr, D.params, skipped_res, out_hdr, np);
    np.planar = np.color_transform() ? 0 : 1;       // as the decoder derives it (Decoder::read_headers)
  } else {
    np = D.params;
    out_hdr = hdr;
  }
  transcoding = false;                  // a failing setup leaves no half-configured transcoder
  D.out_proto = nullptr;
  params = np;
  params.tilepart_div = (uint32_t)div; params.need_tlm = tlm;
  main_header.swap(out_hdr);
  xc_in_header.swap(hdr);
  xc_skip = skipped_res;
  transcoding = true;
  try { setup(sample_type); plan_block_map(); } catch (...) { transcoding = false; throw; }
}

// The block correspondence of a transcode that drops resolution levels.  The input's blocks of resolution k <= D_c - r
// are the output's blocks of resolution k, band for band, with the same rectangles (reduce_main_header).  But the
// restricted decoder's arena does not match the encoder's: Layout::build lays each tile-component out from its finest
// resolution down, so the dropped resolutions' planes come first and push every kept plane to another offset, and the
// block numbers (band by band in the same order) shift the same way.  So each kept block's prototype gets the
// encoder's plane offset and stride, and the encoder's block b reads the decoder's record map[b].
void Encoder::plan_block_map() {
  Decoder& D = *src;
  D.out_proto = nullptr;
  if (xc_skip == 0) return;
  std::vector<uint32_t> map(layout.num_blocks, 0);
  std::vector<DecBlock> proto(D.h_dec_proto);
  auto same = [](const Rect& a, const Rect& b) { return a.x0 == b.x0 && a.y0 == b.y0 && a.w == b.w && a.h == b.h; };
  for (size_t t = 0; t < layout.tiles.size(); ++t)
    for (size_t c = 0; c < layout.tiles[t].comps.size(); ++c) {
      const TileCompGeom& ec = layout.tiles[t].comps[c];
      const TileCompGeom& dc = D.layout.tiles[t].comps[c];
      if (ec.res.size() + xc_skip != dc.res.size() || !same(ec.rect, dc.res[ec.res.size() - 1].rect))
        fail(0x000B0051, "internal: tile %zu component %zu of the reduced geometry is not the input's", t, c);
      for (size_t k = 0; k < ec.res.size(); ++k)
        for (uint32_t b = 0; b < 4; ++b) {
          const BandGeom& eb = ec.res[k].bands[b];
          const BandGeom& db = dc.res[k].bands[b];
          if (eb.empty != db.empty || (!eb.empty && (!same(eb.rect, db.rect) || eb.nbw != db.nbw || eb.nbh != db.nbh ||
                                                      eb.xcb != db.xcb || eb.ycb != db.ycb || eb.K_max != db.K_max)))
            fail(0x000B0051, "internal: band %u of resolution %zu of the reduced geometry is not the input's", b, k);
          if (eb.empty) continue;
          for (uint32_t by = 0; by < eb.nbh; ++by)
            for (uint32_t bx = 0; bx < eb.nbw; ++bx) {
              const uint32_t i = by * eb.nbw + bx;
              const Rect r = eb.block_rect(bx, by);
              DecBlock& p = proto[db.block_base + i];
              map[eb.block_base + i] = db.block_base + i;
              p.dst_off = eb.plane_off + eb.plane_pad_x + (uint64_t)(r.y0 - eb.rect.y0) * eb.plane_stride + (r.x0 - eb.rect.x0);
              p.stride = eb.plane_stride;
            }
        }
    }
  d_xmap.reserve(std::max<size_t>(1, map.size()) * 4);
  d_xproto.reserve(std::max<size_t>(1, proto.size()) * sizeof(DecBlock));
  if (!map.empty()) CK(cudaMemcpy(d_xmap.p, map.data(), map.size() * 4, cudaMemcpyHostToDevice));
  if (!proto.empty()) CK(cudaMemcpy(d_xproto.p, proto.data(), proto.size() * sizeof(DecBlock), cudaMemcpyHostToDevice));
  D.out_proto = d_xproto.as<DecBlock>();
}

void Encoder::transcode_headers(const uint8_t* j2c, size_t len, bool on_device, uint32_t sample_type, uint32_t skipped_res) {
  transcoding = false;
  transcode_parse(j2c, len, on_device, sample_type, skipped_res);
}

// the transform's place in the frame: the input to the device, [the source of a quality target: the input decoded as
// the decoder would, synthesised into d_image], the coded words into d_coef and the frame's block array
void Encoder::enqueue_transcode_front() {
  Decoder& D = *src;
  const uint32_t nb = (uint32_t)D.h_dec_proto.size();
  if (xc_cs == D.d_cs.as<uint8_t>()) {
    CK(cudaMemcpyAsync(D.d_cs.p, D.j2c, D.j2c_len, cudaMemcpyHostToDevice, stream));
    CK(cudaMemsetAsync(D.d_cs.as<uint8_t>() + D.j2c_len, 0, 32, stream));
  }
  if (rq_on() && rq_planned) {
    D.enqueue_blocks(xc_source, h_xdyn.as<DecDyn>(), xc_cs, d_rcoef.as<uint32_t>(), stream, &side, last_launches);
    // 32-bit coefficients: transcode_parse refuses an input on the 64-bit path
    enqueue_dwt(false, rq_jobs, d_rq_jobs, img_slot(false), false, d_rcoef.as<uint32_t>());
  }
  D.enqueue_blocks(xc_coded, D.h_dyn.as<DecDyn>(), xc_cs, d_coef.as<uint32_t>(), stream, &side, last_launches);
  if (nb) { launch_ctrl_copy(D.h_bstatus.p, D.d_bstatus.p, (size_t)nb * 4, stream); ++last_launches; }
  launch_transcode_blocks(d_blocks.as<EncBlock>(), D.d_dec.as<DecBlock>(), xc_skip ? d_xmap.as<uint32_t>() : nullptr,
                          (uint32_t)h_blocks.size(), d_xblocks.as<EncBlock>(), stream);
  ++last_launches;
}

size_t Encoder::transcode(const uint8_t* j2c, size_t len, bool on_device, uint8_t* out, size_t out_cap, bool out_on_device) {
  if (!transcoding)
    fail(0x000B0052, "a transcode needs ojb_enc_transcode_headers first: this encoder is not configured from a codestream");
  const auto t0 = std::chrono::steady_clock::now();
  transcode_parse(j2c, len, on_device, img_type, xc_skip);
  Decoder& D = *src;
  const uint32_t nb = (uint32_t)D.h_dec_proto.size();
  DecDyn* hy = D.h_dyn.as<DecDyn>();
  xc_coded = D.frame_records(DEC_OUT_CODED, hy);
  // what the block decoders and the encoder's slots rely on: every block's bytes inside the stream, and its lowest
  // coded plane q_b at or above its band's least significant one (31 - K_max)
  xc_two_pass = false;
  for (uint32_t b = 0; b < nb; ++b) {
    const DecDyn& y = hy[b];
    if (y.num_passes == 0 || y.len1 == 0) continue;
    if (y.data_off + y.len1 + y.len2 > len) fail(0x000B0051, "the codestream is truncated: code-block %u runs past its end", b);
    const bool refined = y.num_passes > 1 && y.len2 != 0 && y.missing_msbs < 29;
    if (y.missing_msbs >= 30 || (refined ? 29u : 30u) - y.missing_msbs < 31u - D.block_static[b].K_max)
      fail(0x000B0051, "code-block %u of the codestream cannot be decoded: %u missing MSBs", b, (uint32_t)y.missing_msbs);
    if (refined && y.num_passes == 2) xc_two_pass = true;
  }
  if (rq_on()) {
    h_xdyn.reserve(std::max<size_t>(1, nb) * sizeof(DecDyn));
    xc_source = D.frame_records(D.native_out(), h_xdyn.as<DecDyn>());
  }
  if (on_device) xc_cs = j2c;
  else { D.d_cs.reserve(len + 64); xc_cs = D.d_cs.as<uint8_t>(); }
  const float parse_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
  const Frame f = begin_frame(Frame::TRANSCODE, true);
  const size_t n = device_headers ? finish_device(f, out, out_cap, out_on_device) : finish_host(f, out, out_cap, out_on_device);
  host_ms = parse_ms;
  const uint32_t* bs = D.h_bstatus.as<uint32_t>();
  for (uint32_t b = 0; b < nb; ++b)
    if (bs[b] & 1u) fail(0x000B0051, "code-block %u of the codestream failed to decode", b);
  return n;
}

} // namespace ojb
