// ojb_capi.cpp -- the extern "C" surface declared in include/ojph_b200.h.
#include "../../include/ojph_b200.h"
#include "ojb_codec.h"
#include <cstring>
#include <new>
#include <algorithm>

using namespace ojb;

// an object belongs to the device that was current when it was created; every entry point makes
// that device current again, so objects may be driven from any host thread
static int current_device() { int d = 0; cudaGetDevice(&d); return d; }
struct ojb_encoder { int device = current_device(); Encoder enc; bool configured = false; std::vector<Comment> comments; DeviceBuf d_raster; };
struct ojb_decoder {
  int device = current_device(); Decoder dec; bool have_headers = false;
  // line interface (pull): library-owned frame, cursor in the reference's line order
  PinnedBuf frame; std::vector<size_t> plane_off; std::vector<uint32_t> line_cur;
  uint32_t cur_comp = 0; int planar = -1; bool pulling = false;
  DeviceBuf d_raster;
};

static thread_local char g_err[1024] = "";

template <typename F> static int guarded(F&& f) {
  try { f(); return 0; }
  catch (const Error& e) { snprintf(g_err, sizeof(g_err), "%s", e.what()); return -(int)((e.code >> 16) ? (e.code >> 16) : 1); }
  catch (const std::bad_alloc&) { snprintf(g_err, sizeof(g_err), "ojph error: out of memory"); return -1000; }
  catch (const std::exception& e) { snprintf(g_err, sizeof(g_err), "%s", e.what()); return -1001; }
  catch (...) { snprintf(g_err, sizeof(g_err), "ojph error: unknown exception"); return -1002; }
}

static void to_params(const ojb_params* s, Params& P) {
  if (s->num_comps == 0 || s->num_comps > 16) fail(0x00040005, "wrong number of components");
  P = Params();
  P.Xsiz = s->width; P.Ysiz = s->height; P.XOsiz = s->off_x; P.YOsiz = s->off_y;
  P.XTsiz = s->tile_w; P.YTsiz = s->tile_h; P.XTOsiz = s->tile_off_x; P.YTOsiz = s->tile_off_y;
  P.comps.resize(s->num_comps);
  for (uint32_t c = 0; c < s->num_comps; ++c) {
    if (s->bit_depth[c] == 0 || s->bit_depth[c] > 32) fail(0x00040006, "wrong bit depth");
    if (s->dx[c] == 0 || s->dy[c] == 0 || s->dx[c] > 255 || s->dy[c] > 255) fail(0x00040007, "wrong component sub-sampling");
    P.comps[c].bit_depth = (uint8_t)s->bit_depth[c]; P.comps[c].is_signed = s->is_signed[c] != 0;
    P.comps[c].dx = (uint8_t)s->dx[c]; P.comps[c].dy = (uint8_t)s->dy[c];
  }
  if (s->num_decomps > 32) fail(0x00050001, "maximum number of decompositions cannot exceed 32");
  P.num_decomps = (uint8_t)s->num_decomps;
  P.set_block_dims(s->block_w, s->block_h);
  if (s->num_precincts) P.set_precincts((int)s->num_precincts, s->precinct_w, s->precinct_h);
  if (s->prog_order > 4) fail(0x00050031, "unknown progression order");
  P.prog_order = (uint8_t)s->prog_order;
  P.mc_trans = s->color_transform ? 1 : 0;
  P.wavelet = s->reversible ? DWT_REV53 : DWT_IRV97;
  if (!s->reversible) {
    if (s->qstep > 0.0f) P.qcd.base_delta = s->qstep;
    if (s->qfactor) {
      if (s->qfactor > 100) fail(0x00050181, "Qfactor must be between 1 and 100, but was set to %i.", s->qfactor);
      P.qcd.qfactor = (uint8_t)s->qfactor;
    }
  }
  {   // per-component quantisation calls, replayed in the order they were made (after the global ones)
    struct Call { uint32_t seq, comp, kind; };
    std::vector<Call> calls;
    for (uint32_t c = 0; c < 16; ++c) {
      if (s->qcc_calls[c] & 1u) calls.push_back(Call{ s->qcc_qstep_seq[c], c, 0 });
      if (s->qcc_calls[c] & 2u) calls.push_back(Call{ s->qcc_qfactor_seq[c], c, 1 });
    }
    std::stable_sort(calls.begin(), calls.end(), [](const Call& a, const Call& b) { return a.seq < b.seq; });
    for (const Call& k : calls) {
      QuantSet* q = P.find_qcc(k.comp);
      if (k.kind == 0) (q ? *q : P.qcd).base_delta = s->qcc_qstep[k.comp];        // set_delta(comp_idx, delta), :2011-2018
      else {
        if (s->qcc_qfactor[k.comp] < 1 || s->qcc_qfactor[k.comp] > 100)
          fail(0x00050191, "Qfactor must be between 1 and 100, but was set to %i.", s->qcc_qfactor[k.comp]);
        if (q == nullptr) q = &P.add_qcc(k.comp);
        q->qfactor = (uint8_t)s->qcc_qfactor[k.comp]; q->ctype = (int)std::min(s->qcc_ctype[k.comp], 2u);
      }
    }
  }
  for (uint32_t c = 0; c < s->num_comps; ++c) {
    if (!s->coc_present[c]) continue;
    CodStyle& cs = P.get_or_add_coc(c);
    if (s->coc_num_decomps[c] > 32) fail(0x00050001, "maximum number of decompositions cannot exceed 32");
    cs.num_decomps = (uint8_t)s->coc_num_decomps[c];
    Params tmp; tmp.set_block_dims(s->coc_block_w[c], s->coc_block_h[c]);      // same argument checks
    cs.cb_w_exp = tmp.cb_w_exp; cs.cb_h_exp = tmp.cb_h_exp;
    cs.wavelet = s->coc_reversible[c] ? DWT_REV53 : DWT_IRV97;
    if (s->coc_num_precincts[c]) {            // same argument checks as the COD form (ojph_params.cpp:188-213)
      Params t; t.num_decomps = cs.num_decomps;
      t.set_precincts((int)std::min(s->coc_num_precincts[c], 33u), s->coc_precinct_w[c], s->coc_precinct_h[c]);
      cs.Scoc |= 1;
      for (uint32_t i = 0; i <= cs.num_decomps; ++i) cs.precinct_size[i] = t.precinct_size[i];
    }
  }
  // NLT: the default entry, then the per-component calls in the order they were made
  if (s->nlt_all) P.set_nonlinear_transform(0xFFFF, s->nlt_all - 1);
  {
    uint32_t order[16], n = 0;
    for (uint32_t c = 0; c < 16; ++c) if (s->nlt_comp[c]) order[n++] = c;
    std::stable_sort(order, order + n, [&](uint32_t a, uint32_t b) { return s->nlt_seq[a] < s->nlt_seq[b]; });
    for (uint32_t i = 0; i < n; ++i) P.set_nonlinear_transform(order[i], s->nlt_comp[order[i]] - 1);
  }
  // Part 2 structures (this library's encoder extension)
  if (s->dfs_num_levels) {
    if (s->dfs_num_levels > 32) fail(0x000B0022, "at most 32 decomposition levels can be described");
    for (uint32_t i = 0; i < s->dfs_num_levels; ++i) P.enc_dfs.push_back((uint8_t)std::min(s->dfs_type[i], 255u));
  }
  if (s->atk_num_steps) {
    if (s->atk_num_steps > 8) fail(0x000B0023, "at most 8 lifting steps go through this structure");
    P.enc_atk_set = true;
    P.enc_atk.Satk = s->atk_reversible ? 0x1000 : 0;
    P.enc_atk.K = s->atk_reversible ? 1.0f : s->atk_K;
    if (!s->atk_reversible && !(s->atk_K > 0.0f)) fail(0x000B0023, "the kernel's scaling factor K must be positive");
    for (uint32_t i = 0; i < s->atk_num_steps; ++i) {
      AtkStep t; t.A = s->atk_A[i];
      if (s->atk_a[i] < -32768 || s->atk_a[i] > 32767 || s->atk_b[i] < -32768 || s->atk_b[i] > 32767 || s->atk_e[i] > 255)
        fail(0x000B0023, "reversible lifting parameters out of range");
      t.a = (int16_t)s->atk_a[i]; t.b = (int16_t)s->atk_b[i]; t.e = (uint8_t)s->atk_e[i];
      P.enc_atk.steps.push_back(t);
    }
    // the kernel decides reversibility for every component
    P.wavelet = s->atk_reversible ? DWT_REV53 : DWT_IRV97;
    if (!s->atk_reversible && s->qstep > 0.0f) P.qcd.base_delta = s->qstep;
  }
  if (s->profile > 2) fail(0x000300A1, "unkownn or unsupported profile");
  P.profile = s->profile;
  P.need_tlm = s->tlm != 0;
  P.tilepart_div = s->tilepart_div & 3u;
  P.planar = s->planar;
}

template <typename F> static int guarded_on(int device, F&& f) {
  return guarded([&] { cuda_check(cudaSetDevice(device), "cudaSetDevice"); f(); });
}

extern "C" {

const char* ojb_last_error(void) { return g_err; }
const char* ojb_version(void) { return "openjph_b200 0.1 (HTJ2K hot path of OpenJPH 0.31.0 on sm_90a)"; }

int ojb_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) return 0; return n; }
int ojb_set_device(int device) { return guarded([&] { cuda_check(cudaSetDevice(device), "cudaSetDevice"); }); }

void ojb_params_default(ojb_params* p) {
  memset(p, 0, sizeof(*p));
  p->num_comps = 1; p->bit_depth[0] = 8;
  for (int c = 0; c < 16; ++c) { p->dx[c] = 1; p->dy[c] = 1; p->bit_depth[c] = 8; }
  p->num_decomps = 5; p->block_w = 64; p->block_h = 64; p->prog_order = 2; p->planar = -1;
  for (int c = 0; c < 16; ++c) { p->coc_num_decomps[c] = 5; p->coc_block_w[c] = 64; p->coc_block_h[c] = 64; }
  p->qstep = -1.0f;
}

void ojb_params_to_internal(const ojb_params* s, Params& P) { to_params(s, P); }      // ojb_shard.cpp

void* ojb_host_alloc(uint64_t bytes) { void* p = nullptr; if (cudaMallocHost(&p, (size_t)bytes) != cudaSuccess) return nullptr; return p; }
void ojb_host_free(void* p) { if (p) cudaFreeHost(p); }

ojb_encoder* ojb_enc_create(void) {
  ojb_encoder* e = nullptr;
  guarded([&] { e = new ojb_encoder(); });
  return e;
}
void ojb_enc_destroy(ojb_encoder* e) { if (e) { cudaSetDevice(e->device); delete e; } }

int ojb_enc_configure(ojb_encoder* e, const ojb_params* p, uint32_t sample_type) {
  return guarded_on(e->device, [&] {
    if (sample_type > 2) fail(0x000B0012, "unknown sample container");
    Params P; to_params(p, P);
    P.comments = e->comments;
    e->configured = false;               // a failing configure leaves no half-built encoder behind
    e->enc.configure(P, sample_type);
    e->configured = true;
  });
}

int ojb_enc_set_comments(ojb_encoder* e, const ojb_comment* comments, uint32_t num_comments) {
  return guarded([&] {
    std::vector<Comment> v(num_comments);
    for (uint32_t i = 0; i < num_comments; ++i) {
      if (comments[i].len > 65531) fail(0x000500C1, "COM marker string length cannot be larger than 65531");
      const uint8_t* d = static_cast<const uint8_t*>(comments[i].data);
      v[i].data.assign(d, d + comments[i].len); v[i].Rcom = comments[i].rcom;
    }
    e->comments.swap(v);
  });
}

int32_t* ojb_enc_exchange(ojb_encoder* e, int32_t* line, uint32_t* next_comp) {
  int32_t* r = nullptr;
  guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    uint32_t nc = 0; r = e->enc.exchange(line, nc); if (next_comp) *next_comp = nc;
  });
  return r;
}

int ojb_enc_flush(ojb_encoder* e, uint8_t* out, uint64_t out_cap, uint64_t* out_len) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    Encoder& E = e->enc;
    uint32_t nc = E.params.num_comps();
    std::vector<const void*> pl(nc);
    // exchanged lines are si32; convert by temporarily treating the frame as an I32 image
    size_t o = 0;
    std::vector<uint32_t> w(nc), h(nc);
    for (uint32_t c = 0; c < nc; ++c) { w[c] = E.params.comp_width(c); h[c] = E.params.comp_height(c); }
    if (E.img_type != ST_I32) fail(0x000B0016, "the line interface needs the 32-bit sample container (OJB_I32)");
    for (uint32_t c = 0; c < nc; ++c) { pl[c] = E.h_frame.as<int32_t>() + o; o += (size_t)w[c] * h[c]; }
    *out_len = E.encode(pl.data(), nullptr, false, out, (size_t)out_cap, false);
  });
}

int ojb_enc_encode_frame(ojb_encoder* e, const void* const* planes, const uint32_t* strides,
                         uint8_t* out, uint64_t out_cap, uint64_t* out_len) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    *out_len = e->enc.encode(planes, strides, false, out, (size_t)out_cap, false);
  });
}

} // extern "C"

// file sample layouts (raster.cu)
namespace ojb {
static uint64_t raster_geometry(CodecBase& cb, uint32_t layout, uint32_t& es, RasterPlanes& pl) {
  const Params& P = cb.params;
  const uint32_t nc = P.num_comps();
  if (layout > 3) fail(0x000B0030, "unknown raster layout");
  if (cb.img_type == ST_I32) fail(0x000B0031, "file payloads need the 8-bit or 16-bit sample container");
  es = esize_of(cb.img_type);
  uint64_t total = 0;
  for (uint32_t c = 0; c < nc; ++c) {
    if ((P.comps[c].bit_depth > 8) != (es == 2))
      fail(0x000B0032, "component %u: %u-bit samples take %u byte(s) in the file; open the codec with the matching container",
           c, P.comps[c].bit_depth, P.comps[c].bit_depth > 8 ? 2u : 1u);
    total += (uint64_t)cb.img_w[c] * cb.img_h[c] * es;
  }
  if (layout == OJB_RASTER_DPX_BE || layout == OJB_RASTER_DPX_LE) {
    const uint32_t bd = P.comps[0].bit_depth;
    if (nc != 3 || (bd != 10 && bd != 16))
      fail(0x03000182, "DPX image formats other than 10-bit packed RGB and 16-bit RGB are not supported (as in the reference)");
    for (uint32_t c = 0; c < nc; ++c) {
      if (cb.img_w[c] != cb.img_w[0] || cb.img_h[c] != cb.img_h[0] || P.comps[c].bit_depth != bd)
        fail(0x000B0034, "a .dpx payload holds three equal components");
      pl.off[c] = cb.img_off[c]; pl.stride[c] = cb.img_w[c];
    }
    const uint64_t row = bd == 10 ? 4ull * cb.img_w[0] : 2ull * ((3ull * cb.img_w[0] + 1) & ~1ull);
    return row * cb.img_h[0];
  }
  if (layout == OJB_RASTER_PNM) {
    if (nc != 1 && nc != 3) fail(0x000B0033, "a .pgm / .ppm payload has 1 or 3 components");
    for (uint32_t c = 0; c < nc; ++c) {
      if (cb.img_w[c] != cb.img_w[0] || cb.img_h[c] != cb.img_h[0])
        fail(0x000B0034, "a .ppm payload cannot hold sub-sampled components");
      pl.off[c] = cb.img_off[c]; pl.stride[c] = cb.img_w[c];
    }
  }
  return total;
}
} // namespace ojb

extern "C" {

int ojb_enc_encode_raster(ojb_encoder* e, uint32_t layout, const void* payload, uint64_t payload_bytes,
                          uint8_t* out, uint64_t out_cap, uint64_t* out_len) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    Encoder& E = e->enc;
    if (E.transcoding) fail(0x000B0053, "this encoder was configured from a codestream: it transcodes, it has no image");
    uint32_t es = 0; RasterPlanes pl; memset(&pl, 0, sizeof(pl));
    const uint64_t need = raster_geometry(E, layout, es, pl);
    if (payload_bytes != need) fail(0x03000011, "not enough data: the frame takes %llu bytes, got %llu",
                                    (unsigned long long)need, (unsigned long long)payload_bytes);
    const uint32_t nc = E.params.num_comps();
    if (layout == OJB_RASTER_YUV) {
      std::vector<const void*> planes(nc);
      const uint8_t* p = static_cast<const uint8_t*>(payload);
      for (uint32_t c = 0; c < nc; ++c) { planes[c] = p; p += (size_t)E.img_w[c] * E.img_h[c] * es; }
      *out_len = E.encode(planes.data(), nullptr, false, out, (size_t)out_cap, false);
      return;
    }
    e->d_raster.reserve(std::max<uint64_t>(need, 16));
    cuda_check(cudaMemcpyAsync(e->d_raster.p, payload, need, cudaMemcpyHostToDevice, E.stream), "upload");
    if (layout == OJB_RASTER_PNM) launch_raster_unpack(e->d_raster.p, E.d_image.p, pl, nc, es, E.img_w[0], E.img_h[0], E.stream);
    else {                                      // words / samples are extracted in the GPU's (little-endian) order
      launch_raster_unpack_dpx(e->d_raster.p, E.d_image.p, pl, E.params.comps[0].bit_depth, layout == OJB_RASTER_DPX_BE,
                               E.img_w[0], E.img_h[0], E.stream);
    }
    *out_len = E.encode(nullptr, nullptr, false, out, (size_t)out_cap, false);
    E.last_launches += 1;
  });
}

int ojb_dec_decode_raster(ojb_decoder* d, uint32_t layout, void* payload, uint64_t payload_cap, uint64_t* payload_bytes) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    Decoder& D = d->dec;
    uint32_t es = 0; RasterPlanes pl; memset(&pl, 0, sizeof(pl));
    const uint64_t need = raster_geometry(D, layout, es, pl);
    if (payload_cap < need) fail(0x000B0035, "payload buffer too small: %llu bytes needed", (unsigned long long)need);
    const uint32_t nc = D.params.num_comps();
    if (layout > OJB_RASTER_YUV) fail(0x000B0037, "the .dpx layout is read-only, as in the reference");
    if (layout == OJB_RASTER_YUV) {
      std::vector<void*> planes(nc);
      uint8_t* p = static_cast<uint8_t*>(payload);
      for (uint32_t c = 0; c < nc; ++c) { planes[c] = p; p += (size_t)D.img_w[c] * D.img_h[c] * es; }
      D.decode(planes.data(), nullptr, false);
    } else {
      D.decode(nullptr, nullptr, false);
      d->d_raster.reserve(std::max<uint64_t>(need, 16));
      launch_raster_pack(d->d_raster.p, D.d_image.p, pl, nc, es, D.img_w[0], D.img_h[0], D.stream);
      cuda_check(cudaMemcpyAsync(payload, d->d_raster.p, need, cudaMemcpyDeviceToHost, D.stream), "download");
      cuda_check(cudaStreamSynchronize(D.stream), "raster pack");
      D.last_launches += 1;
    }
    *payload_bytes = need;
  });
}

} // extern "C"

// device-side accessors
namespace ojb {
static void* img_plane(CodecBase& cb, uint32_t c) { return cb.d_image.as<uint8_t>() + cb.img_off[c]; }
// the caller's image (ojb_device_image) checked against the component sizes of ojb_frame_info
static void caller_image(const CodecBase& cb, const ojb_device_image* in, std::vector<ImgComp>& comps) {
  const uint32_t nc = cb.params.num_comps();
  const uint64_t es = esize_of(cb.img_type);
  comps.assign(nc, ImgComp());
  for (uint32_t c = 0; c < nc; ++c) {
    const uint64_t base = in ? (uint64_t)(uintptr_t)in->base[c] : 0, pitch = in ? in->row_pitch[c] : 0;
    if (base == 0) fail(0x000B003B, "component %u: null base address", c);
    if (base % es || pitch % es)
      fail(0x000B003B, "component %u: base address or row pitch is not a multiple of the %u-byte sample", c, (uint32_t)es);
    const uint32_t col = in->col_stride[c], w = cb.img_w[c], h = cb.img_h[c];
    if (col == 0) fail(0x000B003C, "component %u: column stride 0", c);
    comps[c].base = base; comps[c].pitch = pitch; comps[c].col = col; comps[c].pad = 0;
    if (w == 0 || h == 0) continue;
    const unsigned __int128 row = ((unsigned __int128)(w - 1) * col + 1) * es;
    if (h > 1 && (unsigned __int128)pitch < row)
      fail(0x000B003D, "component %u: row pitch of %llu bytes is smaller than one row of %u samples at column stride %u",
           c, (unsigned long long)pitch, w, col);
    if ((unsigned __int128)(h - 1) * pitch + row >= ((unsigned __int128)1 << 32))
      fail(0x000B003E, "component %u: the %u x %u samples span 4 GiB or more (offsets from base are formed in 32 bits)", c, w, h);
  }
}
static void read_band(CodecBase& cb, uint32_t tile, uint32_t comp, uint32_t res, uint32_t band, uint32_t* out,
                      uint32_t* bw, uint32_t* bh) {
  if (tile >= cb.layout.tiles.size() || comp >= cb.params.num_comps() || res > cb.params.decomps(comp) || band > 3)
    fail(0x000B0014, "no such sub-band");
  const BandGeom& bg = cb.layout.tiles[tile].comps[comp].res[res].bands[band];
  *bw = bg.rect.w; *bh = bg.rect.h;
  if (bg.empty || out == nullptr) return;
  if (cb.wide) fail(0x000B0016, "the band parity hook reads 32-bit planes only");
  for (uint32_t y = 0; y < bg.rect.h; ++y)
    cuda_check(cudaMemcpy(out + (size_t)y * bg.rect.w,
                          cb.d_coef.as<uint32_t>() + bg.plane_off + bg.plane_pad_x + (size_t)y * bg.plane_stride,
                          (size_t)bg.rect.w * 4, cudaMemcpyDeviceToHost), "read_band");
}
}

extern "C" {

void* ojb_enc_device_plane(ojb_encoder* e, uint32_t comp) {
  if (!e->configured || e->enc.transcoding || comp >= e->enc.params.num_comps()) return nullptr;
  return img_plane(e->enc, comp);
}
int ojb_enc_upload_frame(ojb_encoder* e, const void* const* planes, const uint32_t* strides) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    if (e->enc.transcoding) fail(0x000B0053, "this encoder was configured from a codestream: it transcodes, it has no image");
    e->enc.upload_planes(planes, strides);
    cuda_check(cudaStreamSynchronize(e->enc.stream), "upload sync");
  });
}
int ojb_enc_encode_device(ojb_encoder* e, const ojb_device_image* in, void* cuda_stream,
                          uint8_t* out, uint64_t out_cap, uint64_t* out_len, int out_on_device) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B003F, "encoder is not configured");
    std::vector<ImgComp> comps;
    caller_image(e->enc, in, comps);
    e->enc.use_caller_image(comps.data(), static_cast<cudaStream_t>(cuda_stream));
    *out_len = e->enc.encode(nullptr, nullptr, true, out, (size_t)out_cap, out_on_device != 0);
  });
}
int ojb_enc_encode_resident(ojb_encoder* e, uint8_t* out, uint64_t out_cap, uint64_t* out_len, int out_on_device) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    *out_len = e->enc.encode(nullptr, nullptr, false, out, (size_t)out_cap, out_on_device != 0);
  });
}
uint32_t ojb_enc_kernel_launches(ojb_encoder* e) { return e->enc.last_launches; }
int ojb_enc_set_target_size(ojb_encoder* e, uint64_t bytes) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    e->enc.set_target(bytes);
  });
}
int ojb_enc_min_size(ojb_encoder* e, uint64_t* bytes) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    *bytes = e->enc.min_bytes;
  });
}
int ojb_enc_rate_info(ojb_encoder* e, uint32_t* num_blocks, uint32_t* kc, uint8_t* kmax, uint8_t* k, uint32_t* R,
                      double* D, uint64_t* info5, float* ms4) {
  return guarded_on(e->device, [&] {
    Encoder& E = e->enc;
    if (!e->configured || E.rc_kc == 0) fail(0x000B0013, "no frame has been encoded with a target size");
    const uint32_t nb = (uint32_t)E.h_blocks.size(), n = E.rc_kc;
    *num_blocks = nb; *kc = n;
    const RcTables& t = E.rc;
    // where each block's candidates start: 31 - K_max, or for a transcode the input's lowest coded plane q_b
    std::vector<EncBlock> xb;
    if (E.transcoding && nb) {
      xb.resize(nb);
      cuda_check(cudaMemcpy(xb.data(), E.d_xblocks.p, (size_t)nb * sizeof(EncBlock), cudaMemcpyDeviceToHost), "rate_info");
    }
    const EncBlock* blk = xb.empty() ? E.h_blocks.data() : xb.data();
    if (kmax) for (uint32_t b = 0; b < nb; ++b) kmax[b] = (uint8_t)(31u - blk[b].p);
    if (k) cuda_check(cudaMemcpy(k, t.chosen, nb, cudaMemcpyDeviceToHost), "rate_info");
    if (R) {
      std::vector<EncResult> c((size_t)nb * n); std::vector<uint8_t> nc(nb);
      cuda_check(cudaMemcpy(c.data(), t.cand, c.size() * sizeof(EncResult), cudaMemcpyDeviceToHost), "rate_info");
      cuda_check(cudaMemcpy(nc.data(), t.ncand, nb, cudaMemcpyDeviceToHost), "rate_info");
      for (uint32_t b = 0; b < nb; ++b)
        for (uint32_t j = 0; j < n; ++j) {
          const EncResult& r = c[(size_t)b * n + j];
          R[(size_t)b * n + j] = j >= nc[b] ? 0u : (r.len_head == RC_LEN_INVALID ? RC_LEN_INVALID : r.len_head + r.len_tail);
        }
    }
    if (D) {
      cuda_check(cudaMemcpy(D, t.dist, (size_t)nb * n * 8, cudaMemcpyDeviceToHost), "rate_info");
      for (uint32_t b = 0; b < nb; ++b)
        for (uint32_t j = 32u - blk[b].p; j < n; ++j) D[(size_t)b * n + j] = 0.0;     // past K_max: not computed
    }
    if (info5) {
      RcState s; cuda_check(cudaMemcpy(&s, t.state, sizeof(s), cudaMemcpyDeviceToHost), "rate_info");
      info5[0] = (uint64_t)s.budget; info5[1] = s.rounds; info5[2] = s.total - s.body; info5[3] = s.total;
      info5[4] = s.thresh == 0xFFFFFFFFu ? (1ull << 32) : s.thresh;
    }
    if (ms4) for (int i = 0; i < 4; ++i) ms4[i] = E.rc_ms[i];
  });
}
int ojb_enc_transcode_headers_reduced(ojb_encoder* e, const void* j2c, uint64_t len, int on_device, uint32_t sample_type,
                                      uint32_t skipped_res, ojb_frame_info* info) {
  return guarded_on(e->device, [&] {
    if (sample_type > 2) fail(0x000B0012, "unknown sample container");
    e->configured = false;               // a failing call leaves no half-built encoder behind
    e->enc.transcode_headers(static_cast<const uint8_t*>(j2c), (size_t)len, on_device != 0, sample_type, skipped_res);
    e->configured = true;
    if (info) {
      // the output's geometry: what a decoder of the transcoded stream reports
      const Params& P = e->enc.params;
      FrameInfo fi; memset(&fi, 0, sizeof(fi));
      fi.width = P.Xsiz; fi.height = P.Ysiz; fi.off_x = P.XOsiz; fi.off_y = P.YOsiz;
      fi.num_comps = P.num_comps();
      for (uint32_t c = 0; c < fi.num_comps && c < 16; ++c) {
        fi.bit_depth[c] = P.comps[c].bit_depth; fi.is_signed[c] = P.comps[c].is_signed;
        fi.dx[c] = P.comps[c].dx; fi.dy[c] = P.comps[c].dy;
        fi.comp_w[c] = P.comp_width(c); fi.comp_h[c] = P.comp_height(c);
        fi.nlt_type[c] = P.nlt_type(c);
      }
      fi.num_decomps = P.num_decomps; fi.reversible = P.reversible();
      fi.color_transform = P.color_transform();
      fi.num_tiles = (uint32_t)e->enc.layout.tiles.size();
      static_assert(sizeof(FrameInfo) == sizeof(ojb_frame_info), "frame info layout");
      memcpy(info, &fi, sizeof(fi));
    }
  });
}
int ojb_enc_transcode_headers(ojb_encoder* e, const void* j2c, uint64_t len, int on_device, uint32_t sample_type) {
  return ojb_enc_transcode_headers_reduced(e, j2c, len, on_device, sample_type, 0, nullptr);
}
int ojb_enc_transcode(ojb_encoder* e, const void* j2c, uint64_t len, int on_device,
                      uint8_t* out, uint64_t out_cap, uint64_t* out_len, int out_on_device) {
  return guarded_on(e->device, [&] {
    *out_len = e->enc.transcode(static_cast<const uint8_t*>(j2c), (size_t)len, on_device != 0, out, (size_t)out_cap,
                                out_on_device != 0);
  });
}
int ojb_enc_set_target_mse(ojb_encoder* e, double mse) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    e->enc.set_target_mse(mse);
  });
}
int ojb_enc_quality_info(ojb_encoder* e, ojb_quality_info* out) {
  return guarded_on(e->device, [&] {
    Encoder& E = e->enc;
    if (!e->configured || !E.rq_valid) fail(0x000B004B, "no frame has been encoded with a target quality");
    const RqState& q = *E.h_rq.as<RqState>();
    memset(out, 0, sizeof(*out));
    out->num_samples = E.rq_samples; out->limit = E.rq_limit;
    out->sse_lo = q.sse_pass[0]; out->sse_hi = q.sse_pass[1];
    out->num_comps = q.ncomp; out->reached = q.reached;
    for (uint32_t c = 0; c < q.ncomp && c < 16; ++c) out->comp_sse[c] = (double)q.comp_pass[c][1] * 18446744073709551616.0 + (double)q.comp_pass[c][0];
    out->rounds = std::min<uint32_t>(q.rounds, OJB_QUALITY_MAX_ROUNDS);
    for (uint32_t r = 0; r < out->rounds; ++r) {
      out->round_key[r] = q.round[r].key; out->round_body[r] = q.round[r].body;
      out->round_sse_lo[r] = q.round[r].sse_lo; out->round_sse_hi[r] = q.round[r].sse_hi;
    }
    out->pass_key = q.t_pass; out->fail_key = q.t_fail; out->pass_body = q.body_pass; out->fail_body = q.body_fail;
    out->pass_measured = q.pass_measured; out->fail_measured = q.fail_measured; out->body0 = q.body0;
    out->model_round1 = q.model1;
    out->ms_candidates = E.rq_ms[0]; out->ms_rounds = E.rq_ms[1]; out->ms_final = E.rq_ms[2];
  });
}
void ojb_enc_timings(ojb_encoder* e, float* ms8) {
  for (int i = 0; i < 7; ++i) ms8[i] = e->enc.stage_ms[i];
  ms8[7] = (float)e->enc.host_ms;
}
void ojb_dec_timings(ojb_decoder* d, float* ms8) {
  for (int i = 0; i < 5; ++i) ms8[i] = d->dec.stage_ms[i];
  ms8[5] = ms8[6] = 0; ms8[7] = (float)d->dec.host_ms;
}
// absolute positions of the stage marks of the last call on a device-wide time axis (ms since the first
// call of this function family): lets a tool see which kernels of different codec objects ran concurrently
static cudaEvent_t g_ref_event = nullptr;
static void marks_of(CodecBase& cb, int n, float* out) {
  for (int i = 0; i < n; ++i) { out[i] = -1.0f; if (g_ref_event) cudaEventElapsedTime(&out[i], g_ref_event, cb.ev[i]); }
}
int ojb_marks_reference(void) {
  return guarded([&] {
    if (g_ref_event == nullptr) { cuda_check(cudaEventCreate(&g_ref_event), "event"); }
    cuda_check(cudaEventRecord(g_ref_event, 0), "record"); cuda_check(cudaEventSynchronize(g_ref_event), "sync");
  });
}
void ojb_enc_marks(ojb_encoder* e, float* ms8) { marks_of(e->enc, 8, ms8); }
void ojb_dec_marks(ojb_decoder* d, float* ms8) { marks_of(d->dec, 6, ms8); ms8[6] = ms8[7] = -1.0f; }
uint32_t ojb_enc_num_blocks(ojb_encoder* e) { return e->configured ? e->enc.layout.num_blocks : 0; }
int ojb_enc_read_band(ojb_encoder* e, uint32_t tile, uint32_t comp, uint32_t res, uint32_t band,
                      uint32_t* out, uint32_t* band_w, uint32_t* band_h) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    read_band(e->enc, tile, comp, res, band, out, band_w, band_h);
  });
}

int ojb_enc_band_info(ojb_encoder* e, uint32_t tile, uint32_t comp, uint32_t res, uint32_t band, uint32_t* info8, float* delta) {
  return guarded_on(e->device, [&] {
    if (!e->configured) fail(0x000B0013, "encoder is not configured");
    CodecBase& cb = e->enc;
    if (tile >= cb.layout.tiles.size() || comp >= cb.params.num_comps() || res > cb.params.decomps(comp) || band > 3)
      fail(0x000B0014, "no such sub-band");
    const ResGeom& rg = cb.layout.tiles[tile].comps[comp].res[res];
    const BandGeom& bg = rg.bands[band];
    info8[0] = bg.rect.x0; info8[1] = bg.rect.y0; info8[2] = bg.rect.w; info8[3] = bg.rect.h;
    info8[4] = bg.K_max; info8[5] = rg.rect.x0; info8[6] = rg.rect.y0; info8[7] = bg.empty ? 0u : bg.nbw * bg.nbh;
    delta[0] = bg.delta; delta[1] = bg.delta_inv;
  });
}

ojb_decoder* ojb_dec_create(void) {
  ojb_decoder* d = nullptr;
  guarded([&] { d = new ojb_decoder(); });
  return d;
}
void ojb_dec_destroy(ojb_decoder* d) { if (d) { cudaSetDevice(d->device); delete d; } }
int ojb_dec_enable_resilience(ojb_decoder* d) { d->dec.resilient = true; return 0; }

int ojb_dec_read_headers(ojb_decoder* d, const uint8_t* j2c, uint64_t len, uint32_t sample_type,
                         ojb_frame_info* info) {
  return guarded_on(d->device, [&] {
    if (sample_type > 2) fail(0x000B0012, "unknown sample container");
    d->have_headers = false;             // a failing read_headers leaves no half-built decoder behind
    d->dec.read_headers(j2c, (size_t)len, sample_type);
    d->have_headers = true;
    if (info) {
      FrameInfo fi; d->dec.info(fi);
      static_assert(sizeof(FrameInfo) == sizeof(ojb_frame_info), "frame info layout");
      memcpy(info, &fi, sizeof(fi));
    }
  });
}
int ojb_dec_restrict_input_resolution(ojb_decoder* d, uint32_t skip_read, uint32_t skip_recon, ojb_frame_info* info) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    d->dec.restrict_resolution(skip_read, skip_recon);
    d->pulling = false;
    if (info) { FrameInfo fi; d->dec.info(fi); memcpy(info, &fi, sizeof(fi)); }
  });
}
int ojb_dec_decode_frame(ojb_decoder* d, void* const* planes, const uint32_t* strides) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    d->dec.decode(planes, strides, false);
  });
}
int ojb_dec_get_coding_style(ojb_decoder* d, uint32_t comp, ojb_coding_style* out) {
  return guarded([&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    const Params& P = d->dec.params;
    if (comp >= P.num_comps()) fail(0x000B0036, "component %u does not exist", comp);
    memset(out, 0, sizeof(*out));
    out->num_decomps = P.decomps(comp); out->reversible = P.reversible(comp) ? 1u : 0u;
    out->color_transform = P.color_transform() ? 1u : 0u;
    out->block_w = 1u << P.log_cb_w(comp); out->block_h = 1u << P.log_cb_h(comp);
    for (uint32_t r = 0; r <= P.decomps(comp) && r < 33; ++r) {
      out->precinct_w[r] = 1u << P.log_pp_w(comp, r); out->precinct_h[r] = 1u << P.log_pp_h(comp, r);
    }
    out->prog_order = P.prog_order; out->num_layers = P.num_layers;
    out->may_use_sop = P.uses_sop() ? 1u : 0u; out->use_eph = P.uses_eph() ? 1u : 0u;
    out->vertical_causality = P.stripe_causal(comp) ? 1u : 0u;
    out->tile_w = P.XTsiz; out->tile_h = P.YTsiz; out->tile_off_x = P.XTOsiz; out->tile_off_y = P.YTOsiz;
  });
}

int ojb_dec_set_planar(ojb_decoder* d, int planar) { d->planar = planar ? 1 : 0; return 0; }

int ojb_dec_begin_pull(ojb_decoder* d) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    Decoder& D = d->dec;
    if (D.img_type != ST_I32) fail(0x000B0016, "the line interface needs the 32-bit sample container (OJB_I32)");
    const uint32_t nc = D.params.num_comps();
    d->plane_off.assign(nc, 0);
    size_t tot = 0;
    for (uint32_t c = 0; c < nc; ++c) { d->plane_off[c] = tot; tot += (size_t)D.img_w[c] * D.img_h[c]; }
    d->frame.reserve(std::max<size_t>(tot, 1) * 4);
    std::vector<void*> pl(nc);
    for (uint32_t c = 0; c < nc; ++c) pl[c] = d->frame.as<int32_t>() + d->plane_off[c];
    D.decode(pl.data(), nullptr, false);
    d->line_cur.assign(nc, 0); d->cur_comp = 0; d->pulling = true;
    if (d->planar < 0) d->planar = D.params.mc_trans ? 0 : 1;
    // skip components without rows
    while (d->cur_comp < nc && D.img_h[d->cur_comp] == 0) ++d->cur_comp;
  });
}

const int32_t* ojb_dec_pull(ojb_decoder* d, uint32_t* comp_num) {
  const int32_t* line = nullptr;
  if (comp_num) *comp_num = 0;
  guarded([&] {
    if (!d->pulling) fail(0x000B0017, "ojb_dec_begin_pull has not been called");
    Decoder& D = d->dec;
    const uint32_t nc = D.params.num_comps();
    if (d->cur_comp >= nc) { d->pulling = false; return; }        // past the last line
    const uint32_t c = d->cur_comp;
    line = d->frame.as<int32_t>() + d->plane_off[c] + (size_t)d->line_cur[c] * D.img_w[c];
    if (comp_num) *comp_num = c;
    d->line_cur[c]++;
    if (d->planar == 1) {
      while (d->cur_comp < nc && d->line_cur[d->cur_comp] >= D.img_h[d->cur_comp]) ++d->cur_comp;
    } else {
      uint32_t tries = 0, k = c;
      do { k = (k + 1) % nc; ++tries; } while (d->line_cur[k] >= D.img_h[k] && tries <= nc);
      d->cur_comp = tries > nc ? nc : k;
    }
  });
  return line;
}

int ojb_dec_decode_resident(ojb_decoder* d) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    d->dec.decode(nullptr, nullptr, false);
  });
}
int ojb_dec_decode_device(ojb_decoder* d, const ojb_device_image* out, void* cuda_stream) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B003F, "read_headers has not been called");
    std::vector<ImgComp> comps;
    caller_image(d->dec, out, comps);
    d->dec.use_caller_image(comps.data(), static_cast<cudaStream_t>(cuda_stream));
    d->dec.decode(nullptr, nullptr, true);
  });
}
void* ojb_dec_device_plane(ojb_decoder* d, uint32_t comp) {
  if (!d->have_headers || comp >= d->dec.params.num_comps()) return nullptr;
  return img_plane(d->dec, comp);
}
int ojb_dec_read_headers_device(ojb_decoder* d, const void* dev_j2c, uint64_t len, uint32_t sample_type,
                                ojb_frame_info* info) {
  return guarded_on(d->device, [&] {
    if (sample_type > 2) fail(0x000B0012, "unknown sample container");
    d->have_headers = false;
    d->dec.read_headers_device(static_cast<const uint8_t*>(dev_j2c), (size_t)len, sample_type);
    d->have_headers = true;
    if (info) { FrameInfo fi; d->dec.info(fi); memcpy(info, &fi, sizeof(fi)); }
  });
}
uint64_t ojb_dec_mirror_bytes(ojb_decoder* d) { return d->dec.mirrored ? d->dec.mirror.fetched_bytes : 0; }
int ojb_dec_use_device_codestream(ojb_decoder* d, const void* dev_bytes) { d->dec.dev_cs = (const uint8_t*)dev_bytes; return 0; }
uint32_t ojb_dec_failed_blocks(ojb_decoder* d) { return d->dec.failed_blocks; }
int ojb_dec_list_blocks(ojb_decoder* d, ojb_block_desc* out, uint32_t cap, uint32_t* n) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    d->dec.parse_tiles();
    uint32_t nb = (uint32_t)d->dec.h_dec_proto.size();
    *n = nb;
    for (uint32_t i = 0; i < nb && i < cap; ++i) {
      const DecBlock& g = d->dec.h_dec_proto[i];
      const CodedBlock& cb = d->dec.coded[i];
      memset(&out[i], 0, sizeof(out[i]));
      out[i].w = g.w; out[i].h = g.h; out[i].stride = g.stride; out[i].sample_off = g.dst_off;
      out[i].missing_msbs = cb.missing_msbs; out[i].num_passes = cb.num_passes;
      out[i].len1 = cb.pass_len[0]; out[i].len2 = cb.pass_len[1]; out[i].byte_off = cb.data_off;
      out[i].causal = g.flags & 1;
    }
  });
}
uint32_t ojb_dec_kernel_launches(ojb_decoder* d) { return d->dec.last_launches; }
int ojb_dec_read_band(ojb_decoder* d, uint32_t tile, uint32_t comp, uint32_t res, uint32_t band,
                      uint32_t* out, uint32_t* band_w, uint32_t* band_h) {
  return guarded_on(d->device, [&] {
    if (!d->have_headers) fail(0x000B0015, "read_headers has not been called");
    read_band(d->dec, tile, comp, res, band, out, band_w, band_h);
  });
}

// ---- kernel-level batch entry points ------------------------------------------------------
int ojb_encode_blocks(const uint32_t* samples, uint64_t n_words, ojb_block_desc* desc, uint32_t n,
                      uint8_t* bytes, uint64_t bytes_cap, uint64_t* bytes_used) {
  return guarded([&] {
    DeviceBuf d_s, d_b, d_r, d_t, d_sl, d_st;
    d_s.reserve((n_words + 64) * 4);
    cuda_check(cudaMemcpy(d_s.p, samples, n_words * 4, cudaMemcpyHostToDevice), "samples");
    upload_ht_tables(true, d_t);
    std::vector<EncBlock> eb(n);
    uint64_t slot = 0;
    uint32_t nfast = 0;
    for (uint32_t i = 0; i < n; ++i) {
      if (desc[i].w == 0 || desc[i].h == 0 || desc[i].w > 1024 || desc[i].w * desc[i].h > 4096 || desc[i].missing_msbs > 29)
        fail(0x000B0021, "unsupported code-block geometry");
      eb[i].src_off = desc[i].sample_off; eb[i].stride = desc[i].stride; eb[i].w = (uint16_t)desc[i].w; eb[i].h = (uint16_t)desc[i].h;
      eb[i].p = (uint16_t)(30u - desc[i].missing_msbs);
      eb[i].slot_off = slot; eb[i].slot_cap = enc_slot_cap(desc[i].w, desc[i].h, desc[i].missing_msbs + 1, false);
      slot += eb[i].slot_cap;
      if (!getenv("OJB_NO_FAST_BLOCKS") && enc_block_is_fast(eb[i])) { eb[i].flags |= ENC_FLAG_FAST; ++nfast; }
    }
    d_b.reserve(n * sizeof(EncBlock)); d_r.reserve(n * sizeof(EncResult)); d_sl.reserve(slot + 64); d_st.reserve(64);
    cuda_check(cudaMemcpy(d_b.p, eb.data(), n * sizeof(EncBlock), cudaMemcpyHostToDevice), "blocks");
    cuda_check(cudaMemset(d_st.p, 0, 16), "status");
    uint32_t maxw = 4;
    for (uint32_t i = 0; i < n; ++i) maxw = std::max(maxw, desc[i].w);
    if (serial_block_encoder() || maxw > 64)
      launch_ht_encode_serial(d_b.as<EncBlock>(), n, nfast, maxw, d_s.as<uint32_t>(), d_sl.as<uint8_t>(), d_r.as<EncResult>(),
                     d_t.as<uint16_t>(), d_st.as<uint32_t>(), 0);
    else
      launch_ht_encode(d_b.as<EncBlock>(), n, d_s.as<uint32_t>(), d_sl.as<uint8_t>(), d_r.as<EncResult>(),
                     d_t.as<uint16_t>(), d_st.as<uint32_t>(), 0);
    cuda_check(cudaDeviceSynchronize(), "ht_encode");
    cuda_check(cudaGetLastError(), "ht_encode");
    std::vector<EncResult> res(n);
    cuda_check(cudaMemcpy(res.data(), d_r.p, n * sizeof(EncResult), cudaMemcpyDeviceToHost), "results");
    std::vector<uint8_t> sl(slot);
    cuda_check(cudaMemcpy(sl.data(), d_sl.p, slot, cudaMemcpyDeviceToHost), "slots");
    uint64_t pos = 0;
    for (uint32_t i = 0; i < n; ++i) {
      uint32_t len = res[i].len_head + res[i].len_tail;
      desc[i].byte_off = pos; desc[i].len1 = len; desc[i].len2 = 0; desc[i].status = len ? 0 : 1;
      if (pos + len > bytes_cap) fail(0x000B0030, "output buffer too small");
      memcpy(bytes + pos, sl.data() + eb[i].slot_off, res[i].len_head);
      memcpy(bytes + pos + res[i].len_head, sl.data() + eb[i].slot_off + eb[i].slot_cap - res[i].len_tail, res[i].len_tail);
      pos += len;
    }
    *bytes_used = pos;
  });
}

int ojb_decode_blocks(const uint8_t* bytes, uint64_t n_bytes, ojb_block_desc* desc, uint32_t n,
                      uint32_t* samples, uint64_t n_words) {
  return guarded([&] {
    DeviceBuf d_cs, d_b, d_t, d_o, d_sc, d_st;
    d_cs.reserve(n_bytes + 64);
    cuda_check(cudaMemset(d_cs.p, 0, d_cs.cap), "cs");
    cuda_check(cudaMemcpy(d_cs.p, bytes, n_bytes, cudaMemcpyHostToDevice), "cs");
    upload_ht_tables(false, d_t);
    std::vector<DecBlock> db(n);
    size_t scratch = 0;
    uint32_t nfast = 0;
    for (uint32_t i = 0; i < n; ++i) {
      DecBlock& d = db[i]; memset(&d, 0, sizeof(d));
      d.data_off = desc[i].byte_off; d.dst_off = desc[i].sample_off; d.stride = desc[i].stride;
      d.w = (uint16_t)desc[i].w; d.h = (uint16_t)desc[i].h; d.len1 = desc[i].len1; d.len2 = desc[i].len2;
      d.missing_msbs = (uint8_t)desc[i].missing_msbs; d.num_passes = (uint8_t)desc[i].num_passes;
      d.K_max = (uint8_t)(desc[i].missing_msbs + 1); d.flags = desc[i].causal ? 1 : 0;
      uint32_t nq = (d.w + 1u) / 2, qs = (nq + 1) & ~1u, nqr = (d.h + 1u) / 2;
      d.scratch_off = scratch; scratch += (size_t)qs * nqr;        // quad records (even: 8-byte aligned)
      if (!getenv("OJB_NO_FAST_BLOCKS") && dec_block_is_fast(d)) { d.flags |= DEC_FLAG_FAST; ++nfast; }
    }
    d_b.reserve(n * sizeof(DecBlock)); d_o.reserve((n_words + 64) * 4); d_sc.reserve((scratch + 64) * 4); d_st.reserve(n * 4 + 16);
    cuda_check(cudaMemcpy(d_b.p, db.data(), n * sizeof(DecBlock), cudaMemcpyHostToDevice), "blocks");
    cuda_check(cudaMemcpy(d_o.p, samples, n_words * 4, cudaMemcpyHostToDevice), "out init");
    uint32_t maxw = 4;
    for (uint32_t i = 0; i < n; ++i) maxw = std::max(maxw, desc[i].w);
    launch_ht_decode_serial(d_b.as<DecBlock>(), n, nfast, maxw, d_cs.as<uint8_t>(), d_o.as<uint32_t>(), d_sc.as<uint32_t>(),
                            d_t.as<uint16_t>(), DEC_OUT_SIGNMAG, false, d_st.as<uint32_t>(), 0);
    cuda_check(cudaDeviceSynchronize(), "ht_decode");
    cuda_check(cudaGetLastError(), "ht_decode");
    cuda_check(cudaMemcpy(samples, d_o.p, n_words * 4, cudaMemcpyDeviceToHost), "samples");
    std::vector<uint32_t> st(n);
    cuda_check(cudaMemcpy(st.data(), d_st.p, n * 4, cudaMemcpyDeviceToHost), "status");
    for (uint32_t i = 0; i < n; ++i) desc[i].status = st[i] & 1u;
  });
}

} // extern "C"
