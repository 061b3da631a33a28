// ojb_shard.cpp -- one image over the GPUs of a box: tiles are sharded over ranks (one process per GPU), the only
// data-path collective is the final gather of tile-part bytes (encode) / decoded tile samples (decode) to the
// writer rank.
//
// Tiles are independent through colour transform, DWT, quantisation, block coding and packet formation: the
// reference gives every tile its own component / resolution tree (src/core/codestream/ojph_codestream_local.cpp:
// 132-168) and concatenates the tile-parts in tile-index order at flush (:1148-1164, tile::flush
// src/core/codestream/ojph_tile.cpp:584-772).  Every rank therefore keeps ONE encoder / decoder with the geometry
// of the whole image and a tile mask (CodecBase::tile_mask): rank r works on the tiles t with t % world == r, so
// Isot, canvas coordinates and packet contents are what a single encoder produces, and the bytes on the writer are
// byte-identical to the one-GPU codestream.
//
// Encode, per frame:  H2D of the rank's tile rectangles -> DWT + block coding + packet headers of its tiles ->
//   tile-parts in device memory -> allgather of the per-tile sizes (a few hundred bytes) -> ncclSend / ncclRecv of
//   each tile's bytes straight from the producer's device buffer to its final offset in the writer's device buffer
//   (one group) -> main header (+TLM) and EOC added on the writer -> one D2H.
// Decode mirrors it: the codestream is broadcast in device memory (NVLink), every rank reads the headers from
// there (Decoder::read_headers_device: only header pages travel to the host), decodes its tiles, and the tile
// samples are sent to the writer, which delivers them with one strided D2H per tile rectangle.
//
// Transport: NCCL (libnccl.so.2, loaded at run time so that single-GPU users do not need it), communicator built
// from a unique id the caller distributes; or caller-supplied callbacks (the CPU test tier runs this file under
// the SIMT emulator with torch.distributed/gloo behind the callbacks).
#include "../../include/ojph_b200.h"
#include "ojb_codec.h"
#include <cstring>
#include <memory>
#include <algorithm>
#ifndef OJB_EMU_BUILD
#include <dlfcn.h>
#endif

using namespace ojb;

namespace {

struct Xfer { uint32_t peer; void* dev; size_t bytes; };

struct Comm {
  uint32_t rank = 0, world = 1;
  virtual ~Comm() {}
  virtual void allgather(const void* send_host, void* recv_host, size_t bytes_per_rank) = 0;
  virtual void bcast(void* dev, size_t bytes, uint32_t root, cudaStream_t st) = 0;
  // all sends and receives of one exchange step; returns when the data has arrived
  virtual void exchange(const std::vector<Xfer>& sends, const std::vector<Xfer>& recvs, cudaStream_t st) = 0;
};

struct CallbackComm : Comm {
  ojb_comm_callbacks cb;
  explicit CallbackComm(const ojb_comm_callbacks& c, uint32_t r, uint32_t w) : cb(c) { rank = r; world = w; }
  static void ck(int rc, const char* what) { if (rc != 0) fail(0x000B0040, "transport callback %s failed (%d)", what, rc); }
  void allgather(const void* s, void* r, size_t n) override { ck(cb.allgather(cb.ctx, s, r, n), "allgather"); }
  void bcast(void* dev, size_t bytes, uint32_t root, cudaStream_t st) override {
    cuda_check(cudaStreamSynchronize(st), "bcast");
    ck(cb.bcast(cb.ctx, dev, bytes, root), "bcast");
  }
  void exchange(const std::vector<Xfer>& sends, const std::vector<Xfer>& recvs, cudaStream_t st) override {
    cuda_check(cudaStreamSynchronize(st), "exchange");
    for (const Xfer& x : sends) ck(cb.send(cb.ctx, x.dev, x.bytes, x.peer), "send");
    for (const Xfer& x : recvs) ck(cb.recv(cb.ctx, x.dev, x.bytes, x.peer), "recv");
  }
};

#ifndef OJB_EMU_BUILD
// the few NCCL entry points used, resolved from libnccl.so.2 at run time (the process usually has torch's copy
// loaded already; the SONAME is the same)
struct NcclApi {
  typedef struct { char internal[128]; } UniqueId;
  void* h = nullptr;
  int (*GetUniqueId)(UniqueId*) = nullptr;
  int (*CommInitRank)(void**, int, UniqueId, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  static NcclApi& get() {
    static NcclApi a = [] {
      NcclApi x;
      x.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
      if (!x.h) x.h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
      if (!x.h) return x;
      auto sym = [&](const char* n) { return dlsym(x.h, n); };
      x.GetUniqueId = (decltype(x.GetUniqueId))sym("ncclGetUniqueId");
      x.CommInitRank = (decltype(x.CommInitRank))sym("ncclCommInitRank");
      x.CommDestroy = (decltype(x.CommDestroy))sym("ncclCommDestroy");
      x.AllGather = (decltype(x.AllGather))sym("ncclAllGather");
      x.Broadcast = (decltype(x.Broadcast))sym("ncclBroadcast");
      x.Send = (decltype(x.Send))sym("ncclSend");
      x.Recv = (decltype(x.Recv))sym("ncclRecv");
      x.GroupStart = (decltype(x.GroupStart))sym("ncclGroupStart");
      x.GroupEnd = (decltype(x.GroupEnd))sym("ncclGroupEnd");
      x.GetErrorString = (decltype(x.GetErrorString))sym("ncclGetErrorString");
      return x;
    }();
    if (!a.h || !a.CommInitRank || !a.Send || !a.Recv || !a.AllGather || !a.Broadcast || !a.GroupStart || !a.GroupEnd)
      fail(0x000B0041, "libnccl.so.2 could not be loaded: the multi-GPU path needs NCCL");
    return a;
  }
};
enum { NCCL_UINT8 = 1 };      // ncclUint8 (ncclChar 0 / ncclInt8 0, ncclUint8 1)

struct NcclComm : Comm {
  void* comm = nullptr;
  DeviceBuf d_small;
  PinnedBuf h_small;
  static void ck(int rc, const char* what) {
    if (rc != 0) { NcclApi& a = NcclApi::get(); fail(0x000B0042, "NCCL failure in %s: %s", what, a.GetErrorString ? a.GetErrorString(rc) : "?"); }
  }
  NcclComm(uint32_t r, uint32_t w, const uint8_t id[128]) {
    rank = r; world = w;
    NcclApi& a = NcclApi::get();
    NcclApi::UniqueId uid; memcpy(uid.internal, id, 128);
    ck(a.CommInitRank(&comm, (int)w, uid, (int)r), "ncclCommInitRank");
  }
  ~NcclComm() override { if (comm) NcclApi::get().CommDestroy(comm); }
  void allgather(const void* s, void* r, size_t n) override {
    // a few hundred bytes: staged through device memory on the default stream of the calling thread
    NcclApi& a = NcclApi::get();
    d_small.reserve(n * (world + 1)); h_small.reserve(n * (world + 1));
    uint8_t* ds = d_small.as<uint8_t>();
    memcpy(h_small.p, s, n);
    cuda_check(cudaMemcpyAsync(ds, h_small.p, n, cudaMemcpyHostToDevice, 0), "allgather stage");
    ck(a.AllGather(ds, ds + n, n, NCCL_UINT8, comm, 0), "ncclAllGather");
    cuda_check(cudaMemcpyAsync(h_small.as<uint8_t>() + n, ds + n, n * world, cudaMemcpyDeviceToHost, 0), "allgather stage");
    cuda_check(cudaStreamSynchronize(0), "allgather");
    memcpy(r, h_small.as<uint8_t>() + n, n * world);
  }
  void bcast(void* dev, size_t bytes, uint32_t root, cudaStream_t st) override {
    ck(NcclApi::get().Broadcast(dev, dev, bytes, NCCL_UINT8, (int)root, comm, st), "ncclBroadcast");
  }
  void exchange(const std::vector<Xfer>& sends, const std::vector<Xfer>& recvs, cudaStream_t st) override {
    NcclApi& a = NcclApi::get();
    ck(a.GroupStart(), "ncclGroupStart");
    for (const Xfer& x : sends) ck(a.Send(x.dev, x.bytes, NCCL_UINT8, (int)x.peer, comm, st), "ncclSend");
    for (const Xfer& x : recvs) ck(a.Recv(x.dev, x.bytes, NCCL_UINT8, (int)x.peer, comm, st), "ncclRecv");
    ck(a.GroupEnd(), "ncclGroupEnd");
    cuda_check(cudaStreamSynchronize(st), "exchange");
  }
};
#endif

} // namespace

extern "C" void ojb_params_to_internal(const ojb_params* s, ojb::Params& P);     // ojb_capi.cpp (not part of the public header)

struct ojb_shard {
  int device = 0;
  std::unique_ptr<Comm> comm;
  uint32_t writer = 0, sample_type = ST_I32;
  Encoder enc; bool enc_ready = false;
  Decoder dec;
  Params full;                              // finalised parameters of the whole image (writer's main header)
  std::vector<Comment> comments;
  DeviceBuf d_parts, d_final, d_stage, d_cs;
  PinnedBuf h_hdr;
  float ms_encode = 0, ms_gather = 0;       // last call: this rank's codec time, exchange + assembly + D2H
  size_t final_len = 0;                     // writer: length of the codestream in d_final
  // partition: 0 = tiles (t % world), 1 = row regions of every tile-component (CodecBase::region, ojb_codec.h)
  uint32_t partition = 0;
  DeviceBuf d_pack, d_off, d_owner;         // regions: [lengths | packed block bytes] of this rank, block offsets, block owners
  PinnedBuf h_tot;
};

static thread_local char g_serr[1024] = "";
const char* ojb_shard_last_error(void) { return g_serr; }
template <typename F> static int sguarded(ojb_shard* s, F&& f) {
  try { if (s) cuda_check(cudaSetDevice(s->device), "cudaSetDevice"); f(); return 0; }
  catch (const Error& e) { snprintf(g_serr, sizeof(g_serr), "%s", e.what()); return -(int)((e.code >> 16) ? (e.code >> 16) : 1); }
  catch (const std::exception& e) { snprintf(g_serr, sizeof(g_serr), "%s", e.what()); return -1001; }
  catch (...) { snprintf(g_serr, sizeof(g_serr), "ojph error: unknown exception"); return -1002; }
}

extern "C" {

int ojb_shard_unique_id(uint8_t out[128]) {
#ifdef OJB_EMU_BUILD
  memset(out, 0, 128); return 0;
#else
  return sguarded(nullptr, [&] {
    NcclApi::UniqueId id;
    NcclComm::ck(NcclApi::get().GetUniqueId(&id), "ncclGetUniqueId");
    memcpy(out, id.internal, 128);
  });
#endif
}

ojb_shard* ojb_shard_create_nccl(uint32_t rank, uint32_t world, const uint8_t unique_id[128]) {
#ifdef OJB_EMU_BUILD
  (void)rank; (void)world; (void)unique_id;
  snprintf(g_serr, sizeof(g_serr), "no NCCL in the emulator build");
  return nullptr;
#else
  ojb_shard* s = nullptr;
  int rc = sguarded(nullptr, [&] {
    std::unique_ptr<ojb_shard> t(new ojb_shard());
    cuda_check(cudaGetDevice(&t->device), "cudaGetDevice");
    t->comm.reset(new NcclComm(rank, world, unique_id));
    s = t.release();
  });
  return rc == 0 ? s : nullptr;
#endif
}

ojb_shard* ojb_shard_create(uint32_t rank, uint32_t world, const ojb_comm_callbacks* cb) {
  ojb_shard* s = nullptr;
  int rc = sguarded(nullptr, [&] {
    if (!cb || !cb->allgather || !cb->bcast || !cb->send || !cb->recv) fail(0x000B0043, "incomplete transport callbacks");
    std::unique_ptr<ojb_shard> t(new ojb_shard());
    cuda_check(cudaGetDevice(&t->device), "cudaGetDevice");
    t->comm.reset(new CallbackComm(*cb, rank, world));
    s = t.release();
  });
  return rc == 0 ? s : nullptr;
}

void ojb_shard_destroy(ojb_shard* s) { if (s) { cudaSetDevice(s->device); delete s; } }

int ojb_shard_enc_configure(ojb_shard* s, const ojb_params* p, uint32_t sample_type, uint32_t writer_rank) {
  return sguarded(s, [&] {
    if (sample_type > 2) fail(0x000B0012, "unknown sample container");
    if (writer_rank >= s->comm->world) fail(0x000B0044, "writer rank %u of %u", writer_rank, s->comm->world);
    Params P; ojb_params_to_internal(p, P);
    s->enc_ready = false;
    s->writer = writer_rank; s->sample_type = sample_type;
    s->full = P; s->full.finalize_for_encode();
    Layout L; L.build(s->full);
    const uint32_t ntiles = (uint32_t)L.tiles.size();
    s->enc.tile_mask.clear(); s->enc.region = CodecBase::RegionSpec();
    if (s->partition == 1 && s->comm->world > 1) {
      if (s->comm->world > 255) fail(0x000B0044, "row regions: at most 255 ranks");
      s->enc.region.rank = s->comm->rank; s->enc.region.world = s->comm->world;
    } else {
      s->enc.tile_mask.assign(ntiles, 0);
      for (uint32_t t = 0; t < ntiles; ++t) s->enc.tile_mask[t] = (t % s->comm->world == s->comm->rank) ? 1 : 0;
    }
    s->enc.configure(P, sample_type);
    if (s->enc.region.on()) {
      s->d_owner.reserve(std::max<size_t>(1, s->enc.region_owner.size()));
      if (!s->enc.region_owner.empty())
        cuda_check(cudaMemcpy(s->d_owner.p, s->enc.region_owner.data(), s->enc.region_owner.size(), cudaMemcpyHostToDevice), "block owners");
    }
    s->enc_ready = true;
  });
}

// ---- row regions --------------------------------------------------------------------------------------------------
// Encode: every rank uploads the image rows its slab's coefficients depend on (slab + halo), runs its window of every
// DWT level and codes its own code-blocks (Encoder::encode_front).  Then the one exchange of the path: each rank packs
// its blocks' bytes back to back behind the per-block lengths and sends them to the writer (sizes by one 8-byte
// allgather), the writer drops them into its slot arena as if it had coded them (scatter_blocks_kernel) and finishes
// as a single encoder does: packet headers, markers and layout on the device (Encoder::encode_back).  Byte-identical
// to the one-GPU / reference codestream -- also for a single-tile image, which tile sharding cannot split.
static void region_upload(ojb_shard* s, const void* const* planes, const uint32_t* strides) {
  Encoder& E = s->enc; const Params& P = E.params;
  const uint32_t nc = P.num_comps(), es = esize_of(s->sample_type);
  for (const TileGeom& t : E.layout.tiles)
    for (uint32_t c = 0; c < nc; ++c) {
      const Rect& r = t.comps[c].rect;
      const CodecBase::RowSpan rows = E.region_rows[t.idx][c];
      if (r.w == 0 || rows.hi <= rows.lo) continue;
      const uint32_t cx0 = div_ceil(P.XOsiz, P.comps[c].dx), cy0 = div_ceil(P.YOsiz, P.comps[c].dy);
      const uint32_t st = strides ? strides[c] : E.img_w[c];
      const size_t so = ((size_t)(rows.lo - cy0) * st + (r.x0 - cx0)) * es, dof = ((size_t)(rows.lo - cy0) * E.img_w[c] + (r.x0 - cx0)) * es;
      cuda_check(cudaMemcpy2DAsync(E.d_image.as<uint8_t>() + E.img_off[c] + dof, (size_t)E.img_w[c] * es,
                                   (const uint8_t*)planes[c] + so, (size_t)st * es, (size_t)r.w * es, rows.hi - rows.lo,
                                   cudaMemcpyHostToDevice, E.stream), "region upload");
    }
}

static void region_encode(ojb_shard* s, const void* const* planes, const uint32_t* strides,
                          uint8_t* out, uint64_t out_cap, uint64_t* out_len, bool encode_only_upload) {
  Encoder& E = s->enc; Comm& C = *s->comm;
  const uint32_t nb = (uint32_t)E.h_blocks.size();
  cudaEvent_t e0 = E.ev[CodecBase::EV_MAX - 3], e1 = E.ev[CodecBase::EV_MAX - 2], e2 = E.ev[CodecBase::EV_MAX - 1];
  cudaEventRecord(e0, E.stream);
  if (planes) region_upload(s, planes, strides);
  if (encode_only_upload) { cuda_check(cudaStreamSynchronize(E.stream), "region upload"); return; }
  // 1. this rank's share of the transform and of the block coding
  E.encode_front();
  cudaEventRecord(e1, E.stream);
  // 2. how many bytes that made; every rank learns every total
  s->d_off.reserve(((size_t)nb + 4) * 8);
  s->h_tot.reserve(64);
  uint64_t* d_total = s->d_off.as<uint64_t>() + (((size_t)nb + 1) & ~(size_t)1);      // 16-byte aligned (ctrl copy)
  launch_block_offsets(E.d_results.as<EncResult>(), nb, s->d_off.as<uint64_t>(), d_total, E.stream);
  launch_ctrl_copy(s->h_tot.p, d_total, 16, E.stream);
  cuda_check(cudaStreamSynchronize(E.stream), "block totals");
  std::vector<uint64_t> mine(1, s->h_tot.as<uint64_t>()[0]), tot(C.world, 0);
  C.allgather(mine.data(), tot.data(), 8);
  const size_t meta = (size_t)nb * sizeof(EncResult);
  std::vector<Xfer> sends, recvs;
  std::vector<size_t> roff(C.world + 1, 0);
  if (C.rank != s->writer) {
    // 3. [lengths of all blocks | this rank's bytes, packed] -> writer
    s->d_pack.reserve(meta + (size_t)mine[0] + 64);
    if (nb) cuda_check(cudaMemcpyAsync(s->d_pack.p, E.d_results.p, meta, cudaMemcpyDeviceToDevice, E.stream), "lengths");
    launch_gather_blocks(E.d_blocks.as<EncBlock>(), E.d_results.as<EncResult>(), s->d_off.as<uint64_t>(), nb, E.d_slots.as<uint8_t>(),
                         s->d_pack.as<uint8_t>() + meta, E.stream);
    sends.push_back(Xfer{ s->writer, s->d_pack.p, meta + (size_t)mine[0] });
  } else {
    for (uint32_t r = 0; r < C.world; ++r) roff[r + 1] = roff[r] + (r == C.rank ? 0 : ((meta + (size_t)tot[r] + 64 + 255) & ~(size_t)255));
    s->d_stage.reserve(roff[C.world] + 64);
    for (uint32_t r = 0; r < C.world; ++r)
      if (r != C.rank) recvs.push_back(Xfer{ r, s->d_stage.as<uint8_t>() + roff[r], meta + (size_t)tot[r] });
  }
  C.exchange(sends, recvs, E.stream);
  size_t total = 0;
  if (C.rank == s->writer) {
    // 4. the other ranks' blocks into the slot arena, then the back half of a single encoder's frame call
    for (uint32_t r = 0; r < C.world; ++r) {
      if (r == C.rank) continue;
      const uint8_t* base = s->d_stage.as<uint8_t>() + roff[r];
      launch_block_offsets(reinterpret_cast<const EncResult*>(base), nb, s->d_off.as<uint64_t>(), d_total, E.stream);
      launch_scatter_blocks(E.d_blocks.as<EncBlock>(), s->d_owner.as<uint8_t>(), r, reinterpret_cast<const EncResult*>(base),
                            s->d_off.as<uint64_t>(), nb, base + meta, E.d_slots.as<uint8_t>(), E.d_results.as<EncResult>(), E.stream);
    }
    uint64_t sum = 0; for (uint32_t r = 0; r < C.world; ++r) sum += tot[r];
    const size_t cap = (size_t)sum + (size_t)nb * 24 + E.fixed_blob.size() + E.main_header.size() + (1u << 16);
    s->d_final.reserve(cap + 64);
    total = E.encode_back(s->d_final.as<uint8_t>(), cap);
    if (out) {
      if (total > out_cap) fail(0x000B0030, "output buffer too small: need %zu bytes, have %zu", total, (size_t)out_cap);
      cuda_check(cudaMemcpyAsync(out, s->d_final.p, total, cudaMemcpyDeviceToHost, E.stream), "codestream D2H");
    }
    s->final_len = total;
  }
  if (out_len) *out_len = total;
  cudaEventRecord(e2, E.stream);
  cuda_check(cudaStreamSynchronize(E.stream), "region encode");
  cudaEventElapsedTime(&s->ms_encode, e0, e1); cudaEventElapsedTime(&s->ms_gather, e1, e2);
}

// Decode: the codestream is broadcast, every rank parses the headers, decodes the blocks its slab's rows depend on,
// runs its window of every synthesis level and sends the rows of its slab to the writer.
static void region_decode(ojb_shard* s, uint32_t sample_type, uint32_t writer_rank, void* const* planes, const uint32_t* strides,
                          bool keep_on_device, cudaEvent_t e1) {
  Decoder& D = s->dec; Comm& C = *s->comm;
  D.decode(nullptr, nullptr, false);
  cudaEventRecord(e1, D.stream);
  const Params& P = D.params;
  const uint32_t nc = P.num_comps(), es = esize_of(sample_type);
  // every rank's slab of every tile-component, packed tile after tile, component after component
  std::vector<size_t> roff(C.world + 1, 0);
  for (uint32_t r = 0; r < C.world; ++r) {
    size_t b = 0;
    for (const TileGeom& t : D.layout.tiles)
      for (uint32_t c = 0; c < nc; ++c) {
        const CodecBase::RowSpan sp = CodecBase::region_slab(t.comps[c].rect, r, C.world);
        b += (size_t)t.comps[c].rect.w * (sp.hi - sp.lo) * es;
      }
    roff[r + 1] = roff[r] + ((b + 255) & ~(size_t)255);
  }
  auto plane_pos = [&](uint32_t x0, uint32_t y0, uint32_t c, uint32_t pitch) {
    const uint32_t cx0 = div_ceil(P.XOsiz, P.comps[c].dx), cy0 = div_ceil(P.YOsiz, P.comps[c].dy);
    return ((size_t)(y0 - cy0) * pitch + (x0 - cx0)) * es;
  };
  // walk the slab rectangles of rank r: f(tile-component rectangle, rows, offset in the rank's packed piece)
  auto for_slabs = [&](uint32_t r, auto&& f) {
    size_t o = 0;
    for (const TileGeom& t : D.layout.tiles)
      for (uint32_t c = 0; c < nc; ++c) {
        const Rect& rc = t.comps[c].rect;
        const CodecBase::RowSpan sp = CodecBase::region_slab(rc, r, C.world);
        if (rc.w == 0 || sp.hi <= sp.lo) continue;
        f(c, rc, sp, o);
        o += (size_t)rc.w * (sp.hi - sp.lo) * es;
      }
  };
  std::vector<Xfer> sends, recvs;
  s->d_stage.reserve(roff[C.world] + 64);
  if (C.rank != writer_rank) {
    for_slabs(C.rank, [&](uint32_t c, const Rect& rc, const CodecBase::RowSpan& sp, size_t o) {
      cuda_check(cudaMemcpy2DAsync(s->d_stage.as<uint8_t>() + roff[C.rank] + o, (size_t)rc.w * es,
                                   D.d_image.as<uint8_t>() + D.img_off[c] + plane_pos(rc.x0, sp.lo, c, D.img_w[c]), (size_t)D.img_w[c] * es,
                                   (size_t)rc.w * es, sp.hi - sp.lo, cudaMemcpyDeviceToDevice, D.stream), "slab pack");
    });
    if (roff[C.rank + 1] > roff[C.rank]) sends.push_back(Xfer{ writer_rank, s->d_stage.as<uint8_t>() + roff[C.rank], roff[C.rank + 1] - roff[C.rank] });
  } else {
    for (uint32_t r = 0; r < C.world; ++r)
      if (r != C.rank && roff[r + 1] > roff[r]) recvs.push_back(Xfer{ r, s->d_stage.as<uint8_t>() + roff[r], roff[r + 1] - roff[r] });
  }
  C.exchange(sends, recvs, D.stream);
  if (C.rank != writer_rank) return;
  for (uint32_t r = 0; r < C.world; ++r)
    for_slabs(r, [&](uint32_t c, const Rect& rc, const CodecBase::RowSpan& sp, size_t o) {
      const uint8_t* src = (r == C.rank) ? D.d_image.as<uint8_t>() + D.img_off[c] + plane_pos(rc.x0, sp.lo, c, D.img_w[c])
                                         : s->d_stage.as<uint8_t>() + roff[r] + o;
      const size_t spitch = (r == C.rank) ? (size_t)D.img_w[c] * es : (size_t)rc.w * es;
      if (keep_on_device && r != C.rank)
        cuda_check(cudaMemcpy2DAsync(D.d_image.as<uint8_t>() + D.img_off[c] + plane_pos(rc.x0, sp.lo, c, D.img_w[c]), (size_t)D.img_w[c] * es,
                                     src, spitch, (size_t)rc.w * es, sp.hi - sp.lo, cudaMemcpyDeviceToDevice, D.stream), "slab unpack");
      if (planes) {
        const uint32_t st = strides ? strides[c] : D.img_w[c];
        cuda_check(cudaMemcpy2DAsync((uint8_t*)planes[c] + plane_pos(rc.x0, sp.lo, c, st), (size_t)st * es, src, spitch,
                                     (size_t)rc.w * es, sp.hi - sp.lo, cudaMemcpyDeviceToHost, D.stream), "slab D2H");
      }
    });
}

// planes: the WHOLE image on the host (every rank passes the same pointers or at least valid memory for its own
// tiles); out / out_cap / out_len matter on the writer only.
static int shard_encode(ojb_shard* s, const void* const* planes, const uint32_t* strides,
                        uint8_t* out, uint64_t out_cap, uint64_t* out_len, bool encode_only_upload) {
  return sguarded(s, [&] {
    if (!s->enc_ready) fail(0x000B0013, "encoder is not configured");
    if (s->enc.region.on()) { region_encode(s, planes, strides, out, out_cap, out_len, encode_only_upload); return; }
    Encoder& E = s->enc; Comm& C = *s->comm;
    const Params& P = E.params;
    const uint32_t nc = P.num_comps(), es = esize_of(s->sample_type);
    const uint32_t ntiles = (uint32_t)E.layout.tiles.size();
    cudaEvent_t e0 = E.ev[CodecBase::EV_MAX - 3], e1 = E.ev[CodecBase::EV_MAX - 2], e2 = E.ev[CodecBase::EV_MAX - 1];
    cudaEventRecord(e0, E.stream);
    // 1. this rank's tile rectangles -> device image buffer (planes == NULL: they are there already)
    size_t my_in = 0;
    for (const TileGeom& t : E.layout.tiles) {
      if (!E.tile_wanted(t.idx)) continue;
      for (uint32_t c = 0; c < nc; ++c) {
        const Rect& r = t.comps[c].rect;
        if (r.w == 0 || r.h == 0) continue;
        my_in += (size_t)r.w * r.h * es;
        if (!planes) continue;
        const uint32_t cx0 = div_ceil(P.XOsiz, P.comps[c].dx), cy0 = div_ceil(P.YOsiz, P.comps[c].dy);
        const uint32_t st = strides ? strides[c] : E.img_w[c];
        const size_t so = ((size_t)(r.y0 - cy0) * st + (r.x0 - cx0)) * es, dof = ((size_t)(r.y0 - cy0) * E.img_w[c] + (r.x0 - cx0)) * es;
        cuda_check(cudaMemcpy2DAsync(E.d_image.as<uint8_t>() + E.img_off[c] + dof, (size_t)E.img_w[c] * es,
                                     (const uint8_t*)planes[c] + so, (size_t)st * es, (size_t)r.w * es, r.h,
                                     cudaMemcpyHostToDevice, E.stream), "tile upload");
      }
    }
    if (encode_only_upload) { cuda_check(cudaStreamSynchronize(E.stream), "tile upload"); return; }
    // 2. code this rank's tiles: tile-parts, back to back, in device memory
    s->d_parts.reserve(my_in * 2 + (1u << 20));
    const size_t my_bytes = E.encode(nullptr, nullptr, false, s->d_parts.as<uint8_t>(), s->d_parts.cap, true);
    cudaEventRecord(e1, E.stream);
    // 3. sizes: per tile (number of tile-parts, bytes), then the tile-part lengths when a TLM is wanted
    std::vector<uint32_t> mine(2 * ntiles, 0), all((size_t)2 * ntiles * C.world, 0);
    std::vector<uint64_t> my_off(ntiles, 0);
    for (const Encoder::TilePartOut& tp : E.last_tileparts) {
      if (mine[2 * tp.tile] == 0) my_off[tp.tile] = tp.offset;
      mine[2 * tp.tile] += 1; mine[2 * tp.tile + 1] += tp.bytes;
    }
    C.allgather(mine.data(), all.data(), mine.size() * 4);
    std::vector<uint32_t> nparts(ntiles, 0), tbytes(ntiles, 0);
    for (uint32_t t = 0; t < ntiles; ++t) {
      const uint32_t owner = t % C.world;
      nparts[t] = all[(size_t)owner * 2 * ntiles + 2 * t]; tbytes[t] = all[(size_t)owner * 2 * ntiles + 2 * t + 1];
    }
    std::vector<std::vector<uint32_t>> psot(ntiles);
    if (s->full.need_tlm) {
      uint32_t maxp = 0;
      for (uint32_t r = 0; r < C.world; ++r) { uint32_t n = 0; for (uint32_t t = r; t < ntiles; t += C.world) n += nparts[t]; maxp = std::max(maxp, n); }
      std::vector<uint32_t> ml(std::max(1u, maxp), 0), al((size_t)std::max(1u, maxp) * C.world, 0);
      for (size_t i = 0; i < E.last_tileparts.size(); ++i) ml[i] = E.last_tileparts[i].bytes;
      C.allgather(ml.data(), al.data(), ml.size() * 4);
      for (uint32_t r = 0; r < C.world; ++r) {
        size_t k = 0;
        for (uint32_t t = r; t < ntiles; t += C.world)
          for (uint32_t i = 0; i < nparts[t]; ++i) psot[t].push_back(al[(size_t)r * ml.size() + k++]);
      }
    }
    // 4. placement on the writer; 5. the exchange
    std::vector<Xfer> sends, recvs;
    size_t total = 0, hdr_len = 0;
    std::vector<uint8_t> hdr;
    if (C.rank == s->writer) {
      s->full.comments = s->comments;
      s->full.write_main_header(hdr, nullptr, nullptr, 0);
      if (s->full.need_tlm) {
        size_t n_tp = 0; for (uint32_t t = 0; t < ntiles; ++t) n_tp += psot[t].size();
        if (4 + 6 * n_tp > 65535) fail(0x000500B1, "too many tile-parts for one TLM marker segment");
        put_u16(hdr, M_TLM); put_u16(hdr, (uint32_t)(4 + 6 * n_tp)); put_u8(hdr, 0); put_u8(hdr, 0x60);
        for (uint32_t t = 0; t < ntiles; ++t) for (uint32_t l : psot[t]) { put_u16(hdr, t); put_u32(hdr, l); }
      }
      hdr_len = hdr.size();
      total = hdr_len; for (uint32_t t = 0; t < ntiles; ++t) total += tbytes[t];
      total += 2;
      if (out && total > out_cap) fail(0x000B0030, "output buffer too small: need %zu bytes, have %zu", total, (size_t)out_cap);
      s->d_final.reserve(total + 64);
      size_t pos = hdr_len;
      for (uint32_t t = 0; t < ntiles; ++t) {
        const uint32_t owner = t % C.world;
        if (tbytes[t]) {
          if (owner == C.rank)
            cuda_check(cudaMemcpyAsync(s->d_final.as<uint8_t>() + pos, s->d_parts.as<uint8_t>() + my_off[t], tbytes[t],
                                       cudaMemcpyDeviceToDevice, E.stream), "own tile");
          else recvs.push_back(Xfer{ owner, s->d_final.as<uint8_t>() + pos, tbytes[t] });
        }
        pos += tbytes[t];
      }
      hdr.push_back(0xFF); hdr.push_back(0xD9);              // EOC rides behind the header bytes in the staging buffer
      s->h_hdr.reserve(hdr.size()); memcpy(s->h_hdr.p, hdr.data(), hdr.size());
      cuda_check(cudaMemcpyAsync(s->d_final.p, s->h_hdr.p, hdr_len, cudaMemcpyHostToDevice, E.stream), "header");
      cuda_check(cudaMemcpyAsync(s->d_final.as<uint8_t>() + total - 2, s->h_hdr.as<uint8_t>() + hdr_len, 2, cudaMemcpyHostToDevice, E.stream), "EOC");
    } else {
      for (uint32_t t = C.rank; t < ntiles; t += C.world)
        if (tbytes[t]) sends.push_back(Xfer{ s->writer, s->d_parts.as<uint8_t>() + my_off[t], tbytes[t] });
    }
    (void)my_bytes;
    C.exchange(sends, recvs, E.stream);
    if (C.rank == s->writer) {
      if (out) cuda_check(cudaMemcpyAsync(out, s->d_final.p, total, cudaMemcpyDeviceToHost, E.stream), "codestream D2H");
      if (out_len) *out_len = total;
      s->final_len = total;
    } else if (out_len) *out_len = 0;
    cudaEventRecord(e2, E.stream);
    cuda_check(cudaStreamSynchronize(E.stream), "shard encode");
    cudaEventElapsedTime(&s->ms_encode, e0, e1); cudaEventElapsedTime(&s->ms_gather, e1, e2);
  });
}

int ojb_shard_enc_encode(ojb_shard* s, const void* const* planes, const uint32_t* strides,
                         uint8_t* out, uint64_t out_cap, uint64_t* out_len) {
  return shard_encode(s, planes, strides, out, out_cap, out_len, false);
}
// device-resident form: every rank uploads its tiles once (ojb_shard_enc_upload), ojb_shard_enc_encode_resident leaves the
// codestream in the writer's device memory (ojb_shard_device_codestream)
int ojb_shard_enc_upload(ojb_shard* s, const void* const* planes, const uint32_t* strides) {
  return shard_encode(s, planes, strides, nullptr, 0, nullptr, true);
}
int ojb_shard_enc_encode_resident(ojb_shard* s, uint64_t* out_len) {
  return shard_encode(s, nullptr, nullptr, nullptr, 0, out_len, false);
}
const void* ojb_shard_device_codestream(ojb_shard* s) { return s->d_final.p; }

// cs / len: the codestream on the writer's host (ignored elsewhere).  planes: where the writer wants the decoded
// components (whole image, host); ignored on the other ranks.  info (may be NULL) is filled on every rank.
static int shard_decode(ojb_shard* s, const uint8_t* cs, bool cs_on_device, uint64_t len, uint32_t sample_type, uint32_t writer_rank,
                        void* const* planes, const uint32_t* strides, bool keep_on_device, ojb_frame_info* info) {
  return sguarded(s, [&] {
    Decoder& D = s->dec; Comm& C = *s->comm;
    if (sample_type > 2) fail(0x000B0012, "unknown sample container");
    if (writer_rank >= C.world) fail(0x000B0044, "writer rank %u of %u", writer_rank, C.world);
    cudaEvent_t e0 = D.ev[CodecBase::EV_MAX - 3], e1 = D.ev[CodecBase::EV_MAX - 2], e2 = D.ev[CodecBase::EV_MAX - 1];
    // 1. the codestream to every rank's device memory
    std::vector<uint64_t> ln(1, C.rank == writer_rank ? len : 0), lens(C.world, 0);
    C.allgather(ln.data(), lens.data(), 8);
    const size_t n = (size_t)lens[writer_rank];
    if (n < 4) fail(0x00050041, "error reading SIZ marker");
    s->d_cs.reserve(n + 64);
    cudaEventRecord(e0, D.stream);
    if (C.rank == writer_rank)
      cuda_check(cudaMemcpyAsync(s->d_cs.p, cs, n, cs_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, D.stream), "codestream to the broadcast buffer");
    cuda_check(cudaMemsetAsync(s->d_cs.as<uint8_t>() + n, 0, 32, D.stream), "codestream slack");
    C.bcast(s->d_cs.p, n, writer_rank, D.stream);
    cuda_check(cudaStreamSynchronize(D.stream), "codestream broadcast");
    // 2. headers from device memory.  The tile mask follows from the tile count: a first frame (or a change of
    // geometry) is parsed once to learn it and then again with the mask; later frames hit the cached geometry.
    if (s->partition == 1 && C.world > 1) {
      if (C.world > 255) fail(0x000B0044, "row regions: at most 255 ranks");
      D.tile_mask.clear(); D.region.rank = C.rank; D.region.world = C.world;
      D.read_headers_device(s->d_cs.as<uint8_t>(), n, sample_type);
      if (info) { FrameInfo fi; D.info(fi); memcpy(info, &fi, sizeof(fi)); }
      region_decode(s, sample_type, writer_rank, planes, strides, keep_on_device, e1);
      cudaEventRecord(e2, D.stream);
      cuda_check(cudaStreamSynchronize(D.stream), "shard decode");
      cudaEventElapsedTime(&s->ms_encode, e0, e1); cudaEventElapsedTime(&s->ms_gather, e1, e2);
      return;
    }
    D.region = CodecBase::RegionSpec();
    D.read_headers_device(s->d_cs.as<uint8_t>(), n, sample_type);
    const uint32_t ntiles = (uint32_t)D.layout.tiles.size();
    if (D.tile_mask.size() != ntiles) {
      D.tile_mask.assign(ntiles, 0);
      for (uint32_t t = 0; t < ntiles; ++t) D.tile_mask[t] = (t % C.world == C.rank) ? 1 : 0;
      D.read_headers_device(s->d_cs.as<uint8_t>(), n, sample_type);
    }
    if (info) { FrameInfo fi; D.info(fi); memcpy(info, &fi, sizeof(fi)); }
    // 3. decode this rank's tiles (result in the device image buffer)
    D.decode(nullptr, nullptr, false);
    cudaEventRecord(e1, D.stream);
    // 4. tile samples to the writer: every tile packed (component after component, tight rows) in a staging buffer
    const Params& P = D.params;
    const uint32_t nc = P.num_comps(), es = esize_of(sample_type);
    std::vector<size_t> toff(ntiles + 1, 0);
    for (uint32_t t = 0; t < ntiles; ++t) {
      size_t b = 0;
      for (uint32_t c = 0; c < nc; ++c) b += (size_t)D.layout.tiles[t].comps[c].rect.w * D.layout.tiles[t].comps[c].rect.h * es;
      toff[t + 1] = toff[t] + ((b + 15) & ~(size_t)15);
    }
    std::vector<Xfer> sends, recvs;
    auto plane_pos = [&](const Rect& r, uint32_t c, uint32_t pitch) {
      const uint32_t cx0 = div_ceil(P.XOsiz, P.comps[c].dx), cy0 = div_ceil(P.YOsiz, P.comps[c].dy);
      return ((size_t)(r.y0 - cy0) * pitch + (r.x0 - cx0)) * es;
    };
    if (C.rank != writer_rank) {
      s->d_stage.reserve(toff[ntiles] + 64);
      for (uint32_t t = C.rank; t < ntiles; t += C.world) {
        size_t o = toff[t];
        for (uint32_t c = 0; c < nc; ++c) {
          const Rect& r = D.layout.tiles[t].comps[c].rect;
          if (r.w == 0 || r.h == 0) continue;
          cuda_check(cudaMemcpy2DAsync(s->d_stage.as<uint8_t>() + o, (size_t)r.w * es,
                                       D.d_image.as<uint8_t>() + D.img_off[c] + plane_pos(r, c, D.img_w[c]), (size_t)D.img_w[c] * es,
                                       (size_t)r.w * es, r.h, cudaMemcpyDeviceToDevice, D.stream), "tile pack");
          o += (size_t)r.w * r.h * es;
        }
        if (toff[t + 1] > toff[t]) sends.push_back(Xfer{ writer_rank, s->d_stage.as<uint8_t>() + toff[t], toff[t + 1] - toff[t] });
      }
    } else {
      s->d_stage.reserve(toff[ntiles] + 64);
      for (uint32_t t = 0; t < ntiles; ++t)
        if (t % C.world != C.rank && toff[t + 1] > toff[t])
          recvs.push_back(Xfer{ t % C.world, s->d_stage.as<uint8_t>() + toff[t], toff[t + 1] - toff[t] });
    }
    C.exchange(sends, recvs, D.stream);
    if (C.rank == writer_rank && keep_on_device) {        // the other ranks' tiles into the writer's device image buffer
      for (uint32_t t = 0; t < ntiles; ++t) {
        if (t % C.world == C.rank) continue;
        size_t o = toff[t];
        for (uint32_t c = 0; c < nc; ++c) {
          const Rect& r = D.layout.tiles[t].comps[c].rect;
          if (r.w == 0 || r.h == 0) continue;
          cuda_check(cudaMemcpy2DAsync(D.d_image.as<uint8_t>() + D.img_off[c] + plane_pos(r, c, D.img_w[c]), (size_t)D.img_w[c] * es,
                                       s->d_stage.as<uint8_t>() + o, (size_t)r.w * es, (size_t)r.w * es, r.h,
                                       cudaMemcpyDeviceToDevice, D.stream), "tile unpack");
          o += (size_t)r.w * r.h * es;
        }
      }
    }
    if (C.rank == writer_rank && planes) {
      for (uint32_t t = 0; t < ntiles; ++t) {
        size_t o = toff[t];
        for (uint32_t c = 0; c < nc; ++c) {
          const Rect& r = D.layout.tiles[t].comps[c].rect;
          if (r.w == 0 || r.h == 0) continue;
          const uint32_t st = strides ? strides[c] : D.img_w[c];
          uint8_t* dst = (uint8_t*)planes[c] + plane_pos(r, c, st);
          if (t % C.world == C.rank)
            cuda_check(cudaMemcpy2DAsync(dst, (size_t)st * es, D.d_image.as<uint8_t>() + D.img_off[c] + plane_pos(r, c, D.img_w[c]),
                                         (size_t)D.img_w[c] * es, (size_t)r.w * es, r.h, cudaMemcpyDeviceToHost, D.stream), "tile D2H");
          else
            cuda_check(cudaMemcpy2DAsync(dst, (size_t)st * es, s->d_stage.as<uint8_t>() + o, (size_t)r.w * es,
                                         (size_t)r.w * es, r.h, cudaMemcpyDeviceToHost, D.stream), "tile D2H");
          o += (size_t)r.w * r.h * es;
        }
      }
    }
    cudaEventRecord(e2, D.stream);
    cuda_check(cudaStreamSynchronize(D.stream), "shard decode");
    cudaEventElapsedTime(&s->ms_encode, e0, e1); cudaEventElapsedTime(&s->ms_gather, e1, e2);
  });
}

int ojb_shard_dec_decode(ojb_shard* s, const uint8_t* cs, uint64_t len, uint32_t sample_type, uint32_t writer_rank,
                         void* const* planes, const uint32_t* strides, ojb_frame_info* info) {
  return shard_decode(s, cs, false, len, sample_type, writer_rank, planes, strides, false, info);
}
// device-resident form: the codestream is in the writer's device memory, the decoded image stays in the writer's
// device image buffer (ojb_shard_device_plane)
int ojb_shard_dec_decode_resident(ojb_shard* s, const void* dev_cs, uint64_t len, uint32_t sample_type, uint32_t writer_rank,
                                  ojb_frame_info* info) {
  return shard_decode(s, static_cast<const uint8_t*>(dev_cs), true, len, sample_type, writer_rank, nullptr, nullptr, true, info);
}
void* ojb_shard_device_plane(ojb_shard* s, uint32_t comp) {
  if (comp >= s->dec.img_off.size()) return nullptr;
  return s->dec.d_image.as<uint8_t>() + s->dec.img_off[comp];
}

// variable-length gather of device buffers (whole codestreams of a frame-parallel batch, BASELINE configs[4]):
// every rank contributes `bytes` bytes at dev; on the writer they land back to back, in rank order, in out_dev
// (capacity out_cap) and offsets[world + 1] receives where each rank's piece starts.
int ojb_shard_gatherv(ojb_shard* s, const void* dev, uint64_t bytes, uint32_t writer_rank, void* out_dev, uint64_t out_cap,
                      uint64_t* offsets) {
  return sguarded(s, [&] {
    Comm& C = *s->comm;
    std::vector<uint64_t> mine(1, bytes), all(C.world, 0);
    C.allgather(mine.data(), all.data(), 8);
    std::vector<uint64_t> off(C.world + 1, 0);
    for (uint32_t r = 0; r < C.world; ++r) off[r + 1] = off[r] + all[r];
    if (offsets) memcpy(offsets, off.data(), off.size() * 8);
    std::vector<Xfer> sends, recvs;
    cudaStream_t st = s->enc.stream;
    if (C.rank == writer_rank) {
      if (off[C.world] > out_cap) fail(0x000B0030, "output buffer too small: need %zu bytes, have %zu", (size_t)off[C.world], (size_t)out_cap);
      for (uint32_t r = 0; r < C.world; ++r) {
        if (!all[r]) continue;
        if (r == C.rank) cuda_check(cudaMemcpyAsync((uint8_t*)out_dev + off[r], dev, all[r], cudaMemcpyDeviceToDevice, st), "own piece");
        else recvs.push_back(Xfer{ r, (uint8_t*)out_dev + off[r], (size_t)all[r] });
      }
    } else if (bytes) sends.push_back(Xfer{ writer_rank, const_cast<void*>(dev), (size_t)bytes });
    C.exchange(sends, recvs, st);
    cuda_check(cudaStreamSynchronize(st), "gatherv");
  });
}

int ojb_shard_set_partition(ojb_shard* s, uint32_t kind) {
  return sguarded(s, [&] {
    if (kind > 1) fail(0x000B0047, "unknown partition %u (0: tiles, 1: row regions)", kind);
    if (kind != s->partition) { s->partition = kind; s->enc_ready = false; }
  });
}
uint32_t ojb_shard_region_rows(ojb_shard* s, uint32_t comp, uint32_t* lo, uint32_t* hi) {
  // image rows of component `comp` (tile 0) this rank's encoder reads: its slab plus the halo
  if (!s->enc_ready || !s->enc.region.on() || s->enc.region_rows.empty() || comp >= s->enc.region_rows[0].size()) return 0;
  if (lo) *lo = s->enc.region_rows[0][comp].lo;
  if (hi) *hi = s->enc.region_rows[0][comp].hi;
  return 1;
}
void ojb_shard_timings(ojb_shard* s, float* ms2) { ms2[0] = s->ms_encode; ms2[1] = s->ms_gather; }
uint32_t ojb_shard_rank(ojb_shard* s) { return s->comm->rank; }
uint32_t ojb_shard_world(ojb_shard* s) { return s->comm->world; }

} // extern "C"
