// pkt_headers.cu -- packet headers, tile-part markers and the final byte layout of the codestream, on the device.
//
// What the reference does with one thread walking every code-block of every precinct (precinct::prepare_precinct,
// src/core/codestream/ojph_precinct.cpp:94-278: tag trees for inclusion and missing MSBs, pass count, Lblock,
// lengths, through a bit-stuffing writer, ojph_bitbuffer_write.h:85-143; tile::flush, ojph_tile.cpp:584-772: SOT /
// Psot, packet order) is split here into data-parallel steps so that an encode needs no host round trip between the
// block coder and the finished codestream:
//
//   hdr_trees   one CTA per (precinct, band): the two tag trees bottom-up, with the reference's storage quirk (a
//               level of odd width lets the last column's "right child" alias the first node of the next row,
//               :57-87, :142-165) -- plus, per node, the raster-first INCLUDED leaf below it
//   hdr_items   one thread per code-block: its piece of the header as a bit string.  In a single-layer stream a tag-
//               tree node is sent by exactly one leaf -- the raster-first leaf below it for inclusion, the raster-
//               first included leaf for missing MSBs -- so every block knows its bits without seeing the others'.
//               Also the block's transfer table through the bit-stuffing writer: for each of the 16 writer states
//               (bits already in the current byte, and whether they are all ones) the state it leaves and the number
//               of stuffed bits it causes
//   hdr_groups  one thread per (32 blocks, entry state): composition of the 32 tables
//   hdr_chain   one warp per packet: walks the group compositions -- the only serial part, one shared-memory lookup
//               per 32 blocks -- giving every group its entry state, bit position and body offset, and the packet its
//               header and body sizes
//   hdr_expand  one thread per group: the same for its 32 blocks
//   hdr_write   one thread per block: the bits, stuffed, OR-ed into the packet's header bytes
//   hdr_layout  one CTA: prefix sum over packets (+ 14 bytes of SOT/SOD per tile-part) -> where everything goes;
//               writes SOT segments with their Psot, the TLM entries, EOC and the total length
//   hdr_place   one thread per block: its body's destination (consumed by gather_blocks_kernel, assemble.cu)
//   hdr_copy    warps: header bytes to their place
#include "ojb_device.h"
#include "ojb_kernels.h"

namespace ojb {

namespace {

// ---- the bit-stuffing writer as a finite-state machine ----------------------------------------------------------------
// state = phi | allones << 3: phi bits (0..7) sit in the current byte; allones = they are all 1 and the byte can hold
// eight (a byte after 0xFF holds seven: its first bit is the stuffed 0, so it starts at phi = 1 with allones = 0).
// Start of a packet: phi = 0, allones = 1.
#define HS_START 8u

struct ItemBits {            // MSB-first bit string, up to 160 bits
  uint32_t w[5]; uint32_t n;
  __device__ __forceinline__ void clear() { w[0] = w[1] = w[2] = w[3] = w[4] = 0; n = 0; }
  __device__ __forceinline__ void put(uint32_t v, uint32_t k) {        // the k low bits of v, k <= 32
    while (k) {
      const uint32_t room = 32u - (n & 31u), t = k < room ? k : room;
      const uint32_t chunk = (t == 32u) ? v : ((v >> (k - t)) & ((1u << t) - 1u));
      w[n >> 5] |= chunk << (room - t);
      n += t; k -= t;
    }
  }
  __device__ __forceinline__ void zeros(uint32_t k) { n += k; }
};
// k <= 8 bits of a bit string starting at bit p
__device__ __forceinline__ uint32_t bits_at(const uint32_t* w, uint32_t p, uint32_t k) {
  const uint32_t i = p >> 5, o = p & 31u;
  unsigned long long v = ((unsigned long long)w[i] << 32) | (i + 1 < 5 ? w[i + 1] : 0u);
  return (uint32_t)(v >> (64u - o - k)) & ((1u << k) - 1u);
}

__global__ void __launch_bounds__(256)
hdr_trees_kernel(const HdrSeg* __restrict__ segs, const EncBlock* __restrict__ blocks, const EncResult* __restrict__ results,
                 uint32_t mmsb_base, uint8_t* __restrict__ tinc, uint8_t* __restrict__ tmm, uint32_t* __restrict__ tfi,
                 uint8_t* __restrict__ seg_root)
{
  const HdrSeg sg = segs[blockIdx.x];
  const uint32_t tid = threadIdx.x, n0 = sg.w * sg.h;
  for (uint32_t i = tid; i < n0; i += blockDim.x) {
    const uint32_t y = i / sg.w, x = i - y * sg.w, bi = sg.block0 + y * sg.nbw + x;
    const EncResult r = results[bi];
    const uint32_t len = r.len_head + r.len_tail;
    tinc[sg.tree_off + i] = len ? 0 : 1;
    tmm[sg.tree_off + i] = len ? (uint8_t)(mmsb_base - blocks[bi].p) : 0;       // an empty block enters the minima as 0, as in the reference
    tfi[sg.tree_off + i] = len ? i : 0xFFFFFFFFu;
  }
  __syncthreads();
  uint32_t loff = sg.tree_off, pw = sg.w, ph = sg.h;
  for (uint32_t l = 1; l < sg.nl; ++l) {
    const uint32_t cw = (pw + 1) >> 1, ch = (ph + 1) >> 1, coff = loff + pw * ph, np = pw * ph;
    for (uint32_t i = tid; i < cw * ch; i += blockDim.x) {
      const uint32_t y = i / cw, x = i - y * cw;
      uint32_t vi = 255, vm = 255, vf = 0xFFFFFFFFu;
      #pragma unroll
      for (uint32_t k = 0; k < 4; ++k) {
        const uint32_t X = 2 * x + (k & 1), Y = 2 * y + (k >> 1);
        const uint32_t idx = X + Y * pw;             // linear, as the reference addresses its level arrays: X == pw aliases (0, Y + 1)
        if (idx < np) { vi = min(vi, (uint32_t)tinc[loff + idx]); vm = min(vm, (uint32_t)tmm[loff + idx]); }
        if (X < pw && Y < ph) vf = min(vf, tfi[loff + idx]);
      }
      tinc[coff + i] = (uint8_t)vi; tmm[coff + i] = (uint8_t)vm; tfi[coff + i] = vf;
    }
    __syncthreads();
    loff = coff; pw = cw; ph = ch;
  }
  if (tid == 0) seg_root[blockIdx.x] = tinc[loff];      // the top level has one node
}

// node index of level l above leaf (x, y) inside a segment whose level-0 grid is w x h
__device__ __forceinline__ uint32_t level_off(uint32_t w, uint32_t h, uint32_t l, uint32_t& lw) {
  uint32_t off = 0, pw = w, ph = h;
  for (uint32_t i = 0; i < l; ++i) { off += pw * ph; pw = (pw + 1) >> 1; ph = (ph + 1) >> 1; }
  lw = pw;
  return off;
}

__global__ void __launch_bounds__(128)
hdr_items_kernel(const HdrSeg* __restrict__ segs, const HdrPkt* __restrict__ pkts, const uint32_t* __restrict__ item_seg,
                 uint32_t nitems, const EncResult* __restrict__ results,
                 const uint8_t* __restrict__ tinc, const uint8_t* __restrict__ tmm, const uint32_t* __restrict__ tfi,
                 const uint8_t* __restrict__ seg_root,
                 uint32_t* __restrict__ ibits, uint16_t* __restrict__ inbits, uint16_t* __restrict__ itab, uint32_t* __restrict__ ilen)
{
  const uint32_t it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= nitems) return;
  const uint32_t si = item_seg[it];
  const HdrSeg sg = segs[si];
  const uint32_t local = it - sg.first_item, y = local / sg.w, x = local - y * sg.w;
  const uint32_t bi = sg.block0 + y * sg.nbw + x;
  const EncResult r = results[bi];
  const uint32_t len = r.len_head + r.len_tail;
  const uint32_t root = seg_root[si];
  ItemBits b; b.clear();
  if (local == 0) {
    // what precedes a band's blocks (ojph_precinct.cpp:176-189): the first band with something in it opens the
    // packet with a 1 and a 0 for every band skipped before it; later empty bands cost a 0; a packet with nothing
    // in it is a single 0
    const HdrPkt pk = pkts[sg.pkt];
    bool coded_before = false, coded_any = false; uint32_t skipped = 0;
    for (uint32_t s = pk.first_seg; s < pk.first_seg + pk.nsegs; ++s) {
      const bool c = seg_root[s] == 0;
      if (s < si) { if (c) coded_before = true; else if (!coded_before) ++skipped; }
      coded_any |= c;
    }
    if (!coded_any) { if (si == pk.first_seg) b.zeros(1); }
    else if (root != 0) { if (coded_before) b.zeros(1); }
    else if (!coded_before) { b.put(1, 1); b.zeros(skipped); }
  }
  if (root == 0) {
    // inclusion: this leaf sends the nodes it is the raster-first leaf of, top-down, provided everything above them
    // said "something below" (value 0); a node saying "nothing below" (1) ends the descent
    const uint32_t nl = sg.nl;
    uint32_t L = nl - 1;
    if (x) L = min(L, (uint32_t)__ffs((int)x) - 1u);
    if (y) L = min(L, (uint32_t)__ffs((int)y) - 1u);
    bool open = true;
    for (uint32_t l = nl - 1; l > L && open; --l) {
      uint32_t lw; const uint32_t off = level_off(sg.w, sg.h, l, lw);
      if (tinc[sg.tree_off + off + (x >> l) + (y >> l) * lw]) open = false;
    }
    if (open)
      for (uint32_t l = L + 1; l-- > 0; ) {
        uint32_t lw; const uint32_t off = level_off(sg.w, sg.h, l, lw);
        const uint32_t v = tinc[sg.tree_off + off + (x >> l) + (y >> l) * lw];
        b.put(1u - v, 1);
        if (v) break;
      }
    if (len) {
      // missing MSBs: the nodes whose raster-first included leaf this is, top-down: (value - parent's value) zeros
      // and a one (ojph_precinct.cpp:214-231); the top node's parent counts as 0
      uint32_t Lm = 0;
      while (Lm + 1 < nl) {
        uint32_t lw; const uint32_t off = level_off(sg.w, sg.h, Lm + 1, lw);
        if (tfi[sg.tree_off + off + (x >> (Lm + 1)) + (y >> (Lm + 1)) * lw] != local) break;
        ++Lm;
      }
      uint32_t above = 0;
      if (Lm + 1 < nl) { uint32_t lw; const uint32_t off = level_off(sg.w, sg.h, Lm + 1, lw); above = tmm[sg.tree_off + off + (x >> (Lm + 1)) + (y >> (Lm + 1)) * lw]; }
      for (uint32_t l = Lm + 1; l-- > 0; ) {
        uint32_t lw; const uint32_t off = level_off(sg.w, sg.h, l, lw);
        const uint32_t v = tmm[sg.tree_off + off + (x >> l) + (y >> l) * lw];
        b.zeros(v - above); b.put(1, 1);
        above = v;
      }
      b.zeros(1);                                          // one coding pass (the cleanup pass)
      const uint32_t bits1 = 32u - (uint32_t)__clz((int)len);
      const uint32_t nb = bits1 > 3 ? bits1 - 3 : 0;       // Lblock starts at 3
      b.put(0xFFFFFFFEu, nb + 1);
      b.put(len, nb + 3);
    }
  }
  #pragma unroll
  for (int k = 0; k < 5; ++k) ibits[(size_t)it * 5 + k] = b.w[k];
  inbits[it] = (uint16_t)b.n;
  ilen[it] = len;
  // transfer table through the stuffing writer
  for (uint32_t s = 0; s < 16; ++s) {
    uint32_t phi = s & 7u, a = s >> 3, extra = 0, p = 0;
    if (phi == 0) a = 1;                                   // (0, 0) is not a reachable state; keep the table total
    while (p < b.n) {
      const uint32_t take = min(8u - phi, b.n - p);
      const uint32_t c = bits_at(b.w, p, take);
      a &= (c == ((1u << take) - 1u)) ? 1u : 0u;
      phi += take; p += take;
      if (phi == 8) { if (a) { ++extra; phi = 1; a = 0; } else { phi = 0; a = 1; } }
    }
    itab[(size_t)it * 16 + s] = (uint16_t)(phi | (a << 3) | (extra << 4));
  }
}

// 16 groups x 16 entry states per CTA; the groups' item tables are staged in shared memory first (the walk is a chain
// of 32 dependent look-ups: at global-memory latency it would dominate the kernel)
#define HG_GROUPS 16u
__global__ void __launch_bounds__(256)
hdr_groups_kernel(const HdrGroup* __restrict__ groups, uint32_t ngroups, const uint16_t* __restrict__ itab,
                  const uint16_t* __restrict__ inbits, const uint32_t* __restrict__ ilen,
                  uint32_t* __restrict__ gcomp, uint32_t* __restrict__ gbits, uint32_t* __restrict__ glen)
{
  __shared__ uint32_t stab[HG_GROUPS * 32 * 8];           // 32 items x 16 uint16 per group
  const uint32_t tid = threadIdx.x, gl = tid >> 4, s = tid & 15u;
  const uint32_t g0 = blockIdx.x * HG_GROUPS;
  const uint32_t* itab32 = reinterpret_cast<const uint32_t*>(itab);
  for (uint32_t k = 0; k < HG_GROUPS; ++k) {
    const uint32_t g = g0 + k;
    if (g >= ngroups) break;
    const HdrGroup gr = groups[g];
    if (tid < gr.n * 8) stab[k * 256 + tid] = itab32[(size_t)gr.first_item * 8 + tid];     // 8 words per item
  }
  __syncthreads();
  const uint32_t g = g0 + gl;
  const bool live = g < ngroups;                           // every lane stays for the shuffles below
  HdrGroup gr; gr.first_item = 0; gr.n = 0;
  if (live) gr = groups[g];
  const uint16_t* tab = reinterpret_cast<const uint16_t*>(stab + gl * 256);
  uint32_t st = s, extra = 0;
  for (uint32_t k = 0; k < gr.n; ++k) {
    const uint32_t e = tab[k * 16 + st];
    extra += e >> 4; st = e & 15u;
  }
  if (live) gcomp[(size_t)g * 16 + s] = st | (extra << 4);
  // the group's bit and byte totals: the 16 lanes share the 32 items
  uint32_t nbits = 0, len = 0;
  for (uint32_t k = s; k < gr.n; k += 16) { nbits += inbits[gr.first_item + k]; len += ilen[gr.first_item + k]; }
  #pragma unroll
  for (uint32_t d = 8; d; d >>= 1) { nbits += __shfl_xor_sync(0xFFFFFFFFu, nbits, d, 16); len += __shfl_xor_sync(0xFFFFFFFFu, len, d, 16); }
  if (live && s == 0) { gbits[g] = nbits; glen[g] = len; }
}

#define HC_CHUNK 256u
#define HC_THREADS 256u
__global__ void __launch_bounds__(HC_THREADS)
hdr_chain_kernel(const HdrPkt* __restrict__ pkts, const uint32_t* __restrict__ gcomp, const uint32_t* __restrict__ gbits,
                 const uint32_t* __restrict__ glen, uint32_t* __restrict__ gstate, uint32_t* __restrict__ gpos,
                 uint32_t* __restrict__ gbody, uint32_t* __restrict__ phdr, uint32_t* __restrict__ pbody)
{
  __shared__ uint32_t sc[HC_CHUNK * 16], sb[HC_CHUNK], sl[HC_CHUNK];
  __shared__ uint32_t carry[3];
  const HdrPkt pk = pkts[blockIdx.x];
  const uint32_t tid = threadIdx.x;
  if (tid == 0) { carry[0] = HS_START; carry[1] = 0; carry[2] = 0; }
  for (uint32_t g0 = 0; g0 < pk.ngroups; g0 += HC_CHUNK) {
    const uint32_t n = min(HC_CHUNK, pk.ngroups - g0);
    // the whole CTA fetches the chunk (every thread has its loads in flight at once), one thread walks it
    for (uint32_t i = tid; i < n * 16; i += HC_THREADS) sc[i] = gcomp[(size_t)(pk.first_group + g0) * 16 + i];
    for (uint32_t i = tid; i < n; i += HC_THREADS) { sb[i] = gbits[pk.first_group + g0 + i]; sl[i] = glen[pk.first_group + g0 + i]; }
    __syncthreads();
    if (tid == 0) {
      uint32_t st = carry[0], pos = carry[1], body = carry[2];
      for (uint32_t i = 0; i < n; ++i) {
        const uint32_t g = pk.first_group + g0 + i;
        gstate[g] = st; gpos[g] = pos; gbody[g] = body;
        const uint32_t e = sc[i * 16 + st];
        pos += sb[i] + (e >> 4); st = e & 15u; body += sl[i];
      }
      carry[0] = st; carry[1] = pos; carry[2] = body;
    }
    __syncthreads();
  }
  if (tid == 0) {
    phdr[blockIdx.x] = pk.nitems ? (carry[1] + 7u) >> 3 : 1u;      // a packet without bands is the single zero byte too
    pbody[blockIdx.x] = carry[2];
  }
}

#define HE_GROUPS 32u
__global__ void __launch_bounds__(256)
hdr_expand_kernel(const HdrGroup* __restrict__ groups, uint32_t ngroups, const uint16_t* __restrict__ itab,
                  const uint16_t* __restrict__ inbits, const uint32_t* __restrict__ ilen,
                  const uint32_t* __restrict__ gstate, const uint32_t* __restrict__ gpos, const uint32_t* __restrict__ gbody,
                  uint8_t* __restrict__ istate, uint32_t* __restrict__ ipos, uint32_t* __restrict__ ibody)
{
  // 32 groups per CTA: tables, bit counts and lengths staged by 256 threads, then one thread per group walks its 32 items
  __shared__ uint32_t stab[HE_GROUPS * 256];
  __shared__ uint16_t snb[HE_GROUPS * 32];
  __shared__ uint32_t sln[HE_GROUPS * 32];
  const uint32_t tid = threadIdx.x, g0 = blockIdx.x * HE_GROUPS;
  const uint32_t* itab32 = reinterpret_cast<const uint32_t*>(itab);
  for (uint32_t k = 0; k < HE_GROUPS; ++k) {
    const uint32_t g = g0 + k;
    if (g >= ngroups) break;
    const HdrGroup gr = groups[g];
    if (tid < gr.n * 8) stab[k * 256 + tid] = itab32[(size_t)gr.first_item * 8 + tid];
    if (tid < gr.n) { snb[k * 32 + tid] = inbits[gr.first_item + tid]; sln[k * 32 + tid] = ilen[gr.first_item + tid]; }
  }
  __syncthreads();
  if (tid >= HE_GROUPS) return;
  const uint32_t g = g0 + tid;
  if (g >= ngroups) return;
  const HdrGroup gr = groups[g];
  const uint16_t* tab = reinterpret_cast<const uint16_t*>(stab + tid * 256);
  uint32_t st = gstate[g], pos = gpos[g], body = gbody[g];
  for (uint32_t k = 0; k < gr.n; ++k) {
    const uint32_t it = gr.first_item + k;
    istate[it] = (uint8_t)st; ipos[it] = pos; ibody[it] = body;
    const uint32_t e = tab[k * 16 + st];
    pos += snb[tid * 32 + k] + (e >> 4); st = e & 15u; body += sln[tid * 32 + k];
  }
}

__global__ void __launch_bounds__(128)
hdr_write_kernel(const HdrSeg* __restrict__ segs, const HdrPkt* __restrict__ pkts, const uint32_t* __restrict__ item_seg,
                 uint32_t nitems, const uint32_t* __restrict__ ibits, const uint16_t* __restrict__ inbits,
                 const uint8_t* __restrict__ istate, const uint32_t* __restrict__ ipos, uint32_t* __restrict__ hscr)
{
  const uint32_t it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= nitems) return;
  const uint32_t n = inbits[it];
  if (n == 0) return;
  uint32_t w[5];
  #pragma unroll
  for (int k = 0; k < 5; ++k) w[k] = ibits[(size_t)it * 5 + k];
  const uint64_t base = pkts[segs[item_seg[it]].pkt].hdr_off;        // bytes, multiple of 4
  uint32_t st = istate[it], phi = st & 7u, a = st >> 3, p = 0;
  uint32_t out = ipos[it];                                            // output bit position inside the packet's header
  if (phi == 0) a = 1;
  while (p < n) {
    const uint32_t take = min(8u - phi, n - p);
    const uint32_t c = bits_at(w, p, take);
    a &= (c == ((1u << take) - 1u)) ? 1u : 0u;
    if (c) {
      const uint32_t byte = out >> 3;                                 // phi == out & 7
      const uint32_t v = c << (8u - phi - take);
      atomicOr(hscr + (base >> 2) + (byte >> 2), v << (8u * (byte & 3u)));
    }
    phi += take; p += take; out += take;
    if (phi == 8) { if (a) { ++out; phi = 1; a = 0; } else { phi = 0; a = 1; } }
  }
}

#define HL_THREADS 1024u
__global__ void __launch_bounds__(HL_THREADS)
hdr_layout_kernel(const HdrPkt* __restrict__ pkts, uint32_t npkts, const HdrTp* __restrict__ tps, uint32_t ntps,
                  const uint32_t* __restrict__ phdr, const uint32_t* __restrict__ pbody, uint64_t fixed_len, uint64_t cap,
                  uint32_t write_eoc, uint64_t* __restrict__ ppos, uint8_t* __restrict__ out, uint64_t* __restrict__ total,
                  uint64_t* __restrict__ tp_out)
{
  __shared__ unsigned long long sscan[HL_THREADS];
  __shared__ unsigned long long carry;
  const uint32_t tid = threadIdx.x;
  if (tid == 0) carry = fixed_len;
  __syncthreads();
  for (uint32_t p0 = 0; p0 < npkts; p0 += HL_THREADS) {
    const uint32_t p = p0 + tid;
    unsigned long long v = 0, lead = 0;
    if (p < npkts) { v = (unsigned long long)phdr[p] + pbody[p]; if (pkts[p].tp_first) lead = 14; }   // SOT + SOD ahead of a tile-part's first packet
    sscan[tid] = v + lead;
    __syncthreads();
    for (uint32_t d = 1; d < HL_THREADS; d <<= 1) {
      const unsigned long long t = tid >= d ? sscan[tid - d] : 0;
      __syncthreads();
      sscan[tid] += t;
      __syncthreads();
    }
    if (p < npkts) ppos[p] = carry + sscan[tid] - v;                 // where the packet's header starts
    __syncthreads();
    if (tid == HL_THREADS - 1) carry += sscan[tid];
    __syncthreads();
  }
  const unsigned long long end = carry + (write_eoc ? 2 : 0);
  const bool fits = end <= cap;
  if (tid == 0) { total[0] = end; total[1] = fits ? 0 : 1; }
  if (!fits) return;
  for (uint32_t t = tid; t < ntps; t += HL_THREADS) {
    const HdrTp tp = tps[t];
    const uint32_t last = tp.first_pkt + tp.npkts - 1;
    const unsigned long long start = ppos[tp.first_pkt] - 14;
    const unsigned long long stop = tp.npkts ? ppos[last] + phdr[last] + pbody[last] : start + 14;
    const uint32_t psot = (uint32_t)(stop - start);
    uint8_t* s = out + start;
    s[0] = 0xFF; s[1] = 0x90; s[2] = 0; s[3] = 10; s[4] = (uint8_t)(tp.tile >> 8); s[5] = (uint8_t)tp.tile;
    s[6] = (uint8_t)(psot >> 24); s[7] = (uint8_t)(psot >> 16); s[8] = (uint8_t)(psot >> 8); s[9] = (uint8_t)psot;
    s[10] = (uint8_t)tp.tp_idx; s[11] = (uint8_t)tp.tp_cnt; s[12] = 0xFF; s[13] = 0x93;
    tp_out[2 * t] = start; tp_out[2 * t + 1] = psot;
    if (tp.tlm_off != 0xFFFFFFFFu) {
      uint8_t* m = out + tp.tlm_off;
      m[0] = (uint8_t)(psot >> 24); m[1] = (uint8_t)(psot >> 16); m[2] = (uint8_t)(psot >> 8); m[3] = (uint8_t)psot;
    }
  }
  if (tid == 0 && write_eoc) { out[carry] = 0xFF; out[carry + 1] = 0xD9; }
}

__global__ void __launch_bounds__(128)
hdr_place_kernel(const HdrSeg* __restrict__ segs, const uint32_t* __restrict__ item_seg, uint32_t nitems,
                 const uint32_t* __restrict__ ibody, const uint64_t* __restrict__ ppos, const uint32_t* __restrict__ phdr,
                 const uint64_t* __restrict__ total, uint64_t* __restrict__ dst)
{
  const uint32_t it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it >= nitems) return;
  const HdrSeg sg = segs[item_seg[it]];
  const uint32_t local = it - sg.first_item, y = local / sg.w, x = local - y * sg.w;
  const uint32_t bi = sg.block0 + y * sg.nbw + x;
  dst[bi] = total[1] ? ~0ull : ppos[sg.pkt] + phdr[sg.pkt] + ibody[it];
}

#define HCP_CHUNK 4096u
__global__ void __launch_bounds__(128)
hdr_copy_kernel(const HdrPkt* __restrict__ pkts, uint32_t npkts, const uint32_t* __restrict__ phdr,
                const uint64_t* __restrict__ ppos, const uint64_t* __restrict__ total, const uint8_t* __restrict__ hscr,
                uint8_t* __restrict__ out)
{
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= npkts || total[1]) return;
  const uint32_t n = phdr[warp];
  const uint32_t c0 = blockIdx.y * HCP_CHUNK;
  if (c0 >= n) return;
  const uint32_t m = min(HCP_CHUNK, n - c0);
  const uint8_t* s = hscr + pkts[warp].hdr_off + c0;
  uint8_t* d = out + ppos[warp] + c0;
  for (uint32_t i = lane; i < m; i += 32) d[i] = s[i];
}

} // namespace

void launch_packet_headers(const HdrPlanDev& pl, const EncBlock* blocks, const EncResult* results, uint32_t mmsb_base,
                           uint64_t fixed_len, uint64_t cap, bool write_eoc, uint8_t* out, uint64_t* dst, cudaStream_t st)
{
  if (pl.nsegs)
    OJB_LAUNCH(hdr_trees_kernel, dim3(pl.nsegs), dim3(256), 0, st, pl.segs, blocks, results, mmsb_base, pl.tinc, pl.tmm, pl.tfi, pl.seg_root);
  if (pl.nitems) {
    OJB_LAUNCH(hdr_items_kernel, dim3((pl.nitems + 127) / 128), dim3(128), 0, st, pl.segs, pl.pkts, pl.item_seg, pl.nitems, results,
               pl.tinc, pl.tmm, pl.tfi, pl.seg_root, pl.ibits, pl.inbits, pl.itab, pl.ilen);
    OJB_LAUNCH(hdr_groups_kernel, dim3((pl.ngroups + HG_GROUPS - 1) / HG_GROUPS), dim3(256), 0, st, pl.groups, pl.ngroups, pl.itab, pl.inbits, pl.ilen,
               pl.gcomp, pl.gbits, pl.glen);
  }
  if (pl.npkts)
    OJB_LAUNCH(hdr_chain_kernel, dim3(pl.npkts), dim3(HC_THREADS), 0, st, pl.pkts, pl.gcomp, pl.gbits, pl.glen, pl.gstate, pl.gpos, pl.gbody,
               pl.phdr, pl.pbody);
  if (pl.nitems) {
    OJB_LAUNCH(hdr_expand_kernel, dim3((pl.ngroups + HE_GROUPS - 1) / HE_GROUPS), dim3(256), 0, st, pl.groups, pl.ngroups, pl.itab, pl.inbits, pl.ilen,
               pl.gstate, pl.gpos, pl.gbody, pl.istate, pl.ipos, pl.ibody);
    OJB_LAUNCH(hdr_write_kernel, dim3((pl.nitems + 127) / 128), dim3(128), 0, st, pl.segs, pl.pkts, pl.item_seg, pl.nitems, pl.ibits,
               pl.inbits, pl.istate, pl.ipos, pl.hscr);
  }
  OJB_LAUNCH(hdr_layout_kernel, dim3(1), dim3(HL_THREADS), 0, st, pl.pkts, pl.npkts, pl.tps, pl.ntps, pl.phdr, pl.pbody, fixed_len, cap,
             write_eoc ? 1u : 0u, pl.ppos, out, pl.total, pl.tp_out);
  if (pl.nitems)
    OJB_LAUNCH(hdr_place_kernel, dim3((pl.nitems + 127) / 128), dim3(128), 0, st, pl.segs, pl.item_seg, pl.nitems, pl.ibody, pl.ppos,
               pl.phdr, pl.total, dst);
  if (pl.npkts) {
    const uint32_t chunks = (pl.max_hdr_cap + HCP_CHUNK - 1) / HCP_CHUNK;
    OJB_LAUNCH(hdr_copy_kernel, dim3((pl.npkts + 3) / 4, chunks ? chunks : 1), dim3(128), 0, st, pl.pkts, pl.npkts, pl.phdr, pl.ppos, pl.total,
               (const uint8_t*)pl.hscr, out);
  }
}

// the stream size alone: the header kernels up to the layout's prefix sum, with no room to write (pl.total[0] only)
void launch_packet_header_total(const HdrPlanDev& pl, const EncBlock* blocks, const EncResult* results, uint32_t mmsb_base,
                                uint64_t fixed_len, bool write_eoc, cudaStream_t st)
{
  if (pl.nsegs)
    OJB_LAUNCH(hdr_trees_kernel, dim3(pl.nsegs), dim3(256), 0, st, pl.segs, blocks, results, mmsb_base, pl.tinc, pl.tmm, pl.tfi, pl.seg_root);
  if (pl.nitems) {
    OJB_LAUNCH(hdr_items_kernel, dim3((pl.nitems + 127) / 128), dim3(128), 0, st, pl.segs, pl.pkts, pl.item_seg, pl.nitems, results,
               pl.tinc, pl.tmm, pl.tfi, pl.seg_root, pl.ibits, pl.inbits, pl.itab, pl.ilen);
    OJB_LAUNCH(hdr_groups_kernel, dim3((pl.ngroups + HG_GROUPS - 1) / HG_GROUPS), dim3(256), 0, st, pl.groups, pl.ngroups, pl.itab, pl.inbits, pl.ilen,
               pl.gcomp, pl.gbits, pl.glen);
  }
  if (pl.npkts)
    OJB_LAUNCH(hdr_chain_kernel, dim3(pl.npkts), dim3(HC_THREADS), 0, st, pl.pkts, pl.gcomp, pl.gbits, pl.glen, pl.gstate, pl.gpos, pl.gbody,
               pl.phdr, pl.pbody);
  OJB_LAUNCH(hdr_layout_kernel, dim3(1), dim3(HL_THREADS), 0, st, pl.pkts, pl.npkts, pl.tps, pl.ntps, pl.phdr, pl.pbody, fixed_len, (uint64_t)0,
             write_eoc ? 1u : 0u, pl.ppos, (uint8_t*)nullptr, pl.total, pl.tp_out);
}
uint32_t packet_header_total_launches(const HdrPlanDev& pl) {
  return (pl.nsegs ? 1u : 0u) + (pl.nitems ? 2u : 0u) + (pl.npkts ? 1u : 0u) + 1u;
}

uint32_t packet_header_launches(const HdrPlanDev& pl) {
  return (pl.nsegs ? 1u : 0u) + (pl.nitems ? 5u : 0u) + (pl.npkts ? 2u : 0u) + 1u;
}

} // namespace ojb
