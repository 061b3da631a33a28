// ojb_params.h -- codestream parameters (SIZ / CAP / COD / QCD / QCC / SOT / TLM) for the
// GPU HTJ2K path: the host-side metadata that wraps the GPU kernels in a valid codestream.
//
// Mirrors the behaviour of the reference's parameter classes so that main headers are
// byte-identical for the same settings:
//   SIZ  src/core/codestream/ojph_params.cpp:805-851   (write)  :854-933 (read)
//   CAP  :968-989, check ojph_params_local.h:982-998
//   COD  :1035-1078 (write) :1146-1204 (read)
//   QCD  :1359-1481 (validity / step derivation) :1495-1612 (steps) :1778-1887 (write)
//   SOT  :2343-2388   TLM :2470-2520
#pragma once
#include "ojb_common.h"

namespace ojb {

enum ProgOrder : uint8_t { PO_LRCP = 0, PO_RLCP = 1, PO_RPCL = 2, PO_PCRL = 3, PO_CPRL = 4 };
enum Wavelet : uint8_t { DWT_IRV97 = 0, DWT_REV53 = 1 };
enum TilepartDiv : uint32_t { TP_NONE = 0, TP_RES = 1, TP_COMP = 2 };

struct CompInfo {
  uint8_t bit_depth = 8;
  bool is_signed = false;
  uint8_t dx = 1, dy = 1;
};

// One QCD or QCC marker segment plus the inputs its step sizes are generated from
struct QuantSet {
  bool is_qcc = false;
  bool enabled = true;
  bool is_init = false;
  uint16_t comp_idx = 0xFFFF;
  uint8_t Sqcd = 0;
  uint32_t num_subbands = 0;
  uint16_t SP[97] = {0};        // 8-bit entries (reversible) or 16-bit (scalar expounded)
  float base_delta = -1.0f;
  uint8_t qfactor = 0;          // 0 = unset
  int ctype = 0;                // 0 Y, 1 Cb, 2 Cr
  uint32_t num_decomps = 0, bit_depth = 0;
  bool is_signed = false, is_color_trans = false;
  uint32_t wavelet = 0;
  uint32_t sx = 1, sy = 1;

  uint32_t guard_bits() const { return (uint32_t)(Sqcd >> 5); }
  uint32_t kmax(uint32_t res, uint32_t band) const { return kmax_at(res ? (res - 1) * 3 + band : 0); }   // get_Kmax, ojph_params.cpp:1715
  uint32_t kmax_at(uint32_t idx) const;
  uint32_t largest_kmax() const;                             // :1751
  float irrev_delta(uint32_t res, uint32_t band) const { return irrev_delta_at(res ? (res - 1) * 3 + band : 0, band); }   // get_irrev_delta, :1650
  float irrev_delta_at(uint32_t idx, uint32_t band) const;
  void set_rev_quant(uint32_t num_decomps, uint32_t bit_depth, bool color);   // :1495
  void set_irrev_quant(uint32_t num_decomps);                                // :1542
};

// Part 2 wavelet structures the reference DECODES (it never writes them): down-sampling factor styles (DFS marker,
// param_dfs, ojph_params_local.h:1032-1094, ojph_params.cpp:2530-2645) and arbitrary transformation kernels
// (ATK marker, param_atk, ojph_params_local.h:1103-1232, ojph_params.cpp:2654-2895)
enum DfsType : uint8_t { DFS_NONE = 0, DFS_BIDIR = 1, DFS_HORZ = 2, DFS_VERT = 3 };
struct DfsSpec {
  uint16_t Sdfs = 0;             // index, <= 15
  uint8_t Ids = 0;               // number of decomposition levels described, <= 32 kept
  uint8_t Ddfs[8] = {0};         // 2 bits per level, finest level first
  DfsType type(uint32_t decomp_level) const;                                        // get_dwt_type, :2539
  uint32_t subband_idx(const uint32_t num_decomps, uint32_t res, uint32_t band) const;     // get_subband_idx, :2550
};
struct AtkStep { float A = 0.f; int16_t a = 0, b = 0; uint8_t e = 0; };   // irreversible: A; reversible: (b + a (x[-1] + x[+1])) >> e
struct AtkSpec {
  uint16_t Satk = 0;
  float K = 1.0f;
  std::vector<AtkStep> steps;    // in SYNTHESIS order: step 0 is undone first and acts on the even (low-pass) samples
  uint32_t index() const { return Satk & 0xFFu; }
  uint32_t coeff_type() const { return (Satk >> 8) & 7u; }
  bool reversible() const { return (Satk & 0x1000) != 0; }
  static AtkSpec irv97();        // init_irv97, :2870
  static AtkSpec rev53();        // init_rev53, :2884
};

// per-component coding style (COC marker segment; param_cod with type COC_MAIN,
// ojph_params_local.h:330-440).  A new object starts from the library defaults -- not from the COD
// values -- exactly as param_cod::init does (:630-646)
struct CodStyle {
  uint16_t comp_idx = 0xFFFF;
  uint8_t Scoc = 0;                         // bit 0: user precinct sizes follow
  uint8_t num_decomps = 5, cb_w_exp = 4, cb_h_exp = 4, block_style = 0x40, wavelet = DWT_IRV97;
  uint8_t precinct_size[33] = {0};
  int dfs_idx = -1;                         // >= 0: SPcoc's decomposition byte is 0x80 | index of a DFS marker segment,
                                            // and the number of decompositions is the COD's (get_num_decompositions,
                                            // ojph_params_local.h:503-518)
};

// one NLT marker segment (param_nlt, ojph_params_local.h:840-910): Cnlt = 0xFFFF is the default entry
// for all components
struct NltEntry {
  uint16_t comp_idx = 0xFFFF;
  uint8_t BDnlt = 0;
  uint8_t Tnlt = 0xFF;                      // 0 none, 3 binary complement <-> sign magnitude; 0xFF undefined
  bool enabled = false;
};

struct Comment {                            // comment_exchange, ojph_codestream.h / ojph_params.h
  std::vector<uint8_t> data;
  uint16_t Rcom = 1;                        // 0 binary, 1 Latin text
};

struct Params {
  // ---- SIZ
  uint16_t Rsiz = 0x4000;
  uint32_t Xsiz = 0, Ysiz = 0, XOsiz = 0, YOsiz = 0;
  uint32_t XTsiz = 0, YTsiz = 0, XTOsiz = 0, YTOsiz = 0;
  std::vector<CompInfo> comps;
  // ---- COD
  uint8_t Scod = 0;
  uint8_t prog_order = PO_RPCL;
  uint16_t num_layers = 1;
  uint8_t mc_trans = 0;
  uint8_t num_decomps = 5;
  uint8_t cb_w_exp = 4, cb_h_exp = 4;       // log2(dim) - 2
  uint8_t block_style = 0x40;               // HT
  uint8_t wavelet = DWT_IRV97;
  uint8_t precinct_size[33] = {0};          // PPx | PPy << 4 per resolution (Scod & 1)
  std::vector<CodStyle> coc;                // per-component overrides, in creation order
  // ---- DFS / ATK (Part 2), in marker order
  std::vector<DfsSpec> dfs;
  std::vector<AtkSpec> atk;
  // encoder request (this library's own extension -- the reference has no writer for these): one decomposition
  // structure and / or one kernel for every component.  enc_dfs lists DfsType per level, finest first.
  std::vector<uint8_t> enc_dfs;
  bool enc_atk_set = false;
  AtkSpec enc_atk;
  // ---- QCD / QCC
  QuantSet qcd;
  std::vector<QuantSet> qcc;                // in creation order
  // ---- NLT
  NltEntry nlt_all;                         // the ALL_COMPS entry
  std::vector<NltEntry> nlt;                // per-component entries, in creation order
  // ---- COM (after the library's own signature comment)
  std::vector<Comment> comments;
  // ---- CAP
  uint32_t Pcap = 0x00020000;
  uint16_t Ccap0 = 0;
  // ---- encoder options
  uint32_t profile = 0;                     // codestream::set_profile: 0 none, 1 IMF, 2 BROADCAST
  bool need_tlm = false;
  uint32_t tilepart_div = TP_NONE;
  int planar = -1;

  // helpers
  uint32_t num_comps() const { return (uint32_t)comps.size(); }
  bool reversible() const { return wavelet <= 1 ? wavelet == DWT_REV53 : atk_for(wavelet).reversible(); }
  bool color_transform() const { return mc_trans == 1; }
  uint32_t log_cb_w() const { return cb_w_exp + 2u; }
  uint32_t log_cb_h() const { return cb_h_exp + 2u; }
  uint32_t log_pp_w(uint32_t r) const { return (Scod & 1) ? (precinct_size[r] & 0xF) : 15u; }
  uint32_t log_pp_h(uint32_t r) const { return (Scod & 1) ? (precinct_size[r] >> 4) : 15u; }
  bool stripe_causal() const { return (block_style & 0x8) != 0; }
  // per-component views: the component's COC when it has one, else the COD values
  const CodStyle* find_coc(uint32_t c) const { for (const CodStyle& s : coc) if (s.comp_idx == c) return &s; return nullptr; }
  CodStyle& get_or_add_coc(uint32_t c) {                           // param_cod::get_or_add_coc, ojph_params.cpp:1341
    for (CodStyle& s : coc) if (s.comp_idx == c) return s;
    coc.push_back(CodStyle()); coc.back().comp_idx = (uint16_t)c; return coc.back();
  }
  uint32_t decomps(uint32_t c) const { const CodStyle* s = find_coc(c); return (s && s->dfs_idx < 0) ? s->num_decomps : num_decomps; }
  uint32_t max_decomps() const { uint32_t d = 0; for (uint32_t c = 0; c < num_comps(); ++c) d = std::max(d, decomps(c)); return d; }
  uint32_t wavelet_of(uint32_t c) const { const CodStyle* s = find_coc(c); return s ? s->wavelet : wavelet; }
  bool reversible(uint32_t c) const { uint32_t w = wavelet_of(c); return w <= 1 ? w == DWT_REV53 : atk_for(w).reversible(); }
  // the kernel with index w: 0 and 1 are the built-in 9/7 and 5/3 (param_atk::get_atk, ojph_params.cpp:2654-2684)
  const AtkSpec& atk_for(uint32_t w) const;
  const AtkSpec& atk_of(uint32_t c) const { return atk_for(wavelet_of(c)); }
  const DfsSpec* dfs_of(uint32_t c) const;                         // nullptr: dyadic (Mallat) decomposition
  // how decomposition level `level` (1 = finest) of component c splits its resolution
  DfsType dwt_type(uint32_t c, uint32_t level) const { const DfsSpec* d = dfs_of(c); return d ? d->type(level) : DFS_BIDIR; }
  bool is_part2(uint32_t c) const { return dfs_of(c) != nullptr || wavelet_of(c) > 1; }
  bool any_part2() const { for (uint32_t c = 0; c < num_comps(); ++c) if (is_part2(c)) return true; return false; }
  // resolution down-sampling after `skipped` levels from the top (param_dfs::get_res_downsamp, :2575)
  void res_downsamp(uint32_t c, uint32_t skipped, uint32_t& fx, uint32_t& fy) const;
  // index of (resolution, band) in the component's QCD / QCC step list
  uint32_t subband_index(uint32_t c, uint32_t res, uint32_t band) const;
  uint32_t band_kmax(uint32_t c, uint32_t res, uint32_t band) const { return quant_for(c).kmax_at(subband_index(c, res, band)); }
  float band_delta(uint32_t c, uint32_t res, uint32_t band) const { return quant_for(c).irrev_delta_at(subband_index(c, res, band), band); }
  // squared L2 norm of one coefficient's synthesis waveform, per sub-band index of component c (rate control's weights)
  std::vector<double> band_energy_gains(uint32_t c) const;
  uint32_t log_cb_w(uint32_t c) const { const CodStyle* s = find_coc(c); return (s ? s->cb_w_exp : cb_w_exp) + 2u; }
  uint32_t log_cb_h(uint32_t c) const { const CodStyle* s = find_coc(c); return (s ? s->cb_h_exp : cb_h_exp) + 2u; }
  uint32_t log_pp_w(uint32_t c, uint32_t r) const {
    const CodStyle* s = find_coc(c);
    if (s) return (s->Scoc & 1) ? (s->precinct_size[r] & 0xF) : 15u;
    return log_pp_w(r);
  }
  uint32_t log_pp_h(uint32_t c, uint32_t r) const {
    const CodStyle* s = find_coc(c);
    if (s) return (s->Scoc & 1) ? (s->precinct_size[r] >> 4) : 15u;
    return log_pp_h(r);
  }
  bool stripe_causal(uint32_t c) const { const CodStyle* s = find_coc(c); return ((s ? s->block_style : block_style) & 0x8) != 0; }
  bool mixed_wavelets() const { for (uint32_t c = 0; c < num_comps(); ++c) if (wavelet_of(c) != wavelet_of(0)) return true; return false; }
  bool uses_sop() const { return (Scod & 2) != 0; }
  bool uses_eph() const { return (Scod & 4) != 0; }
  uint32_t comp_width(uint32_t c) const
  { return div_ceil(Xsiz, comps[c].dx) - div_ceil(XOsiz, comps[c].dx); }
  uint32_t comp_height(uint32_t c) const
  { return div_ceil(Ysiz, comps[c].dy) - div_ceil(YOsiz, comps[c].dy); }
  const QuantSet& quant_for(uint32_t c) const;
  QuantSet* find_qcc(uint32_t c);
  QuantSet& add_qcc(uint32_t c);
  uint32_t precision(uint32_t c) const;     // propose_precision, ojph_params.cpp:1684
  // true when some component needs more than 32 bits (the reference's 64-bit line buffers and code-block words,
  // ojph_codeblock.cpp:85-91); fails when such a component is irreversible (not built here)
  bool needs_wide() const;

  // NLT (param_nlt, ojph_params.cpp:2087-2330)
  void set_nonlinear_transform(uint32_t comp, uint32_t type);      // comp 65535 = all components
  void nlt_check_validity();
  // the transform in force for component c (0 or 3); raises on a BDnlt / SIZ mismatch as tile setup does
  uint32_t nlt_type(uint32_t c) const;
  bool nlt_any() const { if (nlt_all.enabled) return true; for (const NltEntry& e : nlt) if (e.enabled) return true; return false; }

  // profile rules (check_imf_validity / check_broadcast_validity, ojph_codestream_local.cpp:292-535)
  void check_profile();

  // setters used by the C-ABI (same argument checks as ojph::param_cod / param_qcd setters)
  void set_block_dims(uint32_t w, uint32_t h);                      // ojph_params.cpp:170-181
  void set_precincts(int n, const uint32_t* w, const uint32_t* h);  // :184-209

  // finalisation before writing headers (write_headers, ojph_codestream_local.cpp:556-636)
  void finalize_for_encode();
  // CAP's MAGB field (Ccap0 bits 0-4) for the QCD / QCC step-size lists
  uint32_t cap_magb() const;
  void write_main_header(std::vector<uint8_t>& out, const char* const* comments,
                         const uint32_t* comment_lens, uint32_t n_comments) const;
  // decoder: parse from SOC up to (not including) the first SOT; returns offset of that SOT
  size_t read_main_header(const uint8_t* data, size_t len);
};

// The main header `hdr` (SOC up to the first SOT, without TLM / PLM) of a codestream with parameters `in`, rewritten
// for the same codestream with its top r resolution levels dropped, and the parameters of that header.  Every kept
// tile, resolution, band, precinct and code-block keeps its rectangle and its quantisation:
//   SIZ      extent, image offset and tile offset / 2^r rounded up (ceil(ceil(a / b) / c) = ceil(a / (b c)), also with
//            sub-sampling); the tile size / 2^r along a direction with several tiles, else rounded up
//   COD/COC  r fewer levels; user precinct sizes 0 .. D_c - r
//   QCD/QCC  the first 1 + 3 (D_c - r) step-size entries (they are indexed from the LL band up); guard bits and Sqcd kept
//   CAP      MAGB recomputed from the cut lists
// Every other segment is copied byte for byte.  Refused: r above some component's level count (0x000300A2, 0x000B0007,
// as restrict_input_resolution), a DFS decomposition (0x000B0054), a tile grid whose tiles would not all keep samples
// or whose tile size along a direction with several tiles is not a multiple of 2^r (0x000B0055), and a profile the
// input's Rsiz claims that the reduced parameters break (0x000B0056).
void reduce_main_header(const std::vector<uint8_t>& hdr, const Params& in, uint32_t r, std::vector<uint8_t>& out,
                        Params& outp);

// marker codes
enum Marker : uint16_t {
  M_SOC = 0xFF4F, M_CAP = 0xFF50, M_SIZ = 0xFF51, M_COD = 0xFF52, M_COC = 0xFF53,
  M_TLM = 0xFF55, M_PRF = 0xFF56, M_PLM = 0xFF57, M_PLT = 0xFF58, M_CPF = 0xFF59,
  M_QCD = 0xFF5C, M_QCC = 0xFF5D, M_RGN = 0xFF5E, M_POC = 0xFF5F, M_PPM = 0xFF60,
  M_PPT = 0xFF61, M_CRG = 0xFF63, M_COM = 0xFF64, M_DFS = 0xFF72, M_ADS = 0xFF73,
  M_NLT = 0xFF76, M_ATK = 0xFF79, M_SOT = 0xFF90, M_SOP = 0xFF91, M_EPH = 0xFF92,
  M_SOD = 0xFF93, M_EOC = 0xFFD9
};

inline void put_u8(std::vector<uint8_t>& o, uint32_t v) { o.push_back((uint8_t)v); }
inline void put_u16(std::vector<uint8_t>& o, uint32_t v)
{ o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }
inline void put_u32(std::vector<uint8_t>& o, uint32_t v)
{ put_u16(o, v >> 16); put_u16(o, v & 0xFFFF); }

} // namespace ojb
