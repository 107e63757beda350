// Host launchers of the wgmma GEMMs: TMA descriptor construction (driver entry point
// resolved at run time, so the library loads on a box without libcuda), tile-shape
// selection, stream-K planning and kernel dispatch.
#include "gemm.cuh"
#include "gemm_prefill.cuh"
#include "gemm_prefill_q.cuh"
#include "gemm_vit.cuh"
#include "gemm_ws.cuh"
#include "gemm_wsf.cuh"

#include <cudaTypedefs.h>

#include <cstdio>
#include <algorithm>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "common.h"

namespace vlo {

namespace {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                              CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                              CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  });
  return fn;
}

struct TmapKey {
  const void* ptr;
  int rows, k, box_rows, fmt;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && rows == o.rows && k == o.k && box_rows == o.box_rows && fmt == o.fmt;
  }
};
struct TmapHash {
  size_t operator()(const TmapKey& x) const {
    size_t h = reinterpret_cast<size_t>(x.ptr);
    h ^= (static_cast<size_t>(x.rows) * 0x9E3779B97F4A7C15ull) + (h << 6) + (h >> 2);
    h ^= (static_cast<size_t>(x.k) * 0xC2B2AE3D27D4EB4Full) + (h << 6) + (h >> 2);
    h ^= static_cast<size_t>(x.box_rows * 2 + x.fmt) + (h << 6) + (h >> 2);
    return h;
  }
};

std::mutex g_tmap_mu;
std::unordered_map<TmapKey, CUtensorMap, TmapHash> g_tmaps;

// [rows, k] row-major 16-bit matrix, box = 64 (k) x box_rows, 128-byte swizzle; FMT_E4M3: bytes, box = 64 B x box_rows,
// no swizzle (the consumer reads the stage with plain loads); FMT_E4M3_A8: bytes, box = 64 B x box_rows, 64-byte swizzle
// (the FP8 wgmma reads the stage).
int get_tmap(const void* ptr, int rows, int k, int box_rows, int fmt, CUtensorMap* out) {
  TmapKey key{ptr, rows, k, box_rows, fmt};
  {
    std::lock_guard<std::mutex> g(g_tmap_mu);
    auto it = g_tmaps.find(key);
    if (it != g_tmaps.end()) {
      *out = it->second;
      return 0;
    }
  }
  EncodeFn enc = get_encode();
  if (enc == nullptr) return fail("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) return fail("TMA operand not 16-byte aligned");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows)};
  const bool a8 = fmt == FMT_E4M3_A8;
  const bool f8 = fmt == FMT_E4M3 || a8;
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(k) * (f8 ? 1 : 2)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kGemmBK), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUtensorMap m;
  CUresult r = enc(&m,
                   f8                  ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                   : fmt == FMT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                     : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                   2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   a8 ? CU_TENSOR_MAP_SWIZZLE_64B : f8 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed, CUresult " + std::to_string(r));
  {
    std::lock_guard<std::mutex> g(g_tmap_mu);
    g_tmaps.emplace(key, m);
  }
  *out = m;
  return 0;
}

template <int BN, int EPI>
int launch_one(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& args, dim3 grid,
               cudaStream_t stream) {
  auto kern = gemm_tn_kernel<BN, EPI>;
  if (ensure_max_smem(reinterpret_cast<const void*>(kern), GemmCfg<BN>::kSmemBytes)) return -1;
  if (prof_on()) {
    const double esz = (EPI == EPI_STORE16) ? 2.0 : 4.0;
    const double bytes = 2.0 * args.k * (static_cast<double>(args.rows_a) + args.rows_b) +
                         esz * static_cast<double>(args.rows_a) * args.rows_b;
    prof_begin(PROF_GEMM_VIT, stream, bytes);
  }
  VLO_CUDA(launch_pdl(kern, grid, dim3(kGemmThreads), GemmCfg<BN>::kSmemBytes, stream, ta, tb, args));
  prof_end(stream);
  count_launch();
  return 0;
}

}  // namespace

// N-tile width of the ViT's one-tile GEMMs: prefer a single wave of CTAs (one CTA per SM); two waves cost 2x.
int vit_bn(int rows, int n_out) {
  const int mt = (rows + 127) / 128;
  const int t64 = mt * ((n_out + 63) / 64), t128 = mt * ((n_out + 127) / 128);
  if (t64 <= num_sms()) return 64;     // everything fits in one wave even with the narrow tile
  if (t128 <= num_sms()) return 128;   // one wave with the wide tile
  // multi-wave: wide tiles (better operand reuse) unless the narrow ones waste much less of the last wave
  const double e64 = static_cast<double>(t64) / (((t64 + num_sms() - 1) / num_sms()) * num_sms());
  const double e128 = static_cast<double>(t128) / (((t128 + num_sms() - 1) / num_sms()) * num_sms());
  return e64 > e128 + 0.15 ? 64 : 128;
}

int tmap_2d_sw128(const void* ptr, int rows, int k, int box_rows, int fmt, CUtensorMap* out) {
  return get_tmap(ptr, rows, k, box_rows, fmt, out);
}

int gemm_launch(const GemmCall& c, cudaStream_t stream) {
  VLO_CHECK(c.k > 0 && c.k % kGemmBK == 0, "K must be a positive multiple of 64");
  VLO_CHECK(c.rows_a > 0 && c.rows_b > 0, "empty GEMM operand");
  const int bn = c.bn > 0 ? c.bn : vit_bn(c.rows_a, c.rows_b);
  GemmArgs a{};
  a.rows_a = c.rows_a;
  a.rows_b = c.rows_b;
  a.k = c.k;
  a.out = c.out;
  a.ld_out = c.ld_out;
  a.bias = c.bias;
  a.pos = c.pos;
  a.pos_rows = c.pos_rows > 0 ? c.pos_rows : 1;
  a.act = c.act;

  CUtensorMap ta, tb;
  if (get_tmap(c.a, c.rows_a, c.k, kGemmBM, FMT_F16, &ta) != 0) return -1;
  if (get_tmap(c.b, c.rows_b, c.k, bn, FMT_F16, &tb) != 0) return -1;
  dim3 grid((c.rows_a + kGemmBM - 1) / kGemmBM, (c.rows_b + bn - 1) / bn);

  if (bn == 64 && c.epi == EPI_STORE16) return launch_one<64, EPI_STORE16>(ta, tb, a, grid, stream);
  if (bn == 128 && c.epi == EPI_STORE16) return launch_one<128, EPI_STORE16>(ta, tb, a, grid, stream);
  if (bn == 64 && c.epi == EPI_PATCH32) return launch_one<64, EPI_PATCH32>(ta, tb, a, grid, stream);
  if (bn == 128 && c.epi == EPI_PATCH32) return launch_one<128, EPI_PATCH32>(ta, tb, a, grid, stream);
  return fail("gemm_launch: no kernel instance for bn=" + std::to_string(bn) + " epi=" + std::to_string(c.epi));
}

// ------------------------------------------------------------------------------------------------
// persistent weight-streaming GEMM (gemm_ws.cuh)

// The default single-stream frame step runs the ViT of frame i+1 (gemm_vit_kernel for QKV / fc1, the 64-token
// small-tile configuration of gemm_ws_kernel for out_proj / fc2) next to the decoder step of frame i (16-token tiles).
// One CTA of each fits on one sm_90 SM: 228 KB of shared memory per SM, of which 1 KB is reserved per resident block.
// The fused gate|up GEMM's 8-stage ring leaves no room for a gemm_vit_kernel CTA (a 6-stage ring would, and measured no
// faster: DESIGN.md section 5).
constexpr int kSmemPerSm = 233472, kSmemReservedPerBlock = 1024;
constexpr int kVitBesideBytes = GemmWsCfg<FMT_F16, 64, 3>::kSmemBytes;   // the 64-token ViT GEMM CTA (83 KB)
// Ring depth of the 16-token decoder GEMM of each weight format.  bf16: 6 x 18 KB, measured.  The others: the deepest
// ring that fits beside the ViT trunk GEMM CTA, up to the format's cap (e4m3: 8 stages of 10 KB next to the two
// converted 16 KB tiles, 64 KB of weights in flight; W8A8: 9 KB stages; int4: 24 KB slots of 16 KB of codes and 8 KB of
// activations; DESIGN.md section 5).
constexpr int decoder_stages(int fmt) {
  return fmt == FMT_BF16 ? 6
                         : std::min(ws_max_stages(fmt), (kSmemPerSm - 2 * kSmemReservedPerBlock - GemmVitCfg::kSmemBytes -
                                                         ws_fixed_bytes(fmt, 0)) /
                                                            (ws_slot_bytes_w(fmt, 16) + ws_slot_bytes_x(fmt, 16)));
}
template <int FMT>
constexpr bool decoder_shares_sm() {
  constexpr int dec = GemmWsCfg<FMT, 16, decoder_stages(FMT)>::kSmemBytes + 2 * kSmemReservedPerBlock;
  return dec + GemmVitCfg::kSmemBytes <= kSmemPerSm && dec + kVitBesideBytes <= kSmemPerSm;
}
static_assert(decoder_shares_sm<FMT_BF16>(), "bf16 decoder GEMM CTA and a ViT GEMM CTA no longer share an SM");
static_assert(decoder_shares_sm<FMT_E4M3>(), "e4m3 decoder GEMM CTA and a ViT GEMM CTA no longer share an SM");
static_assert(decoder_shares_sm<FMT_E4M3_A8>(), "W8A8 decoder GEMM CTA and a ViT GEMM CTA no longer share an SM");
static_assert(decoder_shares_sm<FMT_I4>(), "int4 decoder GEMM CTA and a ViT GEMM CTA no longer share an SM");
static_assert(GemmWsCfg<FMT_BF16, 16, ws_default_stages(FMT_BF16, 16, kWsfXchBytes), kWsfXchBytes>::kSmemBytes +
                      GemmVitCfg::kSmemBytes + 2 * kSmemReservedPerBlock > kSmemPerSm,
              "the 8-stage fused decoder GEMM now shares its SM with a ViT trunk GEMM CTA: update the comment above");

// The whole-tile e4m3 and int4 instances (the vocabulary matrices) take the decoder instances' ring depths, so the
// 16-token one still shares its SM with a ViT trunk GEMM CTA next to the frame step.
template <int FMT>
constexpr bool tiles_share_sm() {
  constexpr int dec = GemmWsCfg<FMT, 16, decoder_stages(FMT)>::kSmemBytes + 2 * kSmemReservedPerBlock;
  return ws_tiles_own_instances(FMT) && dec + GemmVitCfg::kSmemBytes <= kSmemPerSm && dec + kVitBesideBytes <= kSmemPerSm;
}
static_assert(tiles_share_sm<FMT_E4M3>(), "16-token whole-tile e4m3 GEMM CTA and a ViT GEMM CTA no longer share an SM");
static_assert(tiles_share_sm<FMT_I4>(), "16-token whole-tile int4 GEMM CTA and a ViT GEMM CTA no longer share an SM");

namespace {
template <int FMT, int BN, int STAGES = ws_default_stages(FMT, BN), bool TILES = false>
int launch_ws(const CUtensorMap& tw, const CUtensorMap& tx, const GemmWsArgs& a, cudaStream_t stream) {
  auto kern = gemm_ws_kernel<FMT, BN, STAGES>;
  if constexpr (TILES) kern = gemm_ws_tiles_kernel<FMT, BN, STAGES>;
  using Cfg = GemmWsCfg<FMT, BN, STAGES>;
  if (ensure_max_smem(reinterpret_cast<const void*>(kern), Cfg::kSmemBytes)) return -1;
  if (prof_on()) {
    const double out_b = a.mode == 0 ? 4.0 * a.rows_x * a.rows_w : 2.0 * a.rows_x * a.rows_w;
    prof_begin(FMT == FMT_F16 ? PROF_GEMM_VIT : PROF_GEMM_STREAM, stream, ws_in_bytes(FMT, a.rows_w, a.rows_x, a.k) + out_b);
  }
  VLO_CUDA(launch_pdl(kern, dim3(a.sk.G), dim3(kGemmThreads), Cfg::kSmemBytes, stream, tw, tx, a));
  prof_end(stream);
  count_launch();
  return 0;
}

// the instances of one format: every decoder token tile, the 16-token one at its decoder ring depth; fp16 also has the
// 192-wide ViT trunk tile and the 3-stage 64-token ring that fits beside a decoder CTA
template <int FMT>
int launch_ws_fmt(int bn, bool beside, const CUtensorMap& tw, const CUtensorMap& tx, const GemmWsArgs& a,
                  cudaStream_t stream) {
  if constexpr (FMT == FMT_F16) {
    if (beside) return launch_ws<FMT_F16, 64, 3>(tw, tx, a, stream);
    if (bn == 192) return launch_ws<FMT_F16, 192>(tw, tx, a, stream);
  }
  switch (bn) {
    case 16: return launch_ws<FMT, 16, FMT == FMT_F16 ? ws_default_stages(FMT, 16) : decoder_stages(FMT)>(tw, tx, a, stream);
    case 32: return launch_ws<FMT, 32>(tw, tx, a, stream);
    case 64: return launch_ws<FMT, 64>(tw, tx, a, stream);
    case 96: return launch_ws<FMT, 96>(tw, tx, a, stream);
    case 128: return launch_ws<FMT, 128>(tw, tx, a, stream);
  }
  return fail("gemm_ws_launch: no kernel instance");
}

// the whole-tile instances of e4m3 and int4 weights, at the token tiles and ring depths of the format's decoder instances
template <int FMT>
int launch_ws_tiles_fmt(int bn, const CUtensorMap& tw, const CUtensorMap& tx, const GemmWsArgs& a, cudaStream_t stream) {
  switch (bn) {
    case 16: return launch_ws<FMT, 16, decoder_stages(FMT), true>(tw, tx, a, stream);
    case 32: return launch_ws<FMT, 32, ws_default_stages(FMT, 32), true>(tw, tx, a, stream);
    case 64: return launch_ws<FMT, 64, ws_default_stages(FMT, 64), true>(tw, tx, a, stream);
    case 96: return launch_ws<FMT, 96, ws_default_stages(FMT, 96), true>(tw, tx, a, stream);
    case 128: return launch_ws<FMT, 128, ws_default_stages(FMT, 128), true>(tw, tx, a, stream);
  }
  return fail("gemm_ws_launch: no whole-tile kernel instance");
}

// Token-tile width for rows_x token rows, of both weight-streaming kernels: the smallest instance covering them (a
// narrower X tile leaves more of the ring to the weight stream: 88 tokens = 8 streams x 11 take the 96-wide instance).
// fp16 takes 128 above 64 rows; bf16 and e4m3 weights (bf16 activations) take 96.  Above 128 rows: 128-wide tiles.
int token_tile(int rows_x, int fmt) {
  if (rows_x <= 16) return 16;
  if (rows_x <= 32) return 32;
  if (rows_x <= 64) return 64;
  return rows_x <= 96 && fmt != FMT_F16 ? 96 : 128;
}

// Token-tile width of the ViT trunk of 3+ frames (many token tiles): the least padding in the last token tile, and in
// mode 1 also the fullest last wave of CTAs.  Ties go to the wider tile (better operand reuse).
int trunk_token_tile(int rows, int n_out, int mode) {
  const int cands[4] = {64, 96, 128, 192};
  int best = 64;
  double best_eff = -1.0;
  for (int bn : cands) {
    const int xt = (rows + bn - 1) / bn;
    const int tiles = ((n_out + 127) / 128) * xt;
    double eff = static_cast<double>(rows) / (static_cast<double>(xt) * bn);          // padding waste
    if (mode == 1) eff *= static_cast<double>(tiles) / (((tiles + num_sms() - 1) / num_sms()) * num_sms());  // wave quantisation
    if (eff >= best_eff - 1e-9) {
      best_eff = eff;
      best = bn;
    }
  }
  return best;
}

// Stream-K decomposition of `tiles` output tiles of k / 64 k-blocks over n_ctas CTAs (<= 0: one per SM); in mode 1
// every CTA owns whole tiles.  Returns the most fp32 partial planes one tile needs.
int gemm_ws_plan(int tiles, int k, int mode, int n_ctas, SkInfo* sk) {
  const int kb = k / kGemmBK;
  sk->kb = kb;
  sk->U = static_cast<long long>(tiles) * kb;
  const long long cap = mode == 0 ? sk->U : tiles;
  int G = n_ctas > 0 ? n_ctas : num_sms();
  if (G > cap) G = static_cast<int>(cap);
  sk->G = G;
  int mp = 1;
  if (mode == 0)
    for (int t = 0; t < tiles; ++t) mp = std::max(mp, sk_planes(t, *sk));
  return mp;
}
}  // namespace

int gemm_ws_launch(const GemmWsCall& c, cudaStream_t stream, GemmWsPlan* plan) {
  VLO_CHECK(c.k > 0 && c.k % kGemmBK == 0, "K must be a positive multiple of 64");
  VLO_CHECK(c.rows_w > 0 && c.rows_x > 0, "empty GEMM operand");
  const int fmt = c.w.fmt;
  const bool beside = c.tiling == WS_TILE_BESIDE_DECODER;
  const int bn = c.bn > 0 ? c.bn
                 : beside ? 64
                 : c.tiling == WS_TILE_TRUNK ? trunk_token_tile(c.rows_x, c.rows_w, c.mode)
                 : token_tile(c.rows_x, fmt);
  VLO_CHECK(!beside || (fmt == FMT_F16 && bn == 64), "gemm_ws: only the 64-token fp16 instance fits beside a decoder CTA");
  const bool a8 = fmt == FMT_E4M3_A8;
  const bool f8 = fmt == FMT_E4M3 || a8;
  const bool i4 = fmt == FMT_I4;
  VLO_CHECK(!f8 || ((c.mode == 0 || (c.mode == 1 && !a8)) && c.tiling == WS_TILE_FIT && (c.bn == 0 || c.bn == bn)),
            "gemm_ws: e4m3 weights run stream-K partials (mode 0), or whole tiles (mode 1) on bf16 activations, on the "
            "token tile token_tile() picks");
  VLO_CHECK(!i4 || ((c.mode == 0 || c.mode == 1) && c.tiling == WS_TILE_FIT && (c.bn == 0 || c.bn == bn) && c.rows_x <= 128),
            "gemm_ws: int4 weights run stream-K partials (mode 0) or whole tiles (mode 1) of 1..128 token rows on the token "
            "tile token_tile() picks");
  VLO_CHECK(!(f8 || i4) || c.mode == 0 || (c.bias == nullptr && c.act == ACT_NONE),
            "gemm_ws: whole tiles of e4m3 or int4 weights store bf16 logits: no bias, no activation");
  VLO_CHECK(!i4 || c.k % kI4Group == 0, "gemm_ws: int4 weights need K to be a multiple of 128 (one scale per 128 k)");
  const int x_tiles = (c.rows_x + bn - 1) / bn;
  GemmWsArgs a{};
  a.rows_w = c.rows_w;
  a.rows_x = c.rows_x;
  a.k = c.k;
  a.tiles = ((c.rows_w + kGemmBM - 1) / kGemmBM) * x_tiles;
  a.x_tiles = x_tiles;
  const int planes = gemm_ws_plan(a.tiles, c.k, c.mode, c.n_ctas, &a.sk);
  if (plan) *plan = GemmWsPlan{a.sk, bn, x_tiles, planes};
  if (c.out == nullptr) return 0;
  VLO_CHECK(c.mode != 0 || static_cast<size_t>(planes) * static_cast<size_t>(c.plane_stride) <= c.out_elems,
            "stream-K workspace too small for " + std::to_string(planes) + " partial planes");
  VLO_CHECK(fmt >= FMT_F16 && fmt <= FMT_I4, "gemm_ws_launch: no kernel instance for fmt " + std::to_string(fmt));
  a.hint_w = x_tiles > 1 ? kEvictNormal : kEvictFirst;   // weights re-read by several token tiles stay in L2
  a.mode = c.mode;
  a.out = c.out;
  a.ld_out = c.ld_out;
  a.plane_stride = c.plane_stride;
  a.bias = c.bias;
  a.act = c.act;
  VLO_CHECK(!f8 || c.w.row_scale != nullptr, "gemm_ws: e4m3 weights need their row scales");
  VLO_CHECK(!a8 || c.a_scale != nullptr, "gemm_ws: e4m3 activations need their token scales");
  VLO_CHECK(!i4 || (c.w.group_scale != nullptr && (reinterpret_cast<uintptr_t>(c.w.w) & 15) == 0),
            "gemm_ws: int4 weights need their group scales and 16-byte aligned codes");
  a.wt = WsWeightArgs{c.w.row_scale, c.a_scale, static_cast<const uint8_t*>(c.w.w), c.w.group_scale};
  CUtensorMap tw, tx;
  if (!i4 && get_tmap(c.w.w, c.rows_w, c.k, kGemmBM, kWsFmtInfo[fmt].w_map, &tw) != 0) return -1;
  if (get_tmap(c.x, c.rows_x, c.k, bn, kWsFmtInfo[fmt].x_map, &tx) != 0) return -1;
  if (i4) tw = tx;   // unused: the codes stream as bulk copies
  if (c.mode == 1 && ws_tiles_own_instances(fmt))
    return fmt == FMT_I4 ? launch_ws_tiles_fmt<FMT_I4>(bn, tw, tx, a, stream) : launch_ws_tiles_fmt<FMT_E4M3>(bn, tw, tx, a, stream);
  switch (fmt) {
    case FMT_F16: return launch_ws_fmt<FMT_F16>(bn, beside, tw, tx, a, stream);
    case FMT_BF16: return launch_ws_fmt<FMT_BF16>(bn, beside, tw, tx, a, stream);
    case FMT_E4M3: return launch_ws_fmt<FMT_E4M3>(bn, beside, tw, tx, a, stream);
    case FMT_E4M3_A8: return launch_ws_fmt<FMT_E4M3_A8>(bn, beside, tw, tx, a, stream);
    default: return launch_ws_fmt<FMT_I4>(bn, beside, tw, tx, a, stream);
  }
}

// ------------------------------------------------------------------------------------------------
// ViT trunk GEMM, tokens on wgmma M (gemm_vit.cuh)

int gemm_vit_launch(const void* x, int rows_x, const void* w, int rows_w, int k, void* out, int ld_out,
                    const float* bias, int act, int n_ctas, cudaStream_t stream) {
  VLO_CHECK(k > 0 && k % kGemmBK == 0, "K must be a positive multiple of 64");
  VLO_CHECK(rows_w > 0 && rows_x > 0, "empty GEMM operand");
  VLO_CHECK(ld_out % 2 == 0 && ld_out >= rows_w, "gemm_vit: even output row stride >= rows_w (pairs of fp16 are stored)");
  GemmVitArgs a{};
  a.rows_x = rows_x;
  a.rows_w = rows_w;
  a.k = k;
  a.m_tiles = (rows_x + kGemmBM - 1) / kGemmBM;
  a.tiles = a.m_tiles * ((rows_w + kGemmBM - 1) / kGemmBM);
  a.out = static_cast<__half*>(out);
  a.ld_out = ld_out;
  a.bias = bias;
  a.act = act;
  const int G = std::min(n_ctas > 0 ? n_ctas : num_sms(), a.tiles);
  CUtensorMap tx, tw;
  if (get_tmap(x, rows_x, k, kGemmBM, FMT_F16, &tx) != 0) return -1;
  if (get_tmap(w, rows_w, k, kGemmBM, FMT_F16, &tw) != 0) return -1;
  auto kern = gemm_vit_kernel;
  if (ensure_max_smem(reinterpret_cast<const void*>(kern), GemmVitCfg::kSmemBytes)) return -1;
  if (prof_on())
    prof_begin(PROF_GEMM_VIT, stream, 2.0 * k * (static_cast<double>(rows_w) + rows_x) + 2.0 * rows_x * rows_w);
  VLO_CUDA(launch_pdl(kern, dim3(G), dim3(kVitGemmThreads), GemmVitCfg::kSmemBytes, stream, tx, tw, a));
  prof_end(stream);
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// prefill GEMMs with the chunked path's stream-K k-ranges: bf16 weights with tokens on wgmma M (gemm_prefill.cuh), the
// quantized formats with weights on wgmma M (gemm_prefill_q.cuh)

namespace {
// the quantized instances (gemm_prefill_q.cuh)
template <int FMT, int EPI>
int launch_prefill_q(const CUtensorMap& tx, const CUtensorMap& tw, const GemmPrefillQArgs& a, int G, double prof_bytes,
                     cudaStream_t stream) {
  using Cfg = GemmPrefillQCfg<FMT, EPI>;
  auto kern = gemm_prefill_q_kernel<FMT, EPI>;
  if (ensure_max_smem(reinterpret_cast<const void*>(kern), Cfg::kSmemBytes)) return -1;
  if (prof_on()) prof_begin(PROF_GEMM_STREAM, stream, prof_bytes);
  VLO_CUDA(launch_pdl(kern, dim3(G), dim3(kPrefillQThreads), Cfg::kSmemBytes, stream, tx, tw, a));
  return 0;
}
template <int FMT>
int launch_prefill_q_fmt(int epi, const CUtensorMap& tx, const CUtensorMap& tw, const GemmPrefillQArgs& a, int G,
                         double prof_bytes, cudaStream_t stream) {
  return epi == PREFILL_PLANE ? launch_prefill_q<FMT, PREFILL_PLANE>(tx, tw, a, G, prof_bytes, stream)
                              : launch_prefill_q<FMT, PREFILL_SWIGLU>(tx, tw, a, G, prof_bytes, stream);
}
}  // namespace

int gemm_prefill_launch(int epi, const WeightOperand& w, int rows_w, const void* x, int rows_x, int k, int n_ctas, void* out,
                        cudaStream_t stream, SkInfo* sk, const float* a_scale) {
  VLO_CHECK(k > 0 && k % kGemmBK == 0, "K must be a positive multiple of 64");
  VLO_CHECK(rows_w > 0 && rows_x > 0, "empty GEMM operand");
  VLO_CHECK(epi == PREFILL_PLANE || epi == PREFILL_SWIGLU, "gemm_prefill: unknown epilogue");
  VLO_CHECK(epi != PREFILL_SWIGLU || rows_w % kGemmBM == 0, "gemm_prefill: the SwiGLU epilogue needs whole 128-row tiles");
  VLO_CHECK(out != nullptr, "gemm_prefill: null output");
  const int fmt = w.fmt;
  VLO_CHECK(fmt == FMT_BF16 || fmt == FMT_E4M3 || fmt == FMT_E4M3_A8 || fmt == FMT_I4,
            "gemm_prefill: bf16, e4m3, W8A8 or int4 weights");
  VLO_CHECK(fmt != FMT_E4M3 && fmt != FMT_E4M3_A8 || w.row_scale != nullptr, "gemm_prefill: e4m3 weights need their row scales");
  VLO_CHECK(fmt != FMT_E4M3_A8 || a_scale != nullptr, "gemm_prefill: e4m3 activations need their token scales");
  VLO_CHECK(fmt != FMT_I4 || (w.group_scale != nullptr && k % kI4Group == 0 && (reinterpret_cast<uintptr_t>(w.w) & 15) == 0),
            "gemm_prefill: int4 weights need their group scales, K a multiple of 128 and 16-byte aligned codes");
  GemmPrefillArgs a{};
  a.rows_x = rows_x;
  a.rows_w = rows_w;
  a.k = k;
  a.m_tiles = (rows_x + kGemmBM - 1) / kGemmBM;
  const int w_tiles = (rows_w + kGemmBM - 1) / kGemmBM;
  a.tiles = a.m_tiles * w_tiles;
  gemm_ws_plan(w_tiles, k, 0, n_ctas, &a.sk);   // the plan of one chunk: one token tile
  if (epi == PREFILL_PLANE)
    a.plane = static_cast<float*>(out);
  else
    a.act = static_cast<__nv_bfloat16*>(out);
  if (sk) *sk = SkInfo{a.sk.U, a.sk.kb, 1};      // G = 1: every tile has one plane
  const int G = std::min(num_sms(), a.tiles);
  CUtensorMap tx, tw;
  if (get_tmap(x, rows_x, k, kGemmBM, kWsFmtInfo[fmt].x_map, &tx) != 0) return -1;
  if (fmt != FMT_I4 && get_tmap(w.w, rows_w, k, kGemmBM, kWsFmtInfo[fmt].w_map, &tw) != 0) return -1;
  if (fmt == FMT_I4) tw = tx;   // unused: the codes stream as bulk copies
  const double prof_bytes = ws_in_bytes(fmt, rows_w, rows_x, k) + (epi == PREFILL_PLANE ? 4.0 : 1.0) * rows_x * rows_w;
  if (fmt == FMT_BF16) {
    auto kern = epi == PREFILL_PLANE ? gemm_prefill_kernel<PREFILL_PLANE> : gemm_prefill_kernel<PREFILL_SWIGLU>;
    if (ensure_max_smem(reinterpret_cast<const void*>(kern), GemmPrefillCfg::kSmemBytes)) return -1;
    if (prof_on()) prof_begin(PROF_GEMM_STREAM, stream, prof_bytes);
    VLO_CUDA(launch_pdl(kern, dim3(G), dim3(kPrefillThreads), GemmPrefillCfg::kSmemBytes, stream, tx, tw, a));
  } else {
    const GemmPrefillQArgs qa{a, WsWeightArgs{w.row_scale, a_scale, static_cast<const uint8_t*>(w.w), w.group_scale}};
    const int rc = fmt == FMT_E4M3      ? launch_prefill_q_fmt<FMT_E4M3>(epi, tx, tw, qa, G, prof_bytes, stream)
                   : fmt == FMT_E4M3_A8 ? launch_prefill_q_fmt<FMT_E4M3_A8>(epi, tx, tw, qa, G, prof_bytes, stream)
                                        : launch_prefill_q_fmt<FMT_I4>(epi, tx, tw, qa, G, prof_bytes, stream);
    if (rc) return -1;
  }
  prof_end(stream);
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// stream-K gate|up GEMM with the SwiGLU finisher epilogue (gemm_wsf.cuh)
namespace {
template <int FMT, int BN>
int launch_wsf(const CUtensorMap& tw, const CUtensorMap& tx, const GemmWsfArgs& a, cudaStream_t stream) {
  constexpr int S = ws_default_stages(FMT, BN, kWsfXchBytes);
  auto kern = gemm_wsf_kernel<FMT, BN, S>;
  using Cfg = GemmWsCfg<FMT, BN, S, kWsfXchBytes>;
  if (ensure_max_smem(reinterpret_cast<const void*>(kern), Cfg::kSmemBytes)) return -1;
  if (prof_on()) prof_begin(PROF_GEMM_STREAM, stream, ws_in_bytes(FMT, a.rows_w, a.rows_x, a.k) + 2.0 * a.rows_x * a.rows_w);
  VLO_CUDA(launch_pdl(kern, dim3(a.sk.G), dim3(kGemmThreads), Cfg::kSmemBytes, stream, tw, tx, a));
  prof_end(stream);
  count_launch();
  return 0;
}

template <int FMT>
int launch_wsf_fmt(int bn, const CUtensorMap& tw, const CUtensorMap& tx, const GemmWsfArgs& a, cudaStream_t stream) {
  switch (bn) {
    case 16: return launch_wsf<FMT, 16>(tw, tx, a, stream);
    case 32: return launch_wsf<FMT, 32>(tw, tx, a, stream);
    case 64: return launch_wsf<FMT, 64>(tw, tx, a, stream);
    case 96: return launch_wsf<FMT, 96>(tw, tx, a, stream);
    default: return launch_wsf<FMT, 128>(tw, tx, a, stream);
  }
}
}  // namespace

int gemm_wsf_launch(const WeightOperand& w, int rows_w, const void* x, int rows_x, int k, void* act, float* planes,
                    size_t plane_elems, int* flags, int n_flags, cudaStream_t stream, const float* a_scale) {
  VLO_CHECK(k > 0 && k % kGemmBK == 0, "K must be a positive multiple of 64");
  VLO_CHECK(rows_w > 0 && rows_x > 0 && rows_x <= 128, "gemm_wsf: 1..128 token rows");
  VLO_CHECK(rows_w % kGemmBM == 0, "gemm_wsf: the SwiGLU epilogue needs whole 128-row tiles");
  const int fmt = w.fmt;
  VLO_CHECK(fmt >= FMT_BF16 && fmt <= FMT_I4, "gemm_wsf: bf16, e4m3 or int4 weights");
  const int bn = token_tile(rows_x, FMT_BF16);
  GemmWsfArgs a{};
  a.rows_w = rows_w;
  a.rows_x = rows_x;
  a.k = k;
  const int n_planes = gemm_ws_plan(rows_w / kGemmBM, k, 0, 0, &a.sk);
  a.plane_stride = static_cast<long long>(rows_x) * rows_w;
  VLO_CHECK(static_cast<size_t>(std::max(1, n_planes - 1)) * static_cast<size_t>(a.plane_stride) <= plane_elems,
            "gemm_wsf: stream-K workspace too small");
  VLO_CHECK(rows_w / kGemmBM <= n_flags, "gemm_wsf: stream-K flag array too small");
  a.planes = planes;
  a.flags = flags;
  a.hint_w = kEvictFirst;
  a.act = static_cast<__nv_bfloat16*>(act);
  a.I = rows_w / 2;
  VLO_CHECK(fmt != FMT_E4M3 && fmt != FMT_E4M3_A8 || w.row_scale != nullptr, "gemm_wsf: e4m3 weights need their row scales");
  VLO_CHECK(fmt != FMT_E4M3_A8 || a_scale != nullptr, "gemm_wsf: e4m3 activations need their token scales");
  VLO_CHECK(fmt != FMT_I4 || w.group_scale != nullptr, "gemm_wsf: int4 weights need their group scales");
  VLO_CHECK(fmt != FMT_I4 || k % kI4Group == 0, "gemm_wsf: int4 weights need K to be a multiple of 128 (one scale per 128 k)");
  VLO_CHECK(fmt != FMT_I4 || (reinterpret_cast<uintptr_t>(w.w) & 15) == 0, "gemm_wsf: int4 codes must be 16-byte aligned");
  a.wt = WsWeightArgs{w.row_scale, a_scale, static_cast<const uint8_t*>(w.w), w.group_scale};
  CUtensorMap tw, tx;
  if (fmt != FMT_I4 && get_tmap(w.w, rows_w, k, kGemmBM, kWsFmtInfo[fmt].w_map, &tw) != 0) return -1;
  if (get_tmap(x, rows_x, k, bn, kWsFmtInfo[fmt].x_map, &tx) != 0) return -1;
  if (fmt == FMT_I4) tw = tx;   // unused: the codes stream as bulk copies
  switch (fmt) {
    case FMT_BF16: return launch_wsf_fmt<FMT_BF16>(bn, tw, tx, a, stream);
    case FMT_E4M3: return launch_wsf_fmt<FMT_E4M3>(bn, tw, tx, a, stream);
    case FMT_E4M3_A8: return launch_wsf_fmt<FMT_E4M3_A8>(bn, tw, tx, a, stream);
    default: return launch_wsf_fmt<FMT_I4>(bn, tw, tx, a, stream);
  }
}

}  // namespace vlo
