// Host-side declarations shared by the translation units of libvlo_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#include "streamk.h"

struct vlo_letterbox_frame;  // include/vlo_b200.h
struct vlo_frame_planes;     // include/vlo_b200.h

namespace vlo {

// ---- error plumbing: every C-ABI entry returns 0 / negative and leaves a message here.
void set_error(const std::string& msg);
const char* last_error();
int fail(const std::string& msg);  // set_error + return -1

#define VLO_CUDA(expr)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess)                                                              \
      return ::vlo::fail(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" +    \
                         __FILE__ + ":" + std::to_string(__LINE__));                    \
  } while (0)

#define VLO_CHECK(cond, msg)                                                            \
  do {                                                                                  \
    if (!(cond)) return ::vlo::fail(std::string("check failed: ") + #cond + ": " + msg); \
  } while (0)

#define VLO_LAUNCH_CHECK()                                                              \
  do {                                                                                  \
    cudaError_t _e = cudaGetLastError();                                                \
    if (_e != cudaSuccess)                                                              \
      return ::vlo::fail(std::string("kernel launch: ") + cudaGetErrorString(_e) + " @" + \
                         __FILE__ + ":" + std::to_string(__LINE__));                    \
  } while (0)

// Kernel launch with the PDL attribute (see ptx.cuh: pdl_wait / pdl_trigger).  Every kernel launched through
// this helper calls pdl_wait() before its first dependent global access.  VLO_NO_PDL=1 disables the attribute.
bool pdl_enabled();
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
// Test hook (vlo_op_pdl_arm, capi_ops.cu): launch the armed probe on st and disarm it; nothing when no probe is armed.
// Entry points call it right before their first PDL launch.
int pdl_probe_fire(cudaStream_t st);

inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

int num_sms();  // multiprocessors of the current device (queried once)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device function attribute: set it once per (device, kernel).
int ensure_max_smem(const void* func, int bytes);

// Launch counter (the bench reports how many of OUR kernels ran in the timed region).
void count_launch(int n = 1);
long long launch_count();

// ---- per-kernel-class event profiler (runtime.cu); classes are indices into vlo_profile_read's arrays
enum ProfClass : int {
  PROF_GEMM_STREAM = 0,  // swap-AB weight-streaming GEMMs (decoder, connector, lm_head)
  PROF_ATTN = 1,         // attn_kvappend_kernel (the KV-append attention main kernel)
  PROF_ATTN_MERGE = 2,   // split-KV merge
  PROF_GEMM_VIT = 3,     // ViT trunk GEMMs (activations on MMA-M)
  PROF_VIT_ATTN = 4,
  PROF_OTHER = 5,
  PROF_NUM = 6,
};
void prof_enable(bool on);
bool prof_on();
void prof_begin(int cls, cudaStream_t st, double algo_bytes);
void prof_end(cudaStream_t st);
int prof_read(double* ms, long long* n, double* bytes, int ncls);

// ---- GEMM (gemm.cu) ---------------------------------------------------------------
// fp16 out[rows_a, rows_b] from activations A [rows_a, k] (MMA-M) and weights B [rows_b, k], one CTA per 128 x bn tile
struct GemmCall {
  int epi;   // GemmEpi
  int act;   // GemmAct
  const void* a;
  int rows_a;
  const void* b;
  int rows_b;
  int k;
  void* out;
  int ld_out;
  const float* bias;
  const float* pos;
  int pos_rows;
  int bn;    // 64 or 128 (0: one wave of CTAs if possible, else the less wasted last wave; gemm.cu)
};
int gemm_launch(const GemmCall& c, cudaStream_t stream);
// the bn gemm_launch picks when GemmCall::bn is 0
int vit_bn(int rows, int n_out);

// ---- persistent weight-streaming GEMM (gemm_ws.cuh / gemm.cu)
// How gemm_ws_launch picks the token-tile width when GemmWsCall::bn is 0 (the rules sit next to the instances in gemm.cu)
enum WsTiling : int {
  WS_TILE_FIT = 0,             // the smallest instance covering rows_x (one tile up to 128 rows, 128-wide tiles beyond)
  WS_TILE_TRUNK = 1,           // ViT trunk of 3+ frames: least padding, and in mode 1 the fullest last wave of CTAs
  WS_TILE_BESIDE_DECODER = 2,  // ViT trunk of 1-2 frames, fp16: 64-token tiles on a 3-stage ring (83 KB), so the CTA
                               // shares an SM with a decoder weight-streaming CTA
};
// The weight operand of the weight-streaming GEMMs: its format (GemmFmt, gemm.cuh) and what that format stores.
struct WeightOperand {
  int fmt;            // 0 fp16, 1 bf16, 2 e4m3 weights x bf16 activations, 3 e4m3 weights x e4m3 activations,
                      // 4 int4 weights x bf16 activations (3: stream-K partials only; 2, 4: also whole tiles)
  const void* w;      // [rows_w, k]: 16-bit or e4m3 elements, or fmt 4: int4 codes in the engine byte order
  const float* row_scale;       // fmt 2, 3: [rows_w] fp32 row scales, each partial is multiplied by its row's scale once
  const uint16_t* group_scale;  // fmt 4: bf16 [rows_w][k / 128] group scales
};

struct GemmWsCall {
  WeightOperand w;
  int mode;           // 0 stream-K fp32 partial planes, 1 whole tiles + 16-bit epilogue
  int rows_w;
  const void* x;      // [rows_x, k]
  int rows_x;
  int k;
  void* out;          // null: plan only
  size_t out_elems;   // mode 0: capacity of out; a plan that needs more planes is rejected before the launch
  int ld_out;
  long long plane_stride;
  const float* bias;
  int act;
  int n_ctas;         // <= 0: one CTA per SM
  int bn;             // token-tile width; 0: chosen by `tiling`
  int tiling;         // WsTiling
  const float* a_scale;  // w.fmt 3: [rows_x] fp32 token scales, each partial is then multiplied by its token's scale once
};
// What a launch decided, for the kernels that fold its partial planes.
struct GemmWsPlan {
  SkInfo sk;
  int bn;             // token-tile width
  int x_tiles;        // token tiles
  int planes;         // most fp32 partial planes one tile needs (1 in mode 1)
};
// Picks the token tile, plans the stream-K split and launches; out == null only fills *plan.
int gemm_ws_launch(const GemmWsCall& c, cudaStream_t stream, GemmWsPlan* plan = nullptr);

// ---- token-embedding gather (decoder_kernels.cuh / engine.cu): dst row i = row min(ids[i], vocab - 1) of the table
// [vocab, H] (rows with ids[i] < 0 are left alone), from a bf16 table, or dequantized from an e4m3 table (row scales:
// bf16_rn(fp32(q) * s)) or an int4 table (codes in the engine byte order, group scales: bf16_rn(q * s)).  H % 128 == 0.
int embed_rows_launch(const WeightOperand& table, const long long* ids, int n, int vocab, int H, void* dst, cudaStream_t st);

// ---- ViT trunk GEMM, 128-token x 128-feature tiles (gemm_vit.cuh / gemm.cu): fp16 x [rows_x, k], w [rows_w, k] ->
// fp16 out[rows_x][ld_out] = act(fp16(x w^T + bias)); n_ctas <= 0 -> one CTA per SM
int gemm_vit_launch(const void* x, int rows_x, const void* w, int rows_w, int k, void* out, int ld_out,
                    const float* bias, int act, int n_ctas, cudaStream_t stream);

// ---- prefill GEMMs (gemm.cu): weights w [rows_w, k] of format 1-4 by x [rows_x, k], any rows_x; bf16 weights run
// gemm_prefill_kernel (tokens on wgmma M, gemm_prefill.cuh), the others gemm_prefill_q_kernel (weights on wgmma M,
// gemm_prefill_q.cuh).  x is bf16, or e4m3 with fp32 token scales a_scale [rows_x] for format 3.  The k-ranges and plane
// order of the chunked path's stream-K plan over n_ctas CTAs (<= 0: one per SM).  epi 0: one fp32 plane
// out[rows_x][rows_w] (fill *sk with the one-plane SkInfo its fix-up kernel reads); epi 1: gate|up + SwiGLU into bf16
// out[rows_x][rows_w / 2] (rows_w % 128 == 0)
int gemm_prefill_launch(int epi, const WeightOperand& w, int rows_w, const void* x, int rows_x, int k, int n_ctas, void* out,
                        cudaStream_t stream, SkInfo* sk = nullptr, const float* a_scale = nullptr);

// ---- stream-K gate|up GEMM with the fused SwiGLU finisher (gemm_wsf.cuh / gemm.cu), one CTA per SM:
// act[rows_x][rows_w / 2] = SwiGLU(x w^T) for weights w of format 1-4; x is bf16, or e4m3 with fp32 token scales
// a_scale [rows_x] for format 3.  planes (plane_elems floats) take the partials of the non-finisher CTAs, flags (n_flags
// counters, zero between launches) their arrivals.
int gemm_wsf_launch(const WeightOperand& w, int rows_w, const void* x, int rows_x, int k, void* act, float* planes,
                    size_t plane_elems, int* flags, int n_flags, cudaStream_t stream, const float* a_scale = nullptr);

// ---- decoder fix-up and decision kernels (decoder_kernels.cuh / engine.cu) -----------
// bf16 tensors; `part` holds fp32 stream-K planes [plane][T][width] of the plan `sk`, as gemm_ws_launch mode 0 leaves
// them with plane_stride T * width (null: no partials, resid_rmsnorm only).
// resid_rmsnorm_kernel: h[T, H] += fix-up, xn[T, H] (may be null) = RMSNorm(h) * w, xn_last[last_index[t]] = xn[t] for
// last_index[t] >= 0 (both may be null); one CTA per row of min(1024, max(32, H / 4)) threads.
int resid_rmsnorm_launch(const float* part, const SkInfo* sk, void* h, const void* w, void* xn, void* xn_last,
                         const int* last_index, int T, int H, float eps, cudaStream_t st);
// resid_rmsnorm_q8_kernel: resid_rmsnorm_kernel that also writes the e4m3 row xq[t] of xn[t] and its fp32 scale xs[t]
// (the per-token rule of quant_rows_e4m3_kernel); xn is the same as without.
int resid_rmsnorm_q8_launch(const float* part, const SkInfo* sk, void* h, const void* w, void* xn, void* xn_last,
                            const int* last_index, uint8_t* xq, float* xs, int T, int H, float eps, cudaStream_t st);
// quant_rows_e4m3_kernel: bf16 x[T, K] (K % 8 == 0) -> e4m3 q[T, K] and fp32 token scales s[T], one CTA per row.
int quant_rows_launch(const void* x, int T, int K, uint8_t* q, float* s, cudaStream_t st);
// qkv_rope_append_kernel: q[T, n_heads, 128] and K / V rows of the token's position (device tables tok_pos / tok_kvrow)
// from the fix-up of the q|k|v planes, RoPE from the bf16 [pos][64] cos / sin tables.
int qkv_rope_launch(const float* part, const SkInfo& sk, const void* cos_tab, const void* sin_tab, const int* tok_pos,
                    const long long* tok_kvrow, int kv_head_stride, void* q, void* k_cache, void* v_cache, int T,
                    int n_heads, int n_kv_heads, cudaStream_t st);
// decision_kernel: one vlo_decision per bf16 logits row [n_rows, vocab].
int decision_launch(const void* logits, int n_rows, int vocab, int interval_id, void* out, cudaStream_t st);

// ---- response sampling (sampling.cuh / engine.cu) -------------------------------------
// The parameters of n rows of a vlo_sample / vlo_op_sample call (vlo_sample_row, include/vlo_b200.h) over n_ids penalty
// ids: 0 when every row is valid, else -1 with the message set.
int sample_check_rows(const void* h_rows, int n_rows, int n_ids);
// sample_kernel: one id per bf16 logits row [n_rows, vocab] (vocab % 8 == 0, 16-byte aligned rows); rows / penalty_ids /
// info are device arrays (info may be null).
int sample_launch(const void* logits, int n_rows, int vocab, const void* rows, const int* penalty_ids, int* out_ids,
                  void* info, cudaStream_t st);

// ---- ViT attention kernels (vit_kernels.cuh / engine.cu) ------------------------------
// vit_attn_kernel: non-causal attention of each of B frames of N tokens over its own tokens, head_dim 64, C / 64 heads;
// qkv fp16 [B * N, 3C] (q | k | v column blocks) -> out fp16 [B * N, C].
int vit_attn_launch(const void* qkv, void* out, int B, int N, int C, cudaStream_t st);
// probe_attn_kernel: the MAP head's one fp32 query q [C] over the N tokens of each frame, kv fp16 [B * N, 2C] (k | v)
// -> out fp16 [B, C].
int probe_attn_launch(const void* kv, const float* q, void* out, int B, int N, int C, cudaStream_t st);

// ---- the other ViT kernels (vit_kernels.cuh / engine.cu), fp16 / fp32 as vlo_vit_encode holds them -------------
// B frames run their trunk GEMMs beside a decoder step (gemm_vit_kernel, WS_TILE_BESIDE_DECODER) rather than on the
// WS_TILE_TRUNK tiling
bool vit_beside_decoder(int B);
// patchify_kernel: u8 frames [B, 3, S, S] -> fp16 patches [B * (S / ps)^2, 3 ps ps]; ps % 8 == 0
int patchify_launch(const uint8_t* frames, void* out, int B, int S, int ps, cudaStream_t st);
// layernorm_kernel: in [rows, C] (fp16 if in_f16, else fp32) -> out16 fp16 and / or out32 fp32 (either may be null)
int vit_layernorm_launch(const void* in, bool in_f16, int rows, int C, const float* w, const float* b, void* out16,
                         float* out32, float eps, cudaStream_t st);
// vit_fix_ln_kernel: the stream-K planes `part` [plane][rows][C] of the fp16 GEMM that made `plan` folded with bias into
// the fp32 residual h [rows, C], then LayerNorm(h) -> out16 (and out32 if not null); C % 4 == 0
int vit_fix_ln_launch(const float* part, const GemmWsPlan& plan, int rows, int C, const float* bias, float* h,
                      const float* ln_w, const float* ln_b, void* out16, float* out32, float eps, cudaStream_t st);
// pool_kernel: adaptive average pool of each frame's g x g grid of in [B, g * g, C] to ph x pw cells, cell j of frame b
// -> tokens[b * n_tok + tok_off + j]
int pool_launch(const float* in, float* tokens, int B, int g, int C, int ph, int pw, int n_tok, int tok_off,
                cudaStream_t st);
// cls_residual_kernel: tokens[b * n_tok] = fp16(resid[b] + mlp[b]), fp16 [B, C] inputs
int cls_residual_launch(const void* resid, const void* mlp, float* tokens, int B, int C, int n_tok, cudaStream_t st);
// f32_to_bf16_kernel: out[i] = bf16(in[i]), i < n
int f32_to_bf16_launch(const float* in, void* out, long long n, cudaStream_t st);

// ---- letterbox (letterbox.cu) ---------------------------------------------------------
// letterbox_kernel: the frames of vlo_letterbox_planes (include/vlo_b200.h) -> uint8 out [n, 3, R, R]; checks each
// descriptor, then one launch per kLetterboxMaxFrames frames (their descriptors travel as kernel parameters, 4 KB)
constexpr int kLetterboxMaxFrames = 48;
int letterbox_planes_launch(const vlo_frame_planes* frames, int n, int R, uint8_t* out, cudaStream_t st);
// vlo_letterbox's packed frames: checks bgr, then letterbox_planes_launch of RGB24 / BGR24 descriptors
int letterbox_launch(const vlo_letterbox_frame* frames, int n, int R, uint8_t* out, cudaStream_t st);

// ---- attention (attn.cu) ------------------------------------------------------------
struct AttnSeq {
  int q_tok0;          // first packed token of the sequence
  int q_len;           // new tokens
  int kv_len;          // cache length INCLUDING the new tokens
  int pt0;             // entry of the page table holding the page of key block 0 (ceil(kv_len / 64) entries follow)
  // > 1: the q_len rows are n_segs consecutive segments of seg_lens[j] rows (host array), each planned exactly as a
  // one-sequence step of that segment alone over the keys up to its end (attn_plan); 0 or 1: one segment
  int n_segs;
  const int* seg_lens;
};
// bytes of scratch attn_launch needs for these sequences (upper bound)
size_t attn_ws_bytes(int total_tokens, int n_seqs, int n_heads, int n_kv_heads);
size_t attn_stage_bytes(int total_tokens, int n_seqs, int n_heads, int n_kv_heads);
struct AttnPlan {
  float* ws_o;
  float* ws_ml;
  void* d_items;
  int* d_tok_item;
  int n_items, max_splits, total_tokens;
  int max_blocks_per_split;  // sizes the page-table staging of the launch
  int blk;            // keys per pipeline block
  // Items [n_plain, n_items) belong to clusters (attn_kvappend_cluster_kernel): n_clusters tables of cluster_size
  // members at d_clusters, max_cluster_splits splits.  n_plain == n_items when no segmented sequence has two items of
  // the same split grid.
  int n_plain, n_clusters, cluster_size, max_cluster_splits;
  void* d_clusters;
  // The last n_packed_items items belong to n_packs runs of one-token segments (attn_kvappend_packed_kernel, tables at
  // d_packs, max_pack_splits splits); 0 when no sequence has two consecutive one-token segments of one split grid.
  int n_packs, n_packed_items, max_pack_splits;
  void* d_packs;
  int skip_merge;     // measurement only: launch the main kernel without the split-KV merge
  double algo_bytes;  // algorithmic HBM bytes of one attn_run over this plan (K+V rows read, Q read, out written)
};
// Build the work-item plan on the host and enqueue its upload.  h_stage (>= attn_stage_bytes())
// must stay untouched until the copies enqueued on `stream` have run.  d_ws == null: plan only (the counts of *plan),
// nothing staged or uploaded.
int attn_plan(AttnPlan* plan, void* d_ws, void* h_stage, const AttnSeq* seqs, int n_seqs, int total_tokens,
              int n_heads, int n_kv_heads, int head_dim, cudaStream_t stream);
// d_k / d_v: one layer's K / V matrices [kv_rows, 128] bf16; key block b of kv head h of a sequence sits at row
// d_page_table[pt0 + b] * page_stride_rows + h * head_stride_rows (attn.cuh); d_q [T, n_heads, 128]; d_out [T, n_heads*128].
int attn_run(const AttnPlan& plan, const void* d_q, const void* d_k, const void* d_v, long long kv_rows,
             const int* d_page_table, long long page_stride_rows, long long head_stride_rows, void* d_out, int n_heads,
             int n_kv_heads, int head_dim, cudaStream_t stream);

// longest sequence, in 64-key blocks, whose page table one attention CTA can stage (any plan of it then succeeds)
int attn_max_key_blocks();

// 2D TMA map over a row-major 16-bit matrix [rows, k], box 64 x box_rows, 128-byte swizzle (cached).
int tmap_2d_sw128(const void* ptr, int rows, int k, int box_rows, int fmt, CUtensorMap* out);

}  // namespace vlo
