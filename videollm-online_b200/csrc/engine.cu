// vlo_engine: weights registry, KV-cache ownership, workspaces and the orchestration of the
// per-frame hot path (vlo_vit_encode, vlo_step) on one GPU.  See include/vlo_b200.h for the ABI
// and DESIGN.md for the memory layout.
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "common.h"
#include "decoder_kernels.cuh"
#include "gemm.cuh"
#include "kv_pages.h"
#include "sampling.cuh"
#include "vit_kernels.cuh"
#include "vlo_b200.h"

using namespace vlo;

static_assert(sizeof(vlo_sample_row) == sizeof(SampleRow), "vlo_sample_row and SampleRow must match");

namespace {

constexpr int kStageSlots = 16;
constexpr int kSamplePenaltyIds = 65536;  // penalty ids one vlo_sample call may pass
constexpr int kSkFlags = 4096;  // stream-K arrival counters of the fused gate|up GEMM: one per 128-row weight tile
constexpr int kRotFloats = 128;  // vlo_kv_evict's cos | sin (head_dim / 2 each), staged ahead of the stream's table

using bf16 = __nv_bfloat16;

struct DecLayer {
  const bf16 *in_norm, *post_norm;
  WeightOperand qkv, o, gate_up, down;   // the layer matrices, all of the engine's layer_fmt
};
struct VitLayer {
  const float *ln1_w, *ln1_b, *ln2_w, *ln2_b, *qkv_b, *out_b, *fc1_b, *fc2_b;
  const __half *qkv_w, *out_w, *fc1_w, *fc2_w;
};

}  // namespace

struct vlo_engine {
  vlo_config cfg{};
  int device = 0;
  std::map<std::string, std::pair<const void*, int64_t>> tensors;
  bool finalized = false;

  // resolved weights
  std::vector<DecLayer> dec;
  // the vocabulary matrices [vocab, hidden]: bf16, or both in the layer matrices' quantized form (vocab_fmt)
  WeightOperand embed{}, lm_head{};
  const bf16 *final_norm = nullptr, *rope_cos = nullptr, *rope_sin = nullptr;
  int64_t rope_positions = 0;
  std::vector<VitLayer> vit;
  const __half *patch_w = nullptr, *head_kv_w = nullptr, *head_out_w = nullptr, *head_fc1_w = nullptr,
               *head_fc2_w = nullptr;
  const float *patch_b = nullptr, *pos_emb = nullptr, *post_ln_w = nullptr, *post_ln_b = nullptr, *head_q = nullptr,
              *head_kv_b = nullptr, *head_out_b = nullptr, *head_ln_w = nullptr, *head_ln_b = nullptr,
              *head_fc1_b = nullptr, *head_fc2_b = nullptr, *conn0_b = nullptr, *conn2_b = nullptr;
  const bf16 *conn0_w = nullptr, *conn2_w = nullptr;
  bool has_vit = false, has_connector = false, has_decoder = false;
  int layer_fmt = FMT_BF16;  // GemmFmt of the layer matrices (vlo_finalize_weights; FMT_E4M3_A8 with fp8_act)
  int vocab_fmt = FMT_BF16;  // GemmFmt of embed and lm_head (vlo_finalize_weights): FMT_BF16, FMT_E4M3 or FMT_I4
  bool fp8_act = false;      // vlo_set_fp8_activations: the layer GEMMs take e4m3 activations with token scales
  bool quant_prefill = false;  // vlo_set_quantized_prefill: quantized layer matrices prefill too

  // derived
  int qkv_width = 0, grid = 0, n_patches = 0, n_frame_tokens = 0, patch_k = 0;

  // device allocations owned by the engine
  std::vector<void*> allocs;
  int64_t device_bytes = 0;
  bf16* kv = nullptr;  // [layer][2][page][kv_head][64][128], pages owned through `pool`
  KvPool pool;              // every stream slot's cache state
  // device page tables of the KV copy / fill calls (two streams' worth), or an eviction's cos | sin then its table
  int* kv_op_pt = nullptr;
  size_t max_pitch = 0;  // cudaDevAttrMaxPitch: the plane stride of a swap's 2D copies must not exceed it

  // decoder workspaces
  bf16 *h = nullptr, *xn = nullptr, *xn_last = nullptr, *q = nullptr, *attn_out = nullptr, *act = nullptr,
       *logits = nullptr;
  float* part = nullptr;
  size_t part_elems = 0;
  // fp8_act only: e4m3 copies of xn, attn_out and act with their fp32 token scales, act_rows rows
  int act_rows = 0;
  uint8_t *xq = nullptr, *aq = nullptr, *actq = nullptr;
  float *xs = nullptr, *as = nullptr, *acts = nullptr;
  int* sk_flags = nullptr;          // kSkFlags counters, zero between launches
  uint8_t* attn_ws = nullptr;
  uint8_t* meta_dev = nullptr;  // the step's tables, laid out as `meta` says
  // Byte offsets of tok_pos | last_index | first_rows | tok_kvrow | page tables in meta_dev and in a staging slot, whose
  // attention plan starts at `bytes` (set by engine_init).
  struct {
    size_t pos, last, first, kvrow, pt, bytes;
  } meta{};
  DecisionOut* decisions = nullptr;
  // vlo_sample parameters: sample_rows rows, then (at sample_ids) up to kSamplePenaltyIds penalty ids; the same layout
  // sits at byte sample_stage of every staging slot
  uint8_t* sample_dev = nullptr;
  int sample_rows = 0;
  size_t sample_ids = 0, sample_stage = 0;
  // host staging ring (pinned)
  uint8_t* stage = nullptr;
  size_t stage_slot_bytes = 0;
  cudaEvent_t stage_events[kStageSlots]{};
  bool stage_used[kStageSlots]{};
  int stage_next = 0;
  int last_step_tokens = 0;
  int token_rows = 0;    // rows the token-row workspaces hold (size_token_rows)
  // rows of one vlo_prefill: kFixMaxPlanes x max_step_tokens (one fp32 plane fits `part`) once vlo_finalize_weights has
  // grown the token-row workspaces of a bf16 engine, or of a quantized one with quant_prefill; 0 before, and on
  // quantized engines without quant_prefill
  int max_prefill = 0;

  // ViT workspaces
  __half *patches = nullptr, *v_xn = nullptr, *v_qkv = nullptr, *v_attn = nullptr, *v_mlp = nullptr, *v_pa = nullptr,
         *v_resid = nullptr, *v_lnh = nullptr, *v_m1 = nullptr, *v_m2 = nullptr;
  float *v_h = nullptr, *v_ln32 = nullptr, *tokens32 = nullptr, *v_part = nullptr;
  size_t v_part_elems = 0;
  bf16 *tokens16 = nullptr, *conn_mid = nullptr;
};

namespace vlo {
int embed_rows_launch(const WeightOperand& table, const long long* ids, int n, int vocab, int H, void* dst, cudaStream_t st) {
  bf16* out = static_cast<bf16*>(dst);
  if (table.fmt == FMT_BF16)
    embed_rows_kernel<<<n, 256, 0, st>>>(ids, nullptr, n, static_cast<const bf16*>(table.w), vocab, H, out);
  else if (table.fmt == FMT_E4M3)
    embed_rows_q_kernel<false><<<n, 256, 0, st>>>(ids, nullptr, n, static_cast<const uint8_t*>(table.w), table.row_scale,
                                                  vocab, H, out);
  else if (table.fmt == FMT_I4)
    embed_rows_q_kernel<true><<<n, 256, 0, st>>>(ids, nullptr, n, static_cast<const uint8_t*>(table.w), table.group_scale,
                                                 vocab, H, out);
  else
    return fail("embed_rows: no gather for weight format " + std::to_string(table.fmt));
  VLO_LAUNCH_CHECK();
  count_launch();
  return 0;
}
}  // namespace vlo

namespace {

int dev_alloc(vlo_engine* e, void** p, size_t bytes, bool zero) {
  bytes = align256(bytes ? bytes : 256);
  VLO_CUDA(cudaMalloc(p, bytes));
  if (zero) VLO_CUDA(cudaMemset(*p, 0, bytes));
  e->allocs.push_back(*p);
  e->device_bytes += static_cast<int64_t>(bytes);
  return 0;
}
template <typename T>
int dev_alloc_t(vlo_engine* e, T** p, size_t n, bool zero = false) {
  return dev_alloc(e, reinterpret_cast<void**>(p), n * sizeof(T), zero);
}
// gives back an allocation of dev_alloc (bytes as passed to it)
template <typename T>
void dev_free(vlo_engine* e, T** p, size_t bytes) {
  if (*p == nullptr) return;
  for (size_t i = 0; i < e->allocs.size(); ++i)
    if (e->allocs[i] == *p) {
      e->allocs.erase(e->allocs.begin() + static_cast<long>(i));
      cudaFree(*p);
      e->device_bytes -= static_cast<int64_t>(align256(bytes ? bytes : 256));
      break;
    }
  *p = nullptr;
}

// The workspaces whose size follows the rows of one pass: h, xn, q, attn_out, act, the attention workspace, the step
// tables (and with them the layout of every pinned staging slot).  `rows` = max_step_tokens at creation; a prefilling
// engine grows them to max_prefill rows in vlo_finalize_weights.  Growing frees the old buffers: no work may be in flight.
int size_token_rows(vlo_engine* e, int rows) {
  const vlo_config& c = e->cfg;
  const size_t H = c.hidden_size, A = static_cast<size_t>(c.num_heads) * c.head_dim, I = c.intermediate_size;
  const int per_stream = kv_pages_for(c.max_kv_tokens);
  const size_t per_token = align256(sizeof(int) * rows);
  const size_t meta_bytes = 3 * per_token + align256(sizeof(long long) * rows) +
                            align256(sizeof(int) * std::max(2, c.max_streams) * per_stream);
  const size_t sample_bytes = e->sample_ids + sizeof(int) * kSamplePenaltyIds;
  if (e->h != nullptr) {
    const size_t old = e->token_rows;
    dev_free(e, &e->h, old * H * sizeof(bf16));
    dev_free(e, &e->xn, old * H * sizeof(bf16));
    dev_free(e, &e->q, old * A * sizeof(bf16));
    dev_free(e, &e->attn_out, old * A * sizeof(bf16));
    dev_free(e, &e->act, old * I * sizeof(bf16));
    dev_free(e, &e->attn_ws, attn_ws_bytes(e->token_rows, c.max_streams, c.num_heads, c.num_kv_heads));
    dev_free(e, &e->meta_dev, e->meta.bytes);
    VLO_CUDA(cudaFreeHost(e->stage));
    e->stage = nullptr;
    for (int i = 0; i < kStageSlots; ++i) e->stage_used[i] = false;
  }
  e->token_rows = rows;
  if (dev_alloc_t(e, &e->h, rows * H)) return -1;
  if (dev_alloc_t(e, &e->xn, rows * H)) return -1;
  if (dev_alloc_t(e, &e->q, rows * A)) return -1;
  if (dev_alloc_t(e, &e->attn_out, rows * A)) return -1;
  if (dev_alloc_t(e, &e->act, rows * I)) return -1;
  const size_t aws = attn_ws_bytes(rows, c.max_streams, c.num_heads, c.num_kv_heads);
  if (dev_alloc(e, reinterpret_cast<void**>(&e->attn_ws), aws, false)) return -1;
  // the table region also stages the two streams' tables of a KV copy (upload_op_tables)
  e->meta.pos = 0;
  e->meta.last = per_token;
  e->meta.first = 2 * per_token;
  e->meta.kvrow = 3 * per_token;
  e->meta.pt = e->meta.kvrow + align256(sizeof(long long) * rows);
  e->meta.bytes = meta_bytes;
  if (dev_alloc(e, reinterpret_cast<void**>(&e->meta_dev), e->meta.bytes, false)) return -1;
  e->sample_stage = align256(e->meta.bytes + attn_stage_bytes(rows, c.max_streams, c.num_heads, c.num_kv_heads));
  e->stage_slot_bytes = align256(e->sample_stage + sample_bytes);
  VLO_CUDA(cudaMallocHost(reinterpret_cast<void**>(&e->stage), e->stage_slot_bytes * kStageSlots));
  return 0;
}

template <typename T>
int lookup(vlo_engine* e, const std::string& name, int64_t expect_elems, const T** out) {
  auto it = e->tensors.find(name);
  if (it == e->tensors.end()) return fail("missing weight tensor '" + name + "'");
  if (expect_elems > 0 && it->second.second != expect_elems * static_cast<int64_t>(sizeof(T)))
    return fail("weight tensor '" + name + "' has " + std::to_string(it->second.second) + " bytes, expected " +
                std::to_string(expect_elems * static_cast<int64_t>(sizeof(T))));
  *out = static_cast<const T*>(it->second.first);
  return 0;
}

// weights [n_out, k] x tokens [rows, k] -> stream-K fp32 partial planes part[plane][rows][n_out] (persistent kernel),
// which a fix-up kernel folds.  x_scale: the token scales of e4m3 activations (w.fmt FMT_E4M3_A8).  The fix-up kernels
// unroll kFixMaxPlanes planes: this is the one check of that limit, made before the fix-up kernel that would read the
// planes is launched.
int gemm_partial(const WeightOperand& w, int n_out, const void* x, const float* x_scale, int rows, int k, float* part,
                 size_t part_elems, int tiling, GemmWsPlan* plan, cudaStream_t st) {
  GemmWsCall c{};
  c.w = w;
  c.a_scale = x_scale;
  c.mode = 0;
  c.rows_w = n_out;
  c.x = x;
  c.rows_x = rows;
  c.k = k;
  c.out = part;
  c.out_elems = part_elems;
  c.ld_out = n_out;
  c.plane_stride = static_cast<long long>(rows) * n_out;
  c.tiling = tiling;
  if (gemm_ws_launch(c, st, plan)) return -1;
  VLO_CHECK(plan->planes <= kFixMaxPlanes, "stream-K produced more partial planes than the fix-up kernels unroll");
  return 0;
}

// gate|up GEMM + SwiGLU: the stream-K finisher CTAs apply the fix-up themselves (gemm_wsf.cuh).  A finisher's epilogue
// (flag acquire -> plane loads -> stores) is a tail at the end of EVERY CTA during which its SM streams nothing, while a
// separate fix-up kernel runs next to the next GEMM's CTA, whose ring is already filling.  Only the gate|up GEMM has
// enough tiles (224, 1.7 per CTA on 132 SMs) to amortise that tail, and fusing it removes the 3.6 MB plane round trip of
// its fix-up; q|k|v, o_proj and down_proj go through gemm_partial and a fix-up kernel (DESIGN.md section 5).
int gemm_swiglu(vlo_engine* e, const WeightOperand& w, int n_out, const void* x, int T, int k, cudaStream_t st,
                const float* x_scale = nullptr) {
  return gemm_wsf_launch(w, n_out, x, T, k, e->act, e->part, e->part_elems, e->sk_flags, kSkFlags, st, x_scale);
}

// whole-tile persistent GEMM with the 16-bit epilogue: out[T, n_out] = act(x W^T + bias)
int gemm_ws_store16(int fmt, const void* w, int n_out, const void* x, int T, int k, void* out, int ld, const float* bias,
                    int act, cudaStream_t st, int tiling = WS_TILE_FIT) {
  GemmWsCall c{};
  c.w = WeightOperand{fmt, w, nullptr, nullptr};
  c.mode = 1;
  c.rows_w = n_out;
  c.x = x;
  c.rows_x = T;
  c.k = k;
  c.out = out;
  c.ld_out = ld;
  c.bias = bias;
  c.act = act;
  c.tiling = tiling;
  return gemm_ws_launch(c, st);
}

// logits [rows, vocab] bf16 = x [rows, hidden] lm_head^T, whole tiles (each row independent of the others).  bf16:
// one launch.  e4m3 / int4: the format's whole-tile instances, in pieces of at most 128 rows (one token tile of int4).
int lm_head_launch(vlo_engine* e, const void* x, int rows, void* out, cudaStream_t st) {
  const vlo_config& c = e->cfg;
  if (e->lm_head.fmt == FMT_BF16)
    return gemm_ws_store16(FMT_BF16, e->lm_head.w, c.vocab_size, x, rows, c.hidden_size, out, c.vocab_size, nullptr,
                           ACT_NONE, st);
  for (int r0 = 0; r0 < rows; r0 += kGemmBM) {
    GemmWsCall g{};
    g.w = e->lm_head;
    g.mode = 1;
    g.rows_w = c.vocab_size;
    g.x = static_cast<const bf16*>(x) + static_cast<size_t>(r0) * c.hidden_size;
    g.rows_x = std::min(kGemmBM, rows - r0);
    g.k = c.hidden_size;
    g.out = static_cast<bf16*>(out) + static_cast<size_t>(r0) * c.vocab_size;
    g.ld_out = c.vocab_size;
    if (gemm_ws_launch(g, st)) return -1;
  }
  return 0;
}

// one-tile fp16 GEMM with the 16-bit epilogue: out[rows_a, rows_b] = act(a b^T + bias)
int gemm_store16(const void* a, int rows_a, const void* b, int rows_b, int k, void* out, int ld, const float* bias, int act,
                 cudaStream_t st) {
  GemmCall c{};
  c.epi = EPI_STORE16;
  c.act = act;
  c.a = a;
  c.rows_a = rows_a;
  c.b = b;
  c.rows_b = rows_b;
  c.k = k;
  c.out = out;
  c.ld_out = ld;
  c.bias = bias;
  return gemm_launch(c, st);
}

// pinned staging slot, recycled behind a CUDA event
int stage_acquire(vlo_engine* e, uint8_t** out, int* slot) {
  const int s = e->stage_next;
  e->stage_next = (s + 1) % kStageSlots;
  if (e->stage_used[s]) VLO_CUDA(cudaEventSynchronize(e->stage_events[s]));
  *out = e->stage + static_cast<size_t>(s) * e->stage_slot_bytes;
  *slot = s;
  return 0;
}
int stage_release(vlo_engine* e, int slot, cudaStream_t st) {
  VLO_CUDA(cudaEventRecord(e->stage_events[slot], st));
  e->stage_used[slot] = true;
  return 0;
}

// Pack the page tables of streams sids[0..n) back to back into the table region of staging slot hs; pt0[i] receives
// the entry of stream i's first page.  Returns the entries written.
int stage_page_tables(const vlo_engine* e, uint8_t* hs, int n, const int* sids, int* pt0) {
  int* dst = reinterpret_cast<int*>(hs + e->meta.pt);
  int used = 0;
  for (int i = 0; i < n; ++i) {
    const std::vector<int>& tab = e->pool.table(sids[i]);
    std::memcpy(dst + used, tab.data(), sizeof(int) * tab.size());
    pt0[i] = used;
    used += static_cast<int>(tab.size());
  }
  return used;
}

// elements of one layer's K or V matrix
inline size_t kv_plane_elems(const vlo_engine* e) { return static_cast<size_t>(e->pool.rows_per_layer()) * e->cfg.head_dim; }
inline bf16* kv_layer_base(vlo_engine* e, int layer, int is_v) {
  return e->kv + (static_cast<size_t>(layer) * 2 + is_v) * kv_plane_elems(e);
}
// the paged side of a KV copy / fill: table of stream `sid` uploaded to d_pt
inline KvSide kv_paged_side(vlo_engine* e, bf16* plane0, const int* d_pt) {
  return KvSide{plane0, d_pt, static_cast<long long>(kv_plane_elems(e)), 0};
}

// Upload the page tables of n <= 2 streams to e->kv_op_pt through a staging slot; d_pt[i] = stream i's table.
int upload_op_tables(vlo_engine* e, int n, const int* sids, const int** d_pt, cudaStream_t st) {
  uint8_t* hs;
  int slot;
  if (stage_acquire(e, &hs, &slot)) return -1;
  int pt0[2];
  const int used = stage_page_tables(e, hs, n, sids, pt0);
  for (int i = 0; i < n; ++i) d_pt[i] = e->kv_op_pt + pt0[i];
  VLO_CUDA(cudaMemcpyAsync(e->kv_op_pt, hs + e->meta.pt, sizeof(int) * used, cudaMemcpyHostToDevice, st));
  return stage_release(e, slot, st);
}

// attention of decoder layer l over the KV pool, e->q -> e->attn_out, through the page tables staged in meta_dev
int attn_layer(vlo_engine* e, const AttnPlan& plan, int l, cudaStream_t st) {
  const vlo_config& c = e->cfg;
  return attn_run(plan, e->q, kv_layer_base(e, l, 0), kv_layer_base(e, l, 1), e->pool.rows_per_layer(),
                  reinterpret_cast<const int*>(e->meta_dev + e->meta.pt), e->pool.page_stride_rows(),
                  KvPool::head_stride_rows(), e->attn_out, c.num_heads, c.num_kv_heads, c.head_dim, st);
}

// Every entry point that touches the device runs on the engine's GPU whatever the caller's current device is
// (one process may own engines on several GPUs); the previous device is restored on return.
struct DevGuard {
  int prev = -1;
  bool switched = false;
  explicit DevGuard(const vlo_engine* e) {
    if (e == nullptr) return;
    if (cudaGetDevice(&prev) == cudaSuccess && prev != e->device) switched = cudaSetDevice(e->device) == cudaSuccess;
  }
  ~DevGuard() {
    if (switched) cudaSetDevice(prev);
  }
};

int check_stream(vlo_engine* e, int sid) {
  if (e == nullptr) return fail("null engine");
  if (sid < 0 || sid >= e->cfg.max_streams || !e->pool.is_open(sid)) return fail("invalid stream id " + std::to_string(sid));
  return 0;
}

// bytes of one page in one layer's K or V matrix
inline size_t kv_page_bytes(const vlo_engine* e) {
  return static_cast<size_t>(e->pool.page_stride_rows()) * e->cfg.head_dim * sizeof(bf16);
}

}  // namespace

// ------------------------------------------------------------------------------ decoder fix-up and decision launches
// The step and the kernel-level entry points (capi_ops.cu) launch these kernels through the helpers below only.
namespace vlo {

int resid_rmsnorm_launch(const float* part, const SkInfo* sk, void* h, const void* w, void* xn, void* xn_last,
                         const int* last_index, int T, int H, float eps, cudaStream_t st) {
  ResidNormParams p{};
  p.part = part;
  if (part) p.sk = *sk;
  p.split_stride = static_cast<long long>(T) * H;
  p.h = static_cast<bf16*>(h);
  p.w = static_cast<const bf16*>(w);
  p.xn = static_cast<bf16*>(xn);
  p.xn_last = static_cast<bf16*>(xn_last);
  p.last_index = last_index;
  p.H = H;
  p.eps = eps;
  VLO_CUDA(launch_pdl(resid_rmsnorm_kernel, dim3(T), dim3(std::min(1024, std::max(32, H / 4))),
                      static_cast<size_t>(H) * sizeof(float), st, p));
  count_launch();
  return 0;
}

int resid_rmsnorm_q8_launch(const float* part, const SkInfo* sk, void* h, const void* w, void* xn, void* xn_last,
                            const int* last_index, uint8_t* xq, float* xs, int T, int H, float eps, cudaStream_t st) {
  ResidNormParams p{};
  p.part = part;
  if (part) p.sk = *sk;
  p.split_stride = static_cast<long long>(T) * H;
  p.h = static_cast<bf16*>(h);
  p.w = static_cast<const bf16*>(w);
  p.xn = static_cast<bf16*>(xn);
  p.xn_last = static_cast<bf16*>(xn_last);
  p.last_index = last_index;
  p.H = H;
  p.eps = eps;
  prof_begin(PROF_OTHER, st, 2.0 * T * H * (part ? 3.0 : 2.0) + 1.0 * T * H);
  VLO_CUDA(launch_pdl(resid_rmsnorm_q8_kernel, dim3(T), dim3(std::min(1024, std::max(32, H / 4))),
                      static_cast<size_t>(H) * sizeof(float), st, p, xq, xs));
  prof_end(st);
  count_launch();
  return 0;
}

int quant_rows_launch(const void* x, int T, int K, uint8_t* q, float* s, cudaStream_t st) {
  VLO_CHECK(T > 0 && K > 0 && K % 8 == 0, "quant_rows: T > 0 and K a positive multiple of 8");
  prof_begin(PROF_OTHER, st, 3.0 * T * K + 4.0 * T);
  VLO_CUDA(launch_pdl(quant_rows_e4m3_kernel, dim3(T), dim3(256), 0, st, static_cast<const bf16*>(x), K, q, s));
  prof_end(st);
  count_launch();
  return 0;
}

int qkv_rope_launch(const float* part, const SkInfo& sk, const void* cos_tab, const void* sin_tab, const int* tok_pos,
                    const long long* tok_kvrow, int kv_head_stride, void* q, void* k_cache, void* v_cache, int T,
                    int n_heads, int n_kv_heads, cudaStream_t st) {
  QkvRopeParams p{};
  p.part = part;
  p.sk = sk;
  p.split_stride = static_cast<long long>(T) * (n_heads + 2 * n_kv_heads) * 128;
  p.cos_tab = static_cast<const bf16*>(cos_tab);
  p.sin_tab = static_cast<const bf16*>(sin_tab);
  p.tok_pos = tok_pos;
  p.tok_kvrow = tok_kvrow;
  p.kv_head_stride = kv_head_stride;
  p.q_out = static_cast<bf16*>(q);
  p.k_cache = static_cast<bf16*>(k_cache);
  p.v_cache = static_cast<bf16*>(v_cache);
  p.n_heads = n_heads;
  p.n_kv_heads = n_kv_heads;
  VLO_CUDA(launch_pdl(qkv_rope_append_kernel, dim3(T, n_heads + 2 * n_kv_heads), dim3(64), 0, st, p));
  count_launch();
  return 0;
}

int decision_launch(const void* logits, int n_rows, int vocab, int interval_id, void* out, cudaStream_t st) {
  VLO_CUDA(launch_pdl(decision_kernel, dim3(n_rows), dim3(1024), 0, st, static_cast<const bf16*>(logits), vocab,
                      interval_id, static_cast<DecisionOut*>(out)));
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------ ViT attention launches
// vlo_vit_encode and the kernel-level entry points (capi_ops.cu) launch the ViT attention kernels through these only.
int vit_attn_launch(const void* qkv, void* out, int B, int N, int C, cudaStream_t st) {
  VLO_CHECK(B > 0 && N > 0 && C > 0 && C % kVitHD == 0, "vit_attn: B, N > 0 and hidden = 64 x heads");
  VLO_CHECK(static_cast<long long>(B) * N < (1ll << 31), "vit_attn: too many token rows for a TMA map");
  if (ensure_max_smem(reinterpret_cast<const void*>(vit_attn_kernel), kVitSmemBytes)) return -1;
  const int rows = B * N;
  CUtensorMap tm_qkv;
  if (tmap_2d_sw128(qkv, rows, 3 * C, kVitBlk, FMT_F16, &tm_qkv)) return -1;
  const float scale_log2 = 1.4426950408889634f / 8.0f;  // head_dim 64
  prof_begin(PROF_VIT_ATTN, st, 4.0 * rows * C * 2);
  VLO_CUDA(launch_pdl(vit_attn_kernel, dim3((N + kVitBlk - 1) / kVitBlk, C / kVitHD, B), dim3(kVitThreads), kVitSmemBytes, st,
                      tm_qkv, static_cast<__half*>(out), N, C, scale_log2));
  prof_end(st);
  count_launch();
  return 0;
}

int probe_attn_launch(const void* kv, const float* q, void* out, int B, int N, int C, cudaStream_t st) {
  VLO_CHECK(B > 0 && N > 0 && C > 0 && C % kVitHD == 0, "probe_attn: B, N > 0 and hidden = 64 x heads");
  // the N scores are staged in shared memory without an opt-in beyond the default 48 KB
  VLO_CHECK(static_cast<size_t>(N) * sizeof(float) <= 48 * 1024, "probe_attn: N <= 12288 tokens per frame");
  probe_attn_kernel<<<dim3(C / kVitHD, B), 128, static_cast<size_t>(N) * sizeof(float), st>>>(
      static_cast<const __half*>(kv), q, static_cast<__half*>(out), N, C, 0.125f);  // head_dim 64
  VLO_LAUNCH_CHECK();
  count_launch();
  return 0;
}

// ------------------------------------------------------------------------------ ViT element-wise launches
// vlo_vit_encode and the kernel-level entry points (capi_ops.cu) launch the other ViT kernels through these only.
bool vit_beside_decoder(int B) { return B <= 2; }

int patchify_launch(const uint8_t* frames, void* out, int B, int S, int ps, cudaStream_t st) {
  const int g = S / ps;
  const long long total = static_cast<long long>(B) * g * g * 3 * ps * ps / 8;
  VLO_CUDA(launch_pdl(patchify_kernel, dim3(static_cast<unsigned>(std::min<long long>((total + 255) / 256, 4096))), dim3(256), 0, st,
                      frames, static_cast<__half*>(out), B, S, ps));
  count_launch();
  return 0;
}

int vit_layernorm_launch(const void* in, bool in_f16, int rows, int C, const float* w, const float* b, void* out16,
                         float* out32, float eps, cudaStream_t st) {
  const size_t smem = static_cast<size_t>(C) * sizeof(float);
  if (in_f16) {
    layernorm_kernel<__half><<<rows, 256, smem, st>>>(static_cast<const __half*>(in), w, b, static_cast<__half*>(out16),
                                                      out32, C, eps);
    VLO_LAUNCH_CHECK();
  } else {
    VLO_CUDA(launch_pdl(layernorm_kernel<float>, dim3(rows), dim3(256), smem, st, static_cast<const float*>(in), w, b,
                        static_cast<__half*>(out16), out32, C, eps));
  }
  count_launch();
  return 0;
}

int vit_fix_ln_launch(const float* part, const GemmWsPlan& plan, int rows, int C, const float* bias, float* h,
                      const float* ln_w, const float* ln_b, void* out16, float* out32, float eps, cudaStream_t st) {
  VitFixLnParams p{};
  p.part = part;
  p.sk = plan.sk;
  p.sk_bn = plan.bn;
  p.sk_xtiles = plan.x_tiles;
  p.split_stride = static_cast<long long>(rows) * C;
  p.bias = bias;
  p.h = h;
  p.ln_w = ln_w;
  p.ln_b = ln_b;
  p.out16 = static_cast<__half*>(out16);
  p.out32 = out32;
  p.C = C;
  p.eps = eps;
  VLO_CUDA(launch_pdl(vit_fix_ln_kernel, dim3(rows), dim3(256), static_cast<size_t>(C) * sizeof(float), st, p));
  count_launch();
  return 0;
}

int pool_launch(const float* in, float* tokens, int B, int g, int C, int ph, int pw, int n_tok, int tok_off,
                cudaStream_t st) {
  const long long total = static_cast<long long>(B) * ph * pw * C;
  pool_kernel<<<static_cast<int>(std::min<long long>((total + 255) / 256, 2048)), 256, 0, st>>>(in, tokens, B, g, C, ph, pw,
                                                                                                 n_tok, tok_off);
  VLO_LAUNCH_CHECK();
  count_launch();
  return 0;
}

int cls_residual_launch(const void* resid, const void* mlp, float* tokens, int B, int C, int n_tok, cudaStream_t st) {
  cls_residual_kernel<<<(B * C + 255) / 256, 256, 0, st>>>(static_cast<const __half*>(resid), static_cast<const __half*>(mlp),
                                                           tokens, B, C, n_tok);
  VLO_LAUNCH_CHECK();
  count_launch();
  return 0;
}

int f32_to_bf16_launch(const float* in, void* out, long long n, cudaStream_t st) {
  f32_to_bf16_kernel<<<static_cast<int>(std::min<long long>((n + 255) / 256, 2048)), 256, 0, st>>>(in, static_cast<bf16*>(out), n);
  VLO_LAUNCH_CHECK();
  count_launch();
  return 0;
}

int sample_check_rows(const void* h_rows, int n_rows, int n_ids) {
  VLO_CHECK(h_rows != nullptr, "sample: null rows");
  const SampleRow* rows = static_cast<const SampleRow*>(h_rows);
  for (int i = 0; i < n_rows; ++i) {
    const SampleRow& r = rows[i];
    const std::string at = "sample: row " + std::to_string(i) + ": ";
    VLO_CHECK(r.temperature >= 0.f && r.temperature <= 3.4e38f, at + "temperature must be finite and >= 0 (0: not sampled)");
    if (r.temperature == 0.f) continue;  // a skipped row: nothing else of it is read
    VLO_CHECK(r.top_k >= 0, at + "top_k must be >= 0 (0: off)");
    VLO_CHECK(r.top_p > 0.f, at + "top_p must be > 0 (>= 1: off)");
    VLO_CHECK(r.repetition_penalty > 0.f && r.repetition_penalty <= 3.4e38f, at + "repetition_penalty must be finite and > 0");
    VLO_CHECK(r.penalty_offset >= 0 && r.penalty_count >= 0 &&
                  static_cast<long long>(r.penalty_offset) + r.penalty_count <= n_ids,
              at + "penalty ids [offset, offset + count) must lie in the call's list");
  }
  return 0;
}

int sample_launch(const void* logits, int n_rows, int vocab, const void* rows, const int* penalty_ids, int* out_ids,
                  void* info, cudaStream_t st) {
  const int smem = static_cast<int>(sizeof(uint32_t)) * ((vocab + 31) / 32);
  if (smem + sizeof(SampleShared) > 48 * 1024 && ensure_max_smem(reinterpret_cast<const void*>(sample_kernel), smem))
    return -1;
  VLO_CUDA(launch_pdl(sample_kernel, dim3(n_rows), dim3(kSampleThreads), smem, st, static_cast<const bf16*>(logits), vocab,
                      static_cast<const SampleRow*>(rows), penalty_ids, out_ids, static_cast<SampleInfo*>(info)));
  count_launch();
  return 0;
}

}  // namespace vlo

extern "C" {

static int engine_init(vlo_engine* e, int64_t kv_pool_tokens);

int vlo_engine_create(const vlo_config* cfg, int device, vlo_engine** out) {
  return vlo_engine_create_pooled(cfg, 0, device, out);
}

int vlo_engine_create_pooled(const vlo_config* cfg, int64_t kv_pool_tokens, int device, vlo_engine** out) {
  VLO_CHECK(cfg != nullptr && out != nullptr, "null argument");
  *out = nullptr;
  int prev_dev = -1;
  cudaGetDevice(&prev_dev);
  VLO_CUDA(cudaSetDevice(device));
  if (!vlo_device_supported(device)) return fail("device is not an sm_90 (Hopper) GPU; there is no fallback path");
  const vlo_config& c = *cfg;
  VLO_CHECK(c.head_dim == 128, "decoder head_dim must be 128");
  VLO_CHECK(c.vocab_size % 8 == 0, "vocab_size must be a multiple of 8 (16-byte aligned logits rows)");
  VLO_CHECK(c.hidden_size % 128 == 0 && c.intermediate_size % 128 == 0, "hidden/intermediate must be multiples of 128");
  VLO_CHECK(c.num_heads % c.num_kv_heads == 0, "num_heads % num_kv_heads");
  VLO_CHECK(c.max_streams >= 1 && c.max_kv_tokens >= 64 && c.max_step_tokens >= 1, "capacities");
  VLO_CHECK(kv_pages_for(c.max_kv_tokens) <= attn_max_key_blocks(),
            "max_kv_tokens above " + std::to_string(attn_max_key_blocks() * kKvPageTokens) +
                " (the attention stages a stream's page table in shared memory)");
  VLO_CHECK(c.max_step_tokens <= 128, "max_step_tokens <= 128 (longer inputs run as prefills or are chunked by the host; chunked == one pass)");
  VLO_CHECK(c.vit_layers == 0 || (c.vit_hidden % 128 == 0 && c.vit_hidden == 64 * c.vit_heads && c.vit_mlp % 64 == 0),
            "vision tower: hidden % 64, head_dim == 64");
  VLO_CHECK(c.vit_layers == 0 || (c.image_size % c.patch_size == 0 && (3 * c.patch_size * c.patch_size) % 64 == 0 &&
                                  c.patch_size % 8 == 0),
            "vision tower: patch geometry");
  vlo_engine* e = new vlo_engine();
  e->cfg = c;
  e->device = device;
  e->qkv_width = (c.num_heads + 2 * c.num_kv_heads) * c.head_dim;
  e->grid = c.vit_layers ? c.image_size / c.patch_size : 0;
  e->n_patches = e->grid * e->grid;
  e->patch_k = 3 * c.patch_size * c.patch_size;
  e->n_frame_tokens = (c.frame_token_cls ? 1 : 0) + c.pool_h * c.pool_w;
  const int rc = engine_init(e, kv_pool_tokens);
  if (rc != 0) {   // no half-built engine escapes: free what was allocated, keep the error text
    const std::string msg = last_error();
    vlo_engine_destroy(e);
    set_error(msg);
  } else {
    *out = e;
  }
  if (prev_dev >= 0 && prev_dev != device) cudaSetDevice(prev_dev);
  return rc;
}

static int engine_init(vlo_engine* e, int64_t kv_pool_tokens) {
  const vlo_config& c = e->cfg;
  const int T = c.max_step_tokens;
  const int H = c.hidden_size;
  // KV cache: a pool of 64-token pages shared by all streams, zero-initialised once.  Attention loads (masked) rows
  // past kv_len inside a stream's last page; they may hold anything.
  const int per_stream = kv_pages_for(c.max_kv_tokens);
  const int64_t pages = kv_pool_tokens > 0 ? (kv_pool_tokens + kKvPageTokens - 1) / kKvPageTokens
                                           : static_cast<int64_t>(c.max_streams) * per_stream;
  VLO_CHECK(pages * c.num_kv_heads * kKvPageTokens < (1ll << 31), "KV pool too large for one TMA map per layer");
  e->pool.init(c.max_streams, c.num_kv_heads, static_cast<int>(pages));
  int max_pitch = 0;
  VLO_CUDA(cudaDeviceGetAttribute(&max_pitch, cudaDevAttrMaxPitch, e->device));
  e->max_pitch = static_cast<size_t>(max_pitch);
  const size_t kv_elems = static_cast<size_t>(c.num_layers) * 2 * e->pool.rows_per_layer() * c.head_dim;
  if (dev_alloc_t(e, &e->kv, kv_elems, true)) return -1;
  if (dev_alloc_t(e, &e->kv_op_pt, static_cast<size_t>(2) * per_stream + kRotFloats)) return -1;
  // decision rows: one per sequence, or one per segment of a segmented step (each segment holds >= 1 of the T tokens)
  const int rows = std::max(c.max_streams, T);
  if (dev_alloc_t(e, &e->xn_last, static_cast<size_t>(rows) * H)) return -1;
  if (dev_alloc_t(e, &e->logits, static_cast<size_t>(rows) * c.vocab_size)) return -1;
  if (dev_alloc_t(e, &e->decisions, static_cast<size_t>(rows))) return -1;
  const int widest = std::max(std::max(e->qkv_width, 2 * c.intermediate_size), H);
  // stream-K needs <= kb/floor(U/G) + 2 planes (<= 4 in practice); a prefill's one plane of max_prefill rows fills it
  e->part_elems = static_cast<size_t>(kFixMaxPlanes) * T * widest;
  if (dev_alloc_t(e, &e->part, e->part_elems)) return -1;
  if (dev_alloc_t(e, &e->sk_flags, kSkFlags, true)) return -1;
  e->sample_rows = rows;
  e->sample_ids = align256(sizeof(SampleRow) * rows);
  const size_t sample_bytes = e->sample_ids + sizeof(int) * kSamplePenaltyIds;
  if (dev_alloc(e, reinterpret_cast<void**>(&e->sample_dev), sample_bytes, false)) return -1;
  if (size_token_rows(e, T)) return -1;
  for (int i = 0; i < kStageSlots; ++i) VLO_CUDA(cudaEventCreateWithFlags(&e->stage_events[i], cudaEventDisableTiming));

  if (c.vit_layers > 0) {
    const size_t rows = static_cast<size_t>(c.max_vit_batch) * e->n_patches;
    const int C = c.vit_hidden, B = c.max_vit_batch;
    if (dev_alloc_t(e, &e->patches, rows * e->patch_k)) return -1;
    if (dev_alloc_t(e, &e->v_h, rows * C)) return -1;
    if (dev_alloc_t(e, &e->v_ln32, rows * C)) return -1;
    e->v_part_elems = static_cast<size_t>(8) * rows * C;
    if (dev_alloc_t(e, &e->v_part, e->v_part_elems)) return -1;
    if (dev_alloc_t(e, &e->v_xn, rows * C)) return -1;
    if (dev_alloc_t(e, &e->v_qkv, rows * 3 * C)) return -1;
    if (dev_alloc_t(e, &e->v_attn, rows * C)) return -1;
    if (dev_alloc_t(e, &e->v_mlp, rows * c.vit_mlp)) return -1;
    if (dev_alloc_t(e, &e->v_pa, static_cast<size_t>(B) * C)) return -1;
    if (dev_alloc_t(e, &e->v_resid, static_cast<size_t>(B) * C)) return -1;
    if (dev_alloc_t(e, &e->v_lnh, static_cast<size_t>(B) * C)) return -1;
    if (dev_alloc_t(e, &e->v_m1, static_cast<size_t>(B) * c.vit_mlp)) return -1;
    if (dev_alloc_t(e, &e->v_m2, static_cast<size_t>(B) * C)) return -1;
  }
  {
    const size_t trows = static_cast<size_t>(std::max(1, c.max_vit_batch)) * std::max(1, e->n_frame_tokens);
    const int C = std::max(64, c.vit_hidden);
    if (dev_alloc_t(e, &e->tokens32, trows * C)) return -1;
    if (dev_alloc_t(e, &e->tokens16, trows * C)) return -1;
    if (dev_alloc_t(e, &e->conn_mid, trows * H)) return -1;
  }
  return 0;
}

int vlo_engine_destroy(vlo_engine* e) {
  if (e == nullptr) return 0;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  for (void* p : e->allocs) cudaFree(p);
  if (e->stage) cudaFreeHost(e->stage);
  for (int i = 0; i < kStageSlots; ++i)
    if (e->stage_events[i]) cudaEventDestroy(e->stage_events[i]);
  delete e;
  return 0;
}

int64_t vlo_engine_device_bytes(vlo_engine* e) { return e ? e->device_bytes : 0; }

namespace {
// The e4m3 copies of xn, attn_out and act and their fp32 token scales, for `rows` token rows (zeroed: vlo_bench_gemm).
// Growing frees the old buffers: no work may be in flight.
int size_fp8_act_rows(vlo_engine* e, int rows) {
  const vlo_config& c = e->cfg;
  const size_t H = c.hidden_size, A = static_cast<size_t>(c.num_heads) * c.head_dim, I = c.intermediate_size;
  if (e->xq != nullptr) {
    const size_t old = e->act_rows;
    dev_free(e, &e->xq, old * H);
    dev_free(e, &e->aq, old * A);
    dev_free(e, &e->actq, old * I);
    dev_free(e, &e->xs, old * sizeof(float));
    dev_free(e, &e->as, old * sizeof(float));
    dev_free(e, &e->acts, old * sizeof(float));
  }
  e->act_rows = rows;
  const size_t T = rows;
  if (dev_alloc_t(e, &e->xq, T * H, true)) return -1;
  if (dev_alloc_t(e, &e->aq, T * A, true)) return -1;
  if (dev_alloc_t(e, &e->actq, T * I, true)) return -1;
  if (dev_alloc_t(e, &e->xs, T, true) || dev_alloc_t(e, &e->as, T, true) || dev_alloc_t(e, &e->acts, T, true)) return -1;
  return 0;
}
}  // namespace

int vlo_set_fp8_activations(vlo_engine* e, int on) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr, "null engine");
  VLO_CHECK(!e->finalized, "set_fp8_activations: the mode is chosen before vlo_finalize_weights");
  e->fp8_act = on != 0;
  // the e4m3 activation copies exist only in this mode
  if (e->fp8_act && e->xq == nullptr && size_fp8_act_rows(e, e->cfg.max_step_tokens)) return -1;
  return 0;
}

int vlo_set_quantized_prefill(vlo_engine* e, int on) {
  VLO_CHECK(e != nullptr, "null engine");
  VLO_CHECK(!e->finalized, "set_quantized_prefill: the mode is chosen before vlo_finalize_weights");
  e->quant_prefill = on != 0;
  return 0;
}

int vlo_load_tensor(vlo_engine* e, const char* name, const void* d_ptr, int64_t n_bytes) {
  VLO_CHECK(e != nullptr && name != nullptr && d_ptr != nullptr && n_bytes > 0, "bad argument");
  VLO_CHECK((reinterpret_cast<uintptr_t>(d_ptr) & 15) == 0, std::string("tensor '") + name + "' is not 16-byte aligned");
  e->tensors[name] = {d_ptr, n_bytes};
  e->finalized = false;
  return 0;
}

namespace {
// Layer matrix `name` [n, k] in exactly one form: bf16 `name` (FMT_BF16), e4m3 bytes `name.f8` with fp32 row scales
// `name.scale` (FMT_E4M3, or FMT_E4M3_A8 with fp8_act), or int4 codes `name.i4` with bf16 group scales `name.gscale`
// (FMT_I4).  *fmt < 0: the first matrix, which sets the format every later one must share.
int lookup_layer_matrix(vlo_engine* e, const std::string& name, int64_t n, int64_t k, int* fmt, WeightOperand* out,
                        const char* one = "layer matrix", const char* group = "layer matrices") {
  const bool has16 = e->tensors.count(name) > 0, has8 = e->tensors.count(name + ".f8") > 0,
             has_s = e->tensors.count(name + ".scale") > 0, has4 = e->tensors.count(name + ".i4") > 0,
             has_g = e->tensors.count(name + ".gscale") > 0;
  if (static_cast<int>(has16) + static_cast<int>(has8 || has_s) + static_cast<int>(has4 || has_g) > 1)
    return fail("weight tensor '" + name + "' is loaded in more than one form (bf16, e4m3 '.f8' + '.scale', int4 '.i4' + '.gscale')");
  if (!has16 && !has8 && !has_s && !has4 && !has_g)
    return fail("missing weight tensor '" + name + "' (or '" + name + ".f8' + '" + name + ".scale', or '" + name + ".i4' + '" +
                name + ".gscale')");
  if (has8 != has_s) return fail("missing weight tensor '" + name + (has8 ? ".scale'" : ".f8'"));
  if (has4 != has_g) return fail("missing weight tensor '" + name + (has4 ? ".gscale'" : ".i4'"));
  out->fmt = has8 ? (e->fp8_act ? FMT_E4M3_A8 : FMT_E4M3) : has4 ? FMT_I4 : FMT_BF16;
  if (*fmt >= 0 && out->fmt != *fmt)
    return fail("weight tensor '" + name + (has8 ? ".f8' is e4m3" : has4 ? ".i4' is int4" : "' is bf16") +
                " but an earlier " + one + " is not: all " + group + " must share one form");
  *fmt = out->fmt;
  out->row_scale = nullptr;
  out->group_scale = nullptr;
  if (has4) {
    if (k % kI4Group != 0)
      return fail("weight tensor '" + name + ".i4': int4 weights need K (" + std::to_string(k) +
                  ") to be a multiple of 128, one scale per 128 weights of a row");
    const uint8_t* w;
    if (lookup(e, name + ".i4", (n + kGemmBM - 1) / kGemmBM * kGemmBM * (k / 2), &w) ||
        lookup(e, name + ".gscale", n * (k / kI4Group), &out->group_scale))
      return -1;
    out->w = w;
    return 0;
  }
  if (!has8) {
    const bf16* w;
    if (lookup(e, name, n * k, &w)) return -1;
    out->w = w;
    return 0;
  }
  const uint8_t* w;
  if (lookup(e, name + ".f8", n * k, &w) || lookup(e, name + ".scale", n, &out->row_scale)) return -1;
  out->w = w;
  return 0;
}
}  // namespace

int vlo_finalize_weights(vlo_engine* e) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr, "null engine");
  const vlo_config& c = e->cfg;
  const int64_t H = c.hidden_size, I = c.intermediate_size, V = c.vocab_size;
  e->has_decoder = false;   // any tensor of the embedding table, in any form (a partial form then fails with a message)
  for (const char* n : {"embed", "embed.f8", "embed.scale", "embed.i4", "embed.gscale"}) e->has_decoder |= e->tensors.count(n) > 0;
  if (e->has_decoder) {
    if (lookup(e, "final_norm", H, &e->final_norm)) return -1;
    auto it = e->tensors.find("rope.cos");
    if (it == e->tensors.end()) return fail("missing weight tensor 'rope.cos'");
    e->rope_positions = it->second.second / (64 * 2);
    VLO_CHECK(e->rope_positions >= c.max_kv_tokens, "rope tables shorter than max_kv_tokens");
    if (lookup(e, "rope.cos", e->rope_positions * 64, &e->rope_cos)) return -1;
    if (lookup(e, "rope.sin", e->rope_positions * 64, &e->rope_sin)) return -1;
    std::vector<DecLayer> dec(c.num_layers);   // installed only once every matrix has resolved
    int fmt = -1;
    for (int l = 0; l < c.num_layers; ++l) {
      const std::string p = "L" + std::to_string(l) + ".";
      DecLayer& d = dec[l];
      if (lookup(e, p + "in_norm", H, &d.in_norm)) return -1;
      if (lookup_layer_matrix(e, p + "qkv", e->qkv_width, H, &fmt, &d.qkv)) return -1;
      if (lookup_layer_matrix(e, p + "o", H, static_cast<int64_t>(c.num_heads) * c.head_dim, &fmt, &d.o)) return -1;
      if (lookup(e, p + "post_norm", H, &d.post_norm)) return -1;
      if (lookup_layer_matrix(e, p + "gate_up", 2 * I, H, &fmt, &d.gate_up)) return -1;
      if (lookup_layer_matrix(e, p + "down", H, I, &fmt, &d.down)) return -1;
    }
    VLO_CHECK(!e->fp8_act || fmt != FMT_I4,
              "fp8_activations takes FP8 (e4m3) layer weights, but the layer matrices are int4: 4-bit weights multiply "
              "bf16 activations");
    VLO_CHECK(!e->fp8_act || fmt == FMT_E4M3_A8,
              "fp8_activations needs FP8 (e4m3) layer weights, but the layer matrices are bf16: the FP8 tensor cores "
              "take both operands in e4m3");
    VLO_CHECK(!e->quant_prefill || fmt != FMT_BF16,
              "quantized_prefill needs quantized (FP8 or int4) layer matrices, but they are bf16: a bf16 engine always "
              "prefills");
    // the vocabulary matrices: both bf16, or both in the layer matrices' quantized form (e4m3 on bf16 activations also
    // under fp8_act: the lm_head multiplies the bf16 final-norm rows)
    WeightOperand embed{}, lm_head{};
    int vfmt = -1;
    if (lookup_layer_matrix(e, "embed", V, H, &vfmt, &embed, "vocabulary matrix", "vocabulary matrices") ||
        lookup_layer_matrix(e, "lm_head", V, H, &vfmt, &lm_head, "vocabulary matrix", "vocabulary matrices"))
      return -1;
    if (vfmt == FMT_E4M3_A8) vfmt = embed.fmt = lm_head.fmt = FMT_E4M3;
    const int lfmt = fmt == FMT_E4M3_A8 ? FMT_E4M3 : fmt;
    const char* form_name[] = {"fp16", "bf16", "e4m3", "e4m3", "int4"};
    VLO_CHECK(vfmt == FMT_BF16 || lfmt != FMT_BF16,
              std::string("the vocabulary matrices (embed, lm_head) are ") + form_name[vfmt] +
                  " but the layer matrices are bf16: quantized vocabulary matrices take the layer matrices' form");
    VLO_CHECK(vfmt == FMT_BF16 || vfmt == lfmt,
              std::string("the vocabulary matrices (embed, lm_head) are ") + form_name[vfmt] + " but the layer matrices are " +
                  form_name[lfmt] + ": quantized vocabulary matrices take the layer matrices' form");
    e->dec.swap(dec);
    e->layer_fmt = fmt;
    e->embed = embed;
    e->lm_head = lm_head;
    e->vocab_fmt = vfmt;
  }
  e->has_connector = e->tensors.count("conn.0.w") > 0;
  if (e->has_connector) {
    const int64_t C = c.vit_hidden;
    if (lookup(e, "conn.0.w", H * C, &e->conn0_w)) return -1;
    if (lookup(e, "conn.0.b", H, &e->conn0_b)) return -1;
    if (lookup(e, "conn.2.w", H * H, &e->conn2_w)) return -1;
    if (lookup(e, "conn.2.b", H, &e->conn2_b)) return -1;
  }
  e->has_vit = c.vit_layers > 0 && e->tensors.count("vit.patch.w") > 0;
  if (e->has_vit) {
    const int64_t C = c.vit_hidden, M = c.vit_mlp;
    if (lookup(e, "vit.patch.w", C * e->patch_k, &e->patch_w)) return -1;
    if (lookup(e, "vit.patch.b", C, &e->patch_b)) return -1;
    if (lookup(e, "vit.pos", static_cast<int64_t>(e->n_patches) * C, &e->pos_emb)) return -1;
    if (lookup(e, "vit.post_ln.w", C, &e->post_ln_w)) return -1;
    if (lookup(e, "vit.post_ln.b", C, &e->post_ln_b)) return -1;
    e->vit.resize(c.vit_layers);
    for (int l = 0; l < c.vit_layers; ++l) {
      const std::string p = "vit.L" + std::to_string(l) + ".";
      VitLayer& v = e->vit[l];
      if (lookup(e, p + "ln1.w", C, &v.ln1_w) || lookup(e, p + "ln1.b", C, &v.ln1_b)) return -1;
      if (lookup(e, p + "ln2.w", C, &v.ln2_w) || lookup(e, p + "ln2.b", C, &v.ln2_b)) return -1;
      if (lookup(e, p + "qkv.w", 3 * C * C, &v.qkv_w) || lookup(e, p + "qkv.b", 3 * C, &v.qkv_b)) return -1;
      if (lookup(e, p + "out.w", C * C, &v.out_w) || lookup(e, p + "out.b", C, &v.out_b)) return -1;
      if (lookup(e, p + "fc1.w", M * C, &v.fc1_w) || lookup(e, p + "fc1.b", M, &v.fc1_b)) return -1;
      if (lookup(e, p + "fc2.w", C * M, &v.fc2_w) || lookup(e, p + "fc2.b", C, &v.fc2_b)) return -1;
    }
    if (c.frame_token_cls) {
      if (lookup(e, "vit.head.q", C, &e->head_q)) return -1;
      if (lookup(e, "vit.head.kv.w", 2 * C * C, &e->head_kv_w) || lookup(e, "vit.head.kv.b", 2 * C, &e->head_kv_b)) return -1;
      if (lookup(e, "vit.head.out.w", C * C, &e->head_out_w) || lookup(e, "vit.head.out.b", C, &e->head_out_b)) return -1;
      if (lookup(e, "vit.head.ln.w", C, &e->head_ln_w) || lookup(e, "vit.head.ln.b", C, &e->head_ln_b)) return -1;
      if (lookup(e, "vit.head.fc1.w", M * C, &e->head_fc1_w) || lookup(e, "vit.head.fc1.b", M, &e->head_fc1_b)) return -1;
      if (lookup(e, "vit.head.fc2.w", C * M, &e->head_fc2_w) || lookup(e, "vit.head.fc2.b", C, &e->head_fc2_b)) return -1;
    }
  }
  // A bf16 engine prefills (vlo_prefill): its token-row workspaces grow once to max_prefill rows, and so do those of a
  // quantized engine with quant_prefill (W8A8: with the e4m3 activation copies).  The other quantized engines chunk long
  // inputs into steps and keep them at max_step_tokens.
  if (e->has_decoder && (e->layer_fmt == FMT_BF16 || e->quant_prefill) && e->max_prefill == 0) {
    VLO_CUDA(cudaDeviceSynchronize());   // no step, copy or staging slot of this engine may be in flight
    const int rows = kFixMaxPlanes * c.max_step_tokens;
    if (size_token_rows(e, rows)) return -1;
    if (e->fp8_act && size_fp8_act_rows(e, rows)) return -1;
    e->max_prefill = rows;
  }
  e->finalized = true;
  return 0;
}

// ------------------------------------------------------------------------------ streams
int vlo_stream_open(vlo_engine* e, int* stream_id) {
  VLO_CHECK(e != nullptr && stream_id != nullptr, "null argument");
  return e->pool.open(stream_id);
}
int vlo_stream_reset(vlo_engine* e, int sid) {
  if (check_stream(e, sid)) return -1;
  e->pool.commit(sid, 0);
  return 0;
}
int vlo_stream_close(vlo_engine* e, int sid) {
  if (check_stream(e, sid)) return -1;
  e->pool.close(sid);
  return 0;
}
int vlo_kv_pool_info(vlo_engine* e, int* page_tokens, int64_t* total_pages, int64_t* free_pages) {
  VLO_CHECK(e != nullptr, "null engine");
  if (page_tokens) *page_tokens = kKvPageTokens;
  if (total_pages) *total_pages = e->pool.n_pages;
  if (free_pages) *free_pages = e->pool.free_pages();
  return 0;
}
int vlo_kv_len(vlo_engine* e, int sid, int* out_len) {
  if (check_stream(e, sid)) return -1;
  *out_len = e->pool.len(sid);
  return 0;
}
int vlo_kv_truncate(vlo_engine* e, int sid, int new_len) {
  if (check_stream(e, sid)) return -1;
  VLO_CHECK(new_len >= 0 && new_len <= e->pool.len(sid), "kv_truncate: new_len must be within [0, kv_len]");
  e->pool.commit(sid, new_len);
  return 0;
}
int vlo_kv_fill_synthetic(vlo_engine* e, int sid, int n_tokens, uint64_t seed, void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, sid)) return -1;
  const vlo_config& c = e->cfg;
  VLO_CHECK(n_tokens >= 0 && n_tokens <= c.max_kv_tokens, "kv_fill: n_tokens out of range");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  KvGrowth growth{e->pool};
  if (e->pool.grow(1, &sid, &n_tokens, st)) return -1;
  if (n_tokens > 0) {
    const int* d_pt;
    if (upload_op_tables(e, 1, &sid, &d_pt, st)) return -1;
    kv_fill_kernel<<<dim3(std::min(64, (n_tokens * 128 + 255) / 256), c.num_kv_heads, 2 * c.num_layers), 256, 0, st>>>(
        kv_paged_side(e, e->kv, d_pt), c.num_kv_heads, n_tokens, sid, c.max_kv_tokens, seed);
    VLO_LAUNCH_CHECK();
  }
  e->pool.commit(sid, n_tokens);
  return 0;
}

namespace {
int launch_kv_copy(const KvSide& src, const KvSide& dst, int n_kv, int n_tok, int planes, cudaStream_t st) {
  kv_copy_kernel<<<dim3((n_tok * 16 + 255) / 256, n_kv, planes), 256, 0, st>>>(src, dst, n_kv, n_tok);
  VLO_LAUNCH_CHECK();
  return 0;
}
}  // namespace

int vlo_kv_read(vlo_engine* e, int sid, int layer, int is_v, void* d_out, void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, sid)) return -1;
  const vlo_config& c = e->cfg;
  VLO_CHECK(layer >= 0 && layer < c.num_layers, "layer out of range");
  VLO_CHECK((reinterpret_cast<uintptr_t>(d_out) & 15) == 0, "kv_read: d_out must be 16-byte aligned");
  const int len = e->pool.len(sid);
  if (len == 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const int* d_pt;
  if (upload_op_tables(e, 1, &sid, &d_pt, st)) return -1;
  return launch_kv_copy(kv_paged_side(e, kv_layer_base(e, layer, is_v), d_pt), KvSide{static_cast<bf16*>(d_out), nullptr, 0, len},
                        c.num_kv_heads, len, 1, st);
}
int vlo_kv_write(vlo_engine* e, int sid, int layer, int is_v, const void* d_in, int n_tokens, void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, sid)) return -1;
  const vlo_config& c = e->cfg;
  VLO_CHECK(layer >= 0 && layer < c.num_layers, "layer out of range");
  VLO_CHECK(n_tokens > 0 && n_tokens <= c.max_kv_tokens, "kv_write: n_tokens out of range");
  VLO_CHECK((reinterpret_cast<uintptr_t>(d_in) & 15) == 0, "kv_write: d_in must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  KvGrowth growth{e->pool};
  if (e->pool.grow(1, &sid, &n_tokens, st)) return -1;
  const int* d_pt;
  if (upload_op_tables(e, 1, &sid, &d_pt, st)) return -1;
  if (launch_kv_copy(KvSide{static_cast<bf16*>(const_cast<void*>(d_in)), nullptr, 0, n_tokens},
                     kv_paged_side(e, kv_layer_base(e, layer, is_v), d_pt), c.num_kv_heads, n_tokens, 1, st))
    return -1;
  e->pool.commit(sid, n_tokens);
  return 0;
}

int vlo_kv_copy_prefix(vlo_engine* e, int src_sid, int dst_sid, int n_tokens, void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, src_sid) || check_stream(e, dst_sid)) return -1;
  const vlo_config& c = e->cfg;
  VLO_CHECK(src_sid != dst_sid, "kv_copy_prefix: source and destination streams must differ");
  VLO_CHECK(n_tokens >= 0 && n_tokens <= e->pool.len(src_sid), "kv_copy_prefix: n_tokens exceeds the source length");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  KvGrowth growth{e->pool};
  if (n_tokens > 0) {  // the copy overwrites the destination from position 0: it waits for swap-outs of any of its pages
    if (e->pool.grow(1, &dst_sid, &n_tokens, st, true)) return -1;
    const int sids[2] = {src_sid, dst_sid};
    const int* d_pt[2];
    if (upload_op_tables(e, 2, sids, d_pt, st)) return -1;
    if (launch_kv_copy(kv_paged_side(e, e->kv, d_pt[0]), kv_paged_side(e, e->kv, d_pt[1]), c.num_kv_heads, n_tokens,
                       2 * c.num_layers, st))
      return -1;
  }
  e->pool.commit(dst_sid, n_tokens);
  return 0;
}

int vlo_kv_evict(vlo_engine* e, int sid, int first_token, int n_tokens, const float* h_cos, const float* h_sin,
                 void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, sid)) return -1;
  const vlo_config& c = e->cfg;
  VLO_CHECK(h_cos != nullptr && h_sin != nullptr, "kv_evict: null cos / sin table");
  VLO_CHECK(n_tokens > 0 && first_token >= 0 && first_token % kKvPageTokens == 0 && n_tokens % kKvPageTokens == 0,
            "kv_evict: first_token >= 0 and n_tokens > 0 must be multiples of " + std::to_string(kKvPageTokens));
  const int len = e->pool.len(sid), full = len / kKvPageTokens * kKvPageTokens;
  VLO_CHECK(static_cast<long long>(first_token) + n_tokens <= full,
            "kv_evict: every dropped page must be full: first_token + n_tokens <= " + std::to_string(full) + " (kv_len " +
                std::to_string(len) + ")");
  const int kept = len - first_token - n_tokens;  // positions after the dropped range: their keys move by -n_tokens
  if (kept > 0) {
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    // one staging slot, one copy: cos | sin | the stream's current table (the kernel addresses the old positions)
    uint8_t* hs;
    int slot;
    if (stage_acquire(e, &hs, &slot)) return -1;
    const std::vector<int>& tab = e->pool.table(sid);
    float* rot = reinterpret_cast<float*>(hs + e->meta.pt);
    std::memcpy(rot, h_cos, sizeof(float) * c.head_dim / 2);
    std::memcpy(rot + c.head_dim / 2, h_sin, sizeof(float) * c.head_dim / 2);
    std::memcpy(rot + kRotFloats, tab.data(), sizeof(int) * tab.size());
    VLO_CUDA(cudaMemcpyAsync(e->kv_op_pt, rot, sizeof(float) * kRotFloats + sizeof(int) * tab.size(),
                             cudaMemcpyHostToDevice, st));
    if (stage_release(e, slot, st)) return -1;
    kv_rerotate_kernel<<<dim3((kept * 8 + 255) / 256, c.num_kv_heads, c.num_layers), 256, 0, st>>>(
        kv_paged_side(e, e->kv, e->kv_op_pt + kRotFloats), c.num_kv_heads, first_token + n_tokens, kept,
        reinterpret_cast<const float*>(e->kv_op_pt));
    VLO_LAUNCH_CHECK();
  }
  e->pool.drop(sid, first_token / kKvPageTokens, n_tokens / kKvPageTokens);
  return 0;
}

namespace {
// vlo_kv_compact's tables, laid out the same way in a staging slot and at the start of e->part:
// cos | sin [n][head_dim] fp32, then src [n], dst [n] and the stream's page table, int32
size_t compact_table_bytes(const vlo_engine* e, int n_spans) {
  return sizeof(float) * n_spans * e->cfg.head_dim + sizeof(int) * (2 * static_cast<size_t>(n_spans) +
                                                                     kv_pages_for(e->cfg.max_kv_tokens));
}
// most spans one call may pass: its tables fill at most one staging slot
int compact_max_spans(const vlo_engine* e) {
  const size_t per_span = sizeof(float) * e->cfg.head_dim + 2 * sizeof(int);
  return static_cast<int>((e->stage_slot_bytes - compact_table_bytes(e, 0)) / per_span);
}
}  // namespace

int vlo_kv_compact(vlo_engine* e, int sid, int n_spans, const int32_t* h_keep_first, const int32_t* h_keep_len,
                   const float* h_rot, void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, sid)) return -1;
  const vlo_config& c = e->cfg;
  const int cap = compact_max_spans(e);
  VLO_CHECK(n_spans > 0 && n_spans <= cap, "kv_compact: n_spans must be within [1, " + std::to_string(cap) + "], got " +
                                               std::to_string(n_spans));
  VLO_CHECK(h_keep_first != nullptr && h_keep_len != nullptr && h_rot != nullptr, "kv_compact: null span table");
  const int len = e->pool.len(sid);
  long long kept = 0, end = 0;  // end: first position after the previous span
  int first_moved = -1;         // first span with a shift > 0: every later one has one as well
  for (int i = 0; i < n_spans; ++i) {
    const long long f = h_keep_first[i], n = h_keep_len[i];
    VLO_CHECK(n > 0, "kv_compact: span " + std::to_string(i) + " is empty");
    VLO_CHECK(f >= end, "kv_compact: spans must be sorted and non-overlapping (span " + std::to_string(i) + ")");
    VLO_CHECK(f + n <= len, "kv_compact: span " + std::to_string(i) + " ends past kv_len " + std::to_string(len));
    if (first_moved < 0 && f > kept) first_moved = i;
    kept += n;
    end = f + n;
  }
  VLO_CHECK(kept < len, "kv_compact: the spans keep every position: nothing is dropped");
  const int new_len = static_cast<int>(kept);
  const size_t unit_bytes = kv_page_bytes(e), head = align256(compact_table_bytes(e, n_spans));
  const size_t part_bytes = e->part_elems * sizeof(float);
  const long long batch_units = part_bytes > head ? static_cast<long long>((part_bytes - head) / unit_bytes) : 0;
  VLO_CHECK(batch_units > 0, "kv_compact: the step workspace cannot stage one KV page");
  if (first_moved >= 0) {
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    uint8_t* hs;
    int slot;
    if (stage_acquire(e, &hs, &slot)) return -1;
    const std::vector<int>& tab = e->pool.table(sid);
    float* cs = reinterpret_cast<float*>(hs);
    int* src = reinterpret_cast<int*>(cs + static_cast<size_t>(n_spans) * c.head_dim);
    int* dst = src + n_spans;
    std::memcpy(cs, h_rot, sizeof(float) * n_spans * c.head_dim);
    std::memcpy(src, h_keep_first, sizeof(int) * n_spans);
    for (int i = 0, q = 0; i < n_spans; q += h_keep_len[i++]) dst[i] = q;
    const int q_lo = dst[first_moved];
    std::memcpy(dst + n_spans, tab.data(), sizeof(int) * tab.size());
    uint8_t* d_tab = reinterpret_cast<uint8_t*>(e->part);
    VLO_CUDA(cudaMemcpyAsync(d_tab, hs, compact_table_bytes(e, n_spans), cudaMemcpyHostToDevice, st));
    if (stage_release(e, slot, st)) return -1;
    const float* d_cs = reinterpret_cast<const float*>(d_tab);
    const int* d_src = reinterpret_cast<const int*>(d_cs + static_cast<size_t>(n_spans) * c.head_dim);
    const CompactSpans sp{d_cs, d_src, d_src + n_spans, n_spans};
    const KvSide kv = kv_paged_side(e, e->kv, d_src + 2 * n_spans);
    bf16* stage = reinterpret_cast<bf16*>(d_tab + head);
    // (destination page, plane) units from the page of q_lo on, page-major: page j's units run before page j + 1's
    const int planes = 2 * c.num_layers, j0 = q_lo / kKvPageTokens;
    const long long units = static_cast<long long>(kv_pages_for(new_len) - j0) * planes;
    const long long per_unit = static_cast<long long>(c.num_kv_heads) * kKvPageTokens * 8;
    for (long long u0 = 0; u0 < units; u0 += batch_units) {
      const int n = static_cast<int>(std::min(batch_units, units - u0));
      const dim3 grid(static_cast<unsigned>((n * per_unit + 255) / 256));
      for (int to_stage = 1; to_stage >= 0; --to_stage) {
        kv_compact_kernel<<<grid, 256, 0, st>>>(kv, c.num_kv_heads, planes, j0, static_cast<int>(u0), n, q_lo, new_len,
                                                sp, stage, to_stage);
        VLO_LAUNCH_CHECK();
      }
    }
  }
  e->pool.commit(sid, new_len);
  return 0;
}

// ------------------------------------------------------------------------------ host images of a stream's cache
// One cudaMemcpy2DAsync per page moves the page's 2L planes (K and V of every layer, each at the plane stride of the
// pool) to or from `kv_page_bytes x 2L` contiguous host bytes: copy engines only, no SM is taken from other streams.
namespace {
int swap_copies(vlo_engine* e, int sid, uint8_t* h, bool to_host, cudaStream_t st) {
  const size_t pb = kv_page_bytes(e), pitch = kv_plane_elems(e) * sizeof(bf16);
  const size_t planes = static_cast<size_t>(2) * e->cfg.num_layers;
  VLO_CHECK(pitch <= e->max_pitch, "kv swap: the pool's plane stride (" + std::to_string(pitch) +
                                       " B) exceeds the device's maximum copy pitch");
  const std::vector<int>& tab = e->pool.table(sid);
  for (size_t j = 0; j < tab.size(); ++j) {
    uint8_t* dev = reinterpret_cast<uint8_t*>(e->kv) + static_cast<size_t>(tab[j]) * pb;
    uint8_t* host = h + j * planes * pb;
    if (to_host)
      VLO_CUDA(cudaMemcpy2DAsync(host, pb, dev, pitch, pb, planes, cudaMemcpyDeviceToHost, st));
    else
      VLO_CUDA(cudaMemcpy2DAsync(dev, pitch, host, pb, pb, planes, cudaMemcpyHostToDevice, st));
  }
  return 0;
}

int check_pinned(const void* h, const char* what) {
  cudaPointerAttributes a{};
  VLO_CUDA(cudaPointerGetAttributes(&a, h));
  VLO_CHECK(a.type == cudaMemoryTypeHost, std::string(what) + ": the host image must be pinned (page-locked) memory");
  return 0;
}
}  // namespace

int64_t vlo_kv_image_bytes(vlo_engine* e, int n_tokens) {
  if (e == nullptr || n_tokens < 0) return -1;
  return static_cast<int64_t>(kv_pages_for(n_tokens)) * 2 * e->cfg.num_layers * static_cast<int64_t>(kv_page_bytes(e));
}

int vlo_kv_swap_out(vlo_engine* e, int sid, void* h_dst, int64_t bytes, void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, sid)) return -1;
  const int n = e->pool.len(sid);
  if (n == 0) return 0;
  VLO_CHECK(h_dst != nullptr && bytes >= vlo_kv_image_bytes(e, n),
            "kv_swap_out: the host image needs " + std::to_string(vlo_kv_image_bytes(e, n)) + " bytes");
  if (check_pinned(h_dst, "kv_swap_out")) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  if (swap_copies(e, sid, static_cast<uint8_t*>(h_dst), true, st)) return -1;
  return e->pool.swap_out(sid, st);
}

int vlo_kv_swap_in(vlo_engine* e, int sid, const void* h_src, int n_tokens, void* cuda_stream) {
  DevGuard dev_guard(e);
  if (check_stream(e, sid)) return -1;
  VLO_CHECK(e->pool.len(sid) == 0, "kv_swap_in: the stream must be empty (kv_len " + std::to_string(e->pool.len(sid)) + ")");
  VLO_CHECK(n_tokens >= 0 && n_tokens <= e->cfg.max_kv_tokens, "kv_swap_in: n_tokens out of range");
  if (n_tokens == 0) return 0;
  VLO_CHECK(h_src != nullptr, "kv_swap_in: null host image");
  if (check_pinned(h_src, "kv_swap_in")) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  KvGrowth growth{e->pool};
  if (e->pool.grow(1, &sid, &n_tokens, st) ||
      swap_copies(e, sid, static_cast<uint8_t*>(const_cast<void*>(h_src)), false, st))
    return -1;
  e->pool.commit(sid, n_tokens);
  return 0;
}

// ------------------------------------------------------------------------------ vision
int vlo_connector(vlo_engine* e, const void* d_tokens, int n_rows, void* d_out, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->finalized && e->has_connector, "connector weights not loaded");
  const vlo_config& c = e->cfg;
  const int cap = std::max(1, c.max_vit_batch) * std::max(1, e->n_frame_tokens);
  VLO_CHECK(n_rows > 0 && n_rows <= cap, "connector: n_rows exceeds max_vit_batch * frame_num_tokens");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  // Linear -> GELU (python erf form, bf16) -> Linear   (models/live_llama/modeling_live_llama.py:18-22)
  const bf16* tok = static_cast<const bf16*>(d_tokens);
  bf16* outp = static_cast<bf16*>(d_out);
  for (int r0 = 0; r0 < n_rows; r0 += 128) {  // the persistent kernel takes <= 128 token rows per launch
    const int nr = std::min(128, n_rows - r0);
    if (gemm_ws_store16(FMT_BF16, e->conn0_w, c.hidden_size, tok + static_cast<size_t>(r0) * c.vit_hidden, nr, c.vit_hidden,
                        e->conn_mid, c.hidden_size, e->conn0_b, ACT_GELU_ERF_PY, st))
      return -1;
    if (gemm_ws_store16(FMT_BF16, e->conn2_w, c.hidden_size, e->conn_mid, nr, c.hidden_size,
                        outp + static_cast<size_t>(r0) * c.hidden_size, c.hidden_size, e->conn2_b, ACT_NONE, st))
      return -1;
  }
  return 0;
}

int vlo_vit_encode(vlo_engine* e, const uint8_t* d_frames, int B, void* d_out, float* d_vit_tokens, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->finalized && e->has_vit, "vision tower weights not loaded");
  const vlo_config& c = e->cfg;
  VLO_CHECK(B > 0 && B <= c.max_vit_batch, "vit_encode: batch exceeds max_vit_batch");
  VLO_CHECK(e->n_frame_tokens > 0, "no frame tokens configured");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const int C = c.vit_hidden, M = c.vit_mlp, P = e->n_patches, rows = B * P;

  // K1/K2: normalise + patchify, then patch-embed GEMM with bias + position embedding epilogue
  {
    if (patchify_launch(d_frames, e->patches, B, c.image_size, c.patch_size, st)) return -1;
    GemmCall g{};
    g.epi = EPI_PATCH32;
    g.a = e->patches;
    g.rows_a = rows;
    g.b = e->patch_w;
    g.rows_b = C;
    g.k = e->patch_k;
    g.out = e->v_h;
    g.ld_out = C;
    g.bias = e->patch_b;
    g.pos = e->pos_emb;
    g.pos_rows = P;
    if (gemm_launch(g, st)) return -1;
  }
  // Trunk GEMMs: QKV and fc1 run whole tiles with the fused bias / GELU fp16 epilogue; out_proj and fc2 (few
  // output tiles) run stream-K over all SMs on the persistent swap-AB kernel (weights ride MMA-M, the token rows are
  // tiled along MMA-N) and their partial planes are folded into the fp32 residual stream together with the NEXT
  // LayerNorm by vit_fix_ln_kernel.
  // Small batches (the single-stream case) use CTAs that fit on an SM NEXT TO a decoder weight-streaming CTA (119 KB;
  // gemm.cu checks the sums), so the tensor-bound ViT of frame i+1 and the HBM-bound decoder step of frame i execute
  // concurrently (two CUDA streams): QKV and fc1 on gemm_vit_kernel (128-token x 128-feature tiles, tokens on MMA-M,
  // 97 KB), out_proj and fc2 with 64-token tiles and a 3-stage ring (83 KB).  gemm_vit_kernel gives QKV / fc1 the
  // same bits as 64-token swap-AB tiles would; the stream-K planes keep the 64-token decomposition, whose summation
  // order the frame embeddings depend on.
  const bool small = vit_beside_decoder(B);
  auto tiles_gemm = [&](const __half* x, const __half* w, int n_out, int k, __half* out, const float* bias, int act) -> int {
    if (small) return gemm_vit_launch(x, rows, w, n_out, k, out, n_out, bias, act, 0, st);
    return gemm_ws_store16(FMT_F16, w, n_out, x, rows, k, out, n_out, bias, act, st, WS_TILE_TRUNK);
  };
  auto partial_gemm = [&](const __half* x, const __half* w, int k, GemmWsPlan* plan) -> int {
    return gemm_partial(WeightOperand{FMT_F16, w, nullptr, nullptr}, C, x, nullptr, rows, k, e->v_part, e->v_part_elems,
                        small ? WS_TILE_BESIDE_DECODER : WS_TILE_TRUNK, plan, st);
  };
  auto fix_ln = [&](const GemmWsPlan& plan, const float* bias, const float* lw, const float* lb, float* out32) -> int {
    return vit_fix_ln_launch(e->v_part, plan, rows, C, bias, e->v_h, lw, lb, e->v_xn, out32, c.vit_ln_eps, st);
  };
  if (vit_layernorm_launch(e->v_h, false, rows, C, e->vit[0].ln1_w, e->vit[0].ln1_b, e->v_xn, nullptr, c.vit_ln_eps, st))
    return -1;
  for (int l = 0; l < c.vit_layers; ++l) {
    const VitLayer& v = e->vit[l];
    GemmWsPlan sk{};
    if (tiles_gemm(e->v_xn, v.qkv_w, 3 * C, C, e->v_qkv, v.qkv_b, ACT_NONE)) return -1;
    // ViT attention: mma.sync m16n8k16 over TMA-loaded Q / K / V tiles (vit_kernels.cuh)
    if (vit_attn_launch(e->v_qkv, e->v_attn, B, P, C, st)) return -1;
    if (partial_gemm(e->v_attn, v.out_w, C, &sk)) return -1;
    if (fix_ln(sk, v.out_b, v.ln2_w, v.ln2_b, nullptr)) return -1;
    if (tiles_gemm(e->v_xn, v.fc1_w, M, C, e->v_mlp, v.fc1_b, ACT_GELU_TANH)) return -1;
    if (partial_gemm(e->v_mlp, v.fc2_w, M, &sk)) return -1;
    const bool last = (l == c.vit_layers - 1);
    // the LayerNorm that follows fc2: next block's layer_norm1, or post_layernorm (fp16 copy feeds the MAP
    // head, fp32 copy feeds the pool)
    if (fix_ln(sk, v.fc2_b, last ? e->post_ln_w : e->vit[l + 1].ln1_w, last ? e->post_ln_b : e->vit[l + 1].ln1_b,
               last ? e->v_ln32 : nullptr))
      return -1;
  }
  const int NT = e->n_frame_tokens;
  const int cls = c.frame_token_cls ? 1 : 0;
  if (c.pool_h * c.pool_w > 0 && pool_launch(e->v_ln32, e->tokens32, B, e->grid, C, c.pool_h, c.pool_w, NT, cls, st))
    return -1;
  if (cls) {
    // MAP head: K/V projection of all tokens, 1-query attention, out-proj, LN, MLP, residual
    if (gemm_store16(e->v_xn, rows, e->head_kv_w, 2 * C, C, e->v_qkv, 2 * C, e->head_kv_b, ACT_NONE, st)) return -1;
    if (probe_attn_launch(e->v_qkv, e->head_q, e->v_pa, B, P, C, st)) return -1;
    VLO_CHECK(B <= 128, "MAP head handles <= 128 frames per call");
    if (gemm_ws_store16(FMT_F16, e->head_out_w, C, e->v_pa, B, C, e->v_resid, C, e->head_out_b, ACT_NONE, st)) return -1;
    if (vit_layernorm_launch(e->v_resid, true, B, C, e->head_ln_w, e->head_ln_b, e->v_lnh, nullptr, c.vit_ln_eps, st))
      return -1;
    if (gemm_ws_store16(FMT_F16, e->head_fc1_w, M, e->v_lnh, B, C, e->v_m1, M, e->head_fc1_b, ACT_GELU_TANH, st)) return -1;
    if (gemm_ws_store16(FMT_F16, e->head_fc2_w, C, e->v_m1, B, M, e->v_m2, C, e->head_fc2_b, ACT_NONE, st)) return -1;
    if (cls_residual_launch(e->v_resid, e->v_m2, e->tokens32, B, C, NT, st)) return -1;
  }
  const long long ntok_elems = static_cast<long long>(B) * NT * C;
  if (d_vit_tokens)
    VLO_CUDA(cudaMemcpyAsync(d_vit_tokens, e->tokens32, ntok_elems * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (d_out) {
    if (f32_to_bf16_launch(e->tokens32, e->tokens16, ntok_elems, st)) return -1;
    return vlo_connector(e, e->tokens16, B * NT, d_out, cuda_stream);
  }
  return 0;
}

int vlo_letterbox(vlo_engine* e, const vlo_letterbox_frame* h_frames, int n_frames, uint8_t* d_out, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr, "null engine");
  VLO_CHECK(n_frames > 0 && n_frames <= e->cfg.max_vit_batch, "letterbox: n_frames must lie in [1, max_vit_batch]");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return letterbox_launch(h_frames, n_frames, e->cfg.image_size, d_out, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_letterbox_planes(vlo_engine* e, const vlo_frame_planes* h_frames, int n_frames, uint8_t* d_out, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr, "null engine");
  VLO_CHECK(n_frames > 0 && n_frames <= e->cfg.max_vit_batch, "letterbox: n_frames must lie in [1, max_vit_batch]");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return letterbox_planes_launch(h_frames, n_frames, e->cfg.image_size, d_out, static_cast<cudaStream_t>(cuda_stream));
}

// ------------------------------------------------------------------------------ decoder
int vlo_embed_tokens(vlo_engine* e, const int64_t* d_ids, int n, void* d_out, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->finalized && e->has_decoder, "decoder weights not loaded");
  VLO_CHECK(n > 0, "embed_tokens: n must be positive");
  return embed_rows_launch(e->embed, reinterpret_cast<const long long*>(d_ids), n, e->cfg.vocab_size, e->cfg.hidden_size,
                           d_out, static_cast<cudaStream_t>(cuda_stream));
}

namespace {

// The decoder step.  Sequence i carries h_seg_counts[i] consecutive segments (h_seg_counts == NULL: one each) whose
// lengths follow one another in h_seg_lens; one lm_head row and one decision per segment, read at its last row.
// prefill (vlo_prefill): one sequence of one segment, up to max_prefill rows, whose layer GEMMs run on
// gemm_prefill_kernel (bf16) or gemm_prefill_q_kernel (quantized formats) and whose attention plans each max_step_tokens piece as a step of its own: the bits of the same
// rows fed as max_step_tokens steps.
int step_segments(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, const int32_t* h_seg_counts,
                  const int32_t* h_seg_lens, const int64_t* d_row_ids, const void* d_embeds, void* d_last_logits,
                  vlo_decision* d_decisions, int interval_id, cudaStream_t st, bool prefill = false) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->finalized && e->has_decoder, "decoder weights not loaded");
  const vlo_config& c = e->cfg;
  VLO_CHECK(n_seqs > 0 && n_seqs <= c.max_streams, "step: n_seqs out of range");
  VLO_CHECK(h_stream_ids != nullptr && h_seg_lens != nullptr, "step: null argument");
  const int H = c.hidden_size;
  int T = 0, n_rows = 0;
  std::vector<int> q_lens(n_seqs), seg0(n_seqs), ends(n_seqs);  // seg0[i]: index of sequence i's first segment
  for (int i = 0; i < n_seqs; ++i) {
    if (check_stream(e, h_stream_ids[i])) return -1;
    for (int j = 0; j < i; ++j) VLO_CHECK(h_stream_ids[j] != h_stream_ids[i], "step: a stream appears twice in one batch");
    const int n_segs = h_seg_counts ? h_seg_counts[i] : 1;
    VLO_CHECK(n_segs > 0, "step: a sequence needs at least one segment");
    seg0[i] = n_rows;
    for (int j = 0; j < n_segs; ++j) {
      const int32_t q_len = h_seg_lens[n_rows + j];
      VLO_CHECK(q_len > 0, "step: q_len and segment lengths must be positive");
      q_lens[i] += q_len;
    }
    n_rows += n_segs;
    ends[i] = e->pool.len(h_stream_ids[i]) + q_lens[i];
    VLO_CHECK(ends[i] <= c.max_kv_tokens, "step: KV cache capacity exceeded for stream " + std::to_string(h_stream_ids[i]));
    T += q_lens[i];
  }
  // every segment holds at least one token, so the n_rows <= T decision rows fit the buffers sized in engine_init
  if (prefill)
    VLO_CHECK(n_seqs == 1 && n_rows == 1 && T <= e->max_prefill,
              "prefill: one stream of 1.." + std::to_string(e->max_prefill) + " tokens (max_prefill_tokens)");
  else
    VLO_CHECK(T <= c.max_step_tokens, "step: total new tokens exceed max_step_tokens");
  const int32_t* h_q_lens = q_lens.data();
  // ---- pages for the new tokens, taken before anything is enqueued
  KvGrowth growth{e->pool};
  if (e->pool.grow(n_seqs, h_stream_ids, ends.data(), st)) return -1;

  // ---- per-step metadata: built on the host, one pinned slot, uploaded once, reused by all layers
  uint8_t* hs;
  int slot;
  if (stage_acquire(e, &hs, &slot)) return -1;
  int* tok_pos = reinterpret_cast<int*>(hs + e->meta.pos);
  int* last_index = reinterpret_cast<int*>(hs + e->meta.last);
  int* first_rows = reinterpret_cast<int*>(hs + e->meta.first);
  long long* tok_kvrow = reinterpret_cast<long long*>(hs + e->meta.kvrow);
  std::vector<int> pt0(n_seqs);
  const int n_pt = stage_page_tables(e, hs, n_seqs, h_stream_ids, pt0.data());
  std::vector<AttnSeq> seqs(n_seqs);
  std::vector<int> pieces;   // prefill: the max_step_tokens pieces of the chunked path, each attended as its own step
  for (int o = 0; prefill && o < T; o += c.max_step_tokens) pieces.push_back(std::min(c.max_step_tokens, T - o));
  int t = 0;
  for (int i = 0; i < n_seqs; ++i) {
    const int sid = h_stream_ids[i], ql = h_q_lens[i], past = e->pool.len(sid);
    const int n_segs = h_seg_counts ? h_seg_counts[i] : 1;
    first_rows[i] = t;
    for (int j = 0; j < ql; ++j) {
      tok_pos[t + j] = past + j;
      tok_kvrow[t + j] = e->pool.row(sid, past + j);
      last_index[t + j] = -1;
    }
    for (int s = 0, end = 0; s < n_segs; ++s) {  // the decision row of each segment sits at its last token
      end += h_seg_lens[seg0[i] + s];
      last_index[t + end - 1] = seg0[i] + s;
    }
    seqs[i] = prefill ? AttnSeq{t, ql, past + ql, pt0[i], static_cast<int>(pieces.size()), pieces.data()}
                      : AttnSeq{t, ql, past + ql, pt0[i], n_segs, h_seg_lens + seg0[i]};
    t += ql;
  }
  VLO_CUDA(cudaMemcpyAsync(e->meta_dev, hs, e->meta.pt + sizeof(int) * n_pt, cudaMemcpyHostToDevice, st));
  const int* d_tok_pos = reinterpret_cast<const int*>(e->meta_dev + e->meta.pos);
  const int* d_last_index = reinterpret_cast<const int*>(e->meta_dev + e->meta.last);
  const long long* d_tok_kvrow = reinterpret_cast<const long long*>(e->meta_dev + e->meta.kvrow);
  AttnPlan plan{};
  if (attn_plan(&plan, e->attn_ws, hs + e->meta.bytes, seqs.data(), n_seqs, T, c.num_heads, c.num_kv_heads, c.head_dim, st))
    return -1;
  if (stage_release(e, slot, st)) return -1;

  // ---- residual stream <- packed input embeddings (+ prefix-token rows gathered by id)
  VLO_CUDA(cudaMemcpyAsync(e->h, d_embeds, static_cast<size_t>(T) * H * sizeof(bf16), cudaMemcpyDeviceToDevice, st));
  if (d_row_ids != nullptr &&
      embed_rows_launch(e->embed, reinterpret_cast<const long long*>(d_row_ids), T, c.vocab_size, H, e->h, st))
    return -1;

  // sk == null: no partials (the first layer's input norm).  With fp8_act every norm but the final one also writes the
  // e4m3 copy of xn that the next GEMM reads.
  const bool a8 = e->fp8_act;
  auto resid_norm = [&](const GemmWsPlan* sk, const bf16* w, bool last) -> int {
    if (a8 && !last)
      return resid_rmsnorm_q8_launch(sk ? e->part : nullptr, sk ? &sk->sk : nullptr, e->h, w, e->xn, nullptr, nullptr,
                                     e->xq, e->xs, T, H, c.rms_norm_eps, st);
    return resid_rmsnorm_launch(sk ? e->part : nullptr, sk ? &sk->sk : nullptr, e->h, w, e->xn, last ? e->xn_last : nullptr,
                                last ? d_last_index : nullptr, T, H, c.rms_norm_eps, st);
  };
  const void* xn_in = a8 ? static_cast<const void*>(e->xq) : e->xn;
  const void* attn_in = a8 ? static_cast<const void*>(e->aq) : e->attn_out;
  const void* act_in = a8 ? static_cast<const void*>(e->actq) : e->act;
  // the layer GEMMs: stream-K partial planes of the step's plan, or the prefill GEMM's one plane (fix-up plan: G = 1)
  auto partial = [&](const WeightOperand& w, int n_out, const void* x, int k, GemmWsPlan* sk, const float* x_scale) -> int {
    if (!prefill) return gemm_partial(w, n_out, x, x_scale, T, k, e->part, e->part_elems, WS_TILE_FIT, sk, st);
    VLO_CHECK(static_cast<size_t>(T) * n_out <= e->part_elems, "prefill: the plane exceeds the partial workspace");
    return gemm_prefill_launch(PREFILL_PLANE, w, n_out, x, T, k, 0, e->part, st, &sk->sk, x_scale);
  };
  auto swiglu = [&](const WeightOperand& w) -> int {
    if (!prefill) return gemm_swiglu(e, w, 2 * c.intermediate_size, xn_in, T, H, st, a8 ? e->xs : nullptr);
    return gemm_prefill_launch(PREFILL_SWIGLU, w, 2 * c.intermediate_size, xn_in, T, H, 0, e->act, st, nullptr,
                               a8 ? e->xs : nullptr);
  };

  if (resid_norm(nullptr, e->dec[0].in_norm, false)) return -1;
  const int attn_width = c.num_heads * c.head_dim;
  for (int l = 0; l < c.num_layers; ++l) {
    const DecLayer& d = e->dec[l];
    GemmWsPlan sk{};
    const bool is_last = (l == c.num_layers - 1);
    // ---- q|k|v projection, then RoPE + in-place KV append
    if (partial(d.qkv, e->qkv_width, xn_in, H, &sk, a8 ? e->xs : nullptr)) return -1;
    if (qkv_rope_launch(e->part, sk.sk, e->rope_cos, e->rope_sin, d_tok_pos, d_tok_kvrow, KvPool::head_stride_rows(), e->q,
                        kv_layer_base(e, l, 0), kv_layer_base(e, l, 1), T, c.num_heads, c.num_kv_heads, st))
      return -1;
    if (attn_layer(e, plan, l, st)) return -1;
    // ---- o_proj + residual, then post-attention RMSNorm
    if (a8 && quant_rows_launch(e->attn_out, T, attn_width, e->aq, e->as, st)) return -1;
    if (partial(d.o, H, attn_in, attn_width, &sk, a8 ? e->as : nullptr)) return -1;
    if (resid_norm(&sk, d.post_norm, false)) return -1;
    // ---- gate|up + SwiGLU
    if (swiglu(d.gate_up)) return -1;
    // ---- down_proj + residual, then the next RMSNorm (next layer's input norm, or the final norm + last-row compaction)
    if (a8 && quant_rows_launch(e->act, T, c.intermediate_size, e->actq, e->acts, st)) return -1;
    if (partial(d.down, H, act_in, c.intermediate_size, &sk, a8 ? e->acts : nullptr)) return -1;
    if (resid_norm(&sk, is_last ? e->final_norm : e->dec[l + 1].in_norm, is_last)) return -1;
  }
  // ---- last-position lm_head + on-device decision (one row per segment)
  bf16* logits = d_last_logits ? static_cast<bf16*>(d_last_logits) : e->logits;
  if (lm_head_launch(e, e->xn_last, n_rows, logits, st)) return -1;
  if (decision_launch(logits, n_rows, c.vocab_size, interval_id, d_decisions ? static_cast<void*>(d_decisions) : e->decisions,
                      st))
    return -1;

  for (int i = 0; i < n_seqs; ++i) e->pool.commit(h_stream_ids[i], ends[i]);
  e->last_step_tokens = T;
  return 0;
}

}  // namespace

int vlo_step_ids(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, const int32_t* h_q_lens,
                 const int64_t* d_row_ids, const void* d_embeds, void* d_last_logits, vlo_decision* d_decisions,
                 int interval_id, void* cuda_stream) {
  return step_segments(e, n_seqs, h_stream_ids, nullptr, h_q_lens, d_row_ids, d_embeds, d_last_logits, d_decisions,
                       interval_id, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_step_segments(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, const int32_t* h_seg_counts,
                      const int32_t* h_seg_lens, const int64_t* d_row_ids, const void* d_embeds, void* d_seg_logits,
                      vlo_decision* d_decisions, int interval_id, void* cuda_stream) {
  VLO_CHECK(h_seg_counts != nullptr, "step_segments: null h_seg_counts");
  return step_segments(e, n_seqs, h_stream_ids, h_seg_counts, h_seg_lens, d_row_ids, d_embeds, d_seg_logits, d_decisions,
                       interval_id, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_prefill(vlo_engine* e, int stream_id, int n_tokens, const int64_t* d_row_ids, const void* d_embeds,
                void* d_last_logits, vlo_decision* d_decision, int interval_id, void* cuda_stream) {
  VLO_CHECK(e != nullptr && e->finalized && e->has_decoder, "decoder weights not loaded");
  VLO_CHECK(e->max_prefill > 0,
            "prefill: quantized layer matrices prefill only with quantized_prefill (vlo_set_quantized_prefill); without "
            "it long inputs run as max_step_tokens steps");
  VLO_CHECK(n_tokens > 0 && n_tokens <= e->max_prefill,
            "prefill: n_tokens must lie in [1, max_prefill_tokens] = [1, " + std::to_string(e->max_prefill) + "]");
  VLO_CHECK(d_embeds != nullptr, "prefill: null embeddings");
  return step_segments(e, 1, &stream_id, nullptr, &n_tokens, d_row_ids, d_embeds, d_last_logits, d_decision, interval_id,
                       static_cast<cudaStream_t>(cuda_stream), true);
}

int vlo_max_prefill_tokens(vlo_engine* e) { return e ? e->max_prefill : 0; }

int vlo_step(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, const int32_t* h_q_lens, const void* d_embeds,
             void* d_last_logits, vlo_decision* d_decisions, int interval_id, void* cuda_stream) {
  return vlo_step_ids(e, n_seqs, h_stream_ids, h_q_lens, nullptr, d_embeds, d_last_logits, d_decisions, interval_id,
                      cuda_stream);
}

int vlo_sample(vlo_engine* e, const void* d_logits, int n_rows, const vlo_sample_row* h_rows, const int32_t* h_penalty_ids,
               int n_penalty_ids, int32_t* d_out_ids, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && d_logits != nullptr && d_out_ids != nullptr, "sample: null argument");
  VLO_CHECK(n_rows > 0 && n_rows <= e->sample_rows,
            "sample: n_rows must lie in [1, max(max_streams, max_step_tokens)] = [1, " + std::to_string(e->sample_rows) + "]");
  VLO_CHECK(n_penalty_ids >= 0 && n_penalty_ids <= kSamplePenaltyIds,
            "sample: at most " + std::to_string(kSamplePenaltyIds) + " penalty ids per call");
  VLO_CHECK(n_penalty_ids == 0 || h_penalty_ids != nullptr, "sample: null penalty ids");
  VLO_CHECK((reinterpret_cast<uintptr_t>(d_logits) & 15) == 0, "sample: logits must be 16-byte aligned");
  if (sample_check_rows(h_rows, n_rows, n_penalty_ids)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  // parameters and ids through one pinned slot, one upload
  uint8_t* hs;
  int slot;
  if (stage_acquire(e, &hs, &slot)) return -1;
  std::memcpy(hs + e->sample_stage, h_rows, sizeof(SampleRow) * n_rows);
  if (n_penalty_ids) std::memcpy(hs + e->sample_stage + e->sample_ids, h_penalty_ids, sizeof(int) * n_penalty_ids);
  VLO_CUDA(cudaMemcpyAsync(e->sample_dev, hs + e->sample_stage, e->sample_ids + sizeof(int) * n_penalty_ids,
                           cudaMemcpyHostToDevice, st));
  if (stage_release(e, slot, st)) return -1;
  return sample_launch(d_logits, n_rows, e->cfg.vocab_size, e->sample_dev,
                       reinterpret_cast<const int*>(e->sample_dev + e->sample_ids), d_out_ids, nullptr, st);
}

// ------------------------------------------------------------------------------ kernel-class micro loops
// Back-to-back launches of ONE kernel class on the engine's real buffers and shapes (all layers, so the
// working set is far larger than L2).  bench.py brackets the whole loop with one CUDA-event pair: the average
// per launch then carries no per-launch event overhead and includes the PDL overlap the step really has.
int vlo_bench_attn(vlo_engine* e, int n_seqs, const int32_t* h_stream_ids, int n_tok, int iters, int skip_merge,
                   double* h_algo_bytes_per_launch, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->finalized && e->has_decoder, "decoder weights not loaded");
  const vlo_config& c = e->cfg;
  VLO_CHECK(n_seqs > 0 && n_seqs <= c.max_streams && n_tok > 0 && n_seqs * n_tok <= c.max_step_tokens, "bench_attn: sizes");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  for (int i = 0; i < n_seqs; ++i) {
    if (check_stream(e, h_stream_ids[i])) return -1;
    VLO_CHECK(e->pool.len(h_stream_ids[i]) >= n_tok, "bench_attn: need kv_len >= n_tok");
  }
  // the streams' page tables go up in the same region and memcpy as a step's
  uint8_t* hs;
  int slot;
  if (stage_acquire(e, &hs, &slot)) return -1;
  std::vector<int> pt0(n_seqs);
  const int n_pt = stage_page_tables(e, hs, n_seqs, h_stream_ids, pt0.data());
  std::vector<AttnSeq> seqs(n_seqs);
  for (int i = 0; i < n_seqs; ++i) seqs[i] = AttnSeq{i * n_tok, n_tok, e->pool.len(h_stream_ids[i]), pt0[i]};
  VLO_CUDA(cudaMemcpyAsync(e->meta_dev + e->meta.pt, hs + e->meta.pt, sizeof(int) * n_pt, cudaMemcpyHostToDevice, st));
  AttnPlan plan{};
  if (attn_plan(&plan, e->attn_ws, hs + e->meta.bytes, seqs.data(), n_seqs, n_seqs * n_tok, c.num_heads, c.num_kv_heads,
                c.head_dim, st))
    return -1;
  if (stage_release(e, slot, st)) return -1;
  plan.skip_merge = skip_merge;
  if (h_algo_bytes_per_launch) *h_algo_bytes_per_launch = plan.algo_bytes;
  for (int it = 0; it < iters; ++it)
    for (int l = 0; l < c.num_layers; ++l)
      if (attn_layer(e, plan, l, st)) return -1;
  return 0;
}

int vlo_bench_gemm(vlo_engine* e, int n_tok, int iters, double* h_algo_bytes_per_iter, int* h_launches_per_iter,
                   void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->finalized && e->has_decoder, "decoder weights not loaded");
  const vlo_config& c = e->cfg;
  VLO_CHECK(n_tok > 0 && n_tok <= c.max_step_tokens, "bench_gemm: n_tok out of range");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const int H = c.hidden_size, I = c.intermediate_size, A = c.num_heads * c.head_dim;
  double bytes = 0.0;
  // fp8_act: the W8A8 GEMMs on the e4m3 activation copies with their token scales
  const bool a8 = e->fp8_act;
  const void* xn = a8 ? static_cast<const void*>(e->xq) : e->xn;
  const void* attn = a8 ? static_cast<const void*>(e->aq) : e->attn_out;
  const void* act = a8 ? static_cast<const void*>(e->actq) : e->act;
  auto gemm = [&](const WeightOperand& w, int n_out, const void* x, const float* x_scale, int k) -> int {
    GemmWsPlan sk{};
    return gemm_partial(w, n_out, x, a8 ? x_scale : nullptr, n_tok, k, e->part, e->part_elems, WS_TILE_FIT, &sk, st);
  };
  for (int it = 0; it < iters; ++it)
    for (int l = 0; l < c.num_layers; ++l) {
      const DecLayer& d = e->dec[l];
      if (gemm(d.qkv, e->qkv_width, xn, e->xs, H)) return -1;
      if (gemm(d.o, H, attn, e->as, A)) return -1;
      if (gemm(d.gate_up, 2 * I, xn, e->xs, H)) return -1;
      if (gemm(d.down, H, act, e->acts, I)) return -1;
      if (it == 0)
        bytes += ws_in_bytes(e->layer_fmt, e->qkv_width, n_tok, H) + ws_in_bytes(e->layer_fmt, H, n_tok, A) +
                 ws_in_bytes(e->layer_fmt, 2 * I, n_tok, H) + ws_in_bytes(e->layer_fmt, H, n_tok, I);
    }
  if (h_algo_bytes_per_iter) *h_algo_bytes_per_iter = bytes;
  if (h_launches_per_iter) *h_launches_per_iter = 4 * c.num_layers;
  return 0;
}

int vlo_last_step_hidden(vlo_engine* e, void* d_hidden, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->last_step_tokens > 0, "no decoder step has run");
  VLO_CUDA(cudaMemcpyAsync(d_hidden, e->xn, static_cast<size_t>(e->last_step_tokens) * e->cfg.hidden_size * sizeof(bf16),
                           cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(cuda_stream)));
  return 0;
}

int vlo_last_step_logits(vlo_engine* e, void* d_logits, void* cuda_stream) {
  DevGuard dev_guard(e);
  VLO_CHECK(e != nullptr && e->last_step_tokens > 0, "no decoder step has run");
  return lm_head_launch(e, e->xn, e->last_step_tokens, d_logits, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_vocab_format(vlo_engine* e) { return e != nullptr && e->embed.w != nullptr ? e->vocab_fmt : -1; }

}  // extern "C"
