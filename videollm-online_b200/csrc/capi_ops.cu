// C-ABI: library-level and kernel-level entry points (see include/vlo_b200.h).
#include "vlo_b200.h"

#include <algorithm>
#include <vector>

#include "common.h"
#include "gemm.cuh"
#include "kv_pages.h"

using namespace vlo;

namespace {

// Plan one sequence of n_tok queries over kv_len keys and upload the plan into d_ws.  h_identity_pt: also upload an
// identity page table (the contiguous [n_kv_heads][kv_stride][128] layout, one "page" per 64-key block) behind the
// plan's workspace and return its device address in *d_pt.  The upload is synchronised: the staging is pageable.
// n_segs > 1: the n_tok rows are segments of h_seg_lens[] rows, planned as by a segmented decoder step.
int op_attn_plan(AttnPlan* plan, void* d_ws, int n_tok, int n_heads, int n_kv_heads, int head_dim, int kv_len,
                 bool identity_pt, const int** d_pt, cudaStream_t st, int n_segs = 0, const int* h_seg_lens = nullptr) {
  VLO_CHECK(n_tok > 0 && kv_len >= n_tok, "attn: need 0 < n_tok <= kv_len");
  AttnSeq s{};
  s.q_tok0 = 0;
  s.q_len = n_tok;
  s.kv_len = kv_len;
  s.pt0 = 0;
  s.n_segs = n_segs;
  s.seg_lens = h_seg_lens;
  const size_t plan_stage = attn_stage_bytes(n_tok, 1, n_heads, n_kv_heads);
  const int nblk = kv_pages_for(kv_len);
  static thread_local std::vector<uint8_t> stage;
  stage.resize(plan_stage + sizeof(int) * nblk);
  if (attn_plan(plan, d_ws, stage.data(), &s, 1, n_tok, n_heads, n_kv_heads, head_dim, st)) return -1;
  if (identity_pt) {
    int* h_pt = reinterpret_cast<int*>(stage.data() + plan_stage);
    for (int b = 0; b < nblk; ++b) h_pt[b] = b;
    int* pt = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(d_ws) + attn_ws_bytes(n_tok, 1, n_heads, n_kv_heads));
    VLO_CUDA(cudaMemcpyAsync(pt, h_pt, sizeof(int) * nblk, cudaMemcpyHostToDevice, st));
    *d_pt = pt;
  }
  VLO_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// The stream-K plan of the bf16 partial GEMM that produced a fix-up kernel's planes: the planning query of
// gemm_ws_launch (mode 0) for `width` output features, T token rows, k and n_ctas.
int op_fix_plan(int width, int T, int k, int n_ctas, SkInfo* sk) {
  VLO_CHECK(T > 0 && T <= 128, "fix-up kernels: 1..128 token rows (one token tile)");
  GemmWsCall c{};
  c.w.fmt = FMT_BF16;
  c.mode = 0;
  c.rows_w = width;
  c.rows_x = T;
  c.k = k;
  c.n_ctas = n_ctas;
  GemmWsPlan plan{};
  if (gemm_ws_launch(c, nullptr, &plan)) return -1;
  VLO_CHECK(plan.planes <= kFixMaxPlanes, "the plan needs " + std::to_string(plan.planes) +
                                               " partial planes, more than the fix-up kernels unroll");
  *sk = plan.sk;
  return 0;
}

__global__ void tanh_approx_kernel(const float* x, float* y, long long n) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    y[i] = tanh_approx(x[i]);
}

// Device scratch of a synchronous kernel-level entry point, freed on every return path.
// gemm_ws_launch mode 0 of weights w into the caller-sized planes d_out (null: plan only) on the token tile it picks
int op_gemm_ws_partials(const WeightOperand& w, int rows_w, const void* d_x, const float* d_xscale, int rows_x, int k,
                        float* d_out, long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream) {
  GemmWsCall c{};
  c.w = w;
  c.mode = 0;
  c.rows_w = rows_w;
  c.x = d_x;
  c.a_scale = d_xscale;
  c.rows_x = rows_x;
  c.k = k;
  c.out = d_out;
  c.out_elems = SIZE_MAX;  // the caller sizes d_out from the planning query
  c.ld_out = rows_w;
  c.plane_stride = plane_stride;
  c.n_ctas = n_ctas;
  GemmWsPlan plan{};
  if (d_out != nullptr && pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  const int rc = gemm_ws_launch(c, static_cast<cudaStream_t>(cuda_stream), &plan);
  if (rc == 0 && h_max_planes) *h_max_planes = plan.planes;
  return rc;
}

struct OpScratch {
  void* p = nullptr;
  ~OpScratch() {
    if (p) cudaFree(p);
  }
};

// ---- the PDL-contract probe and canary (vlo_op_pdl_arm, vlo_op_pdl_canary): test hooks, not used by the engine
struct PdlProbe {
  int mode = 0;   // 0: not armed
  uint8_t* dst = nullptr;
  uint8_t* src = nullptr;
  long long bytes = 0, stride = 0, spin_ns = 0;
  int n_chunks = 0;
};
PdlProbe g_probe;
constexpr int kProbeCtas = 4;   // a few CTAs: the kernel under test becomes resident on the other SMs
constexpr long long kProbeMaxSpinNs = 2000000;
__device__ unsigned long long g_probes_done;

// Lets its dependents launch, spins on the global timer (nothing else is waited for), then copies the chunks src -> dst,
// or late_read: exchanges them.
__global__ void __launch_bounds__(256) pdl_probe_kernel(int late_read, uint8_t* dst, uint8_t* src, long long bytes,
                                                        int n_chunks, long long stride, long long spin_ns) {
  pdl_trigger();
  const unsigned long long t0 = globaltimer_ns();
  while (globaltimer_ns() - t0 < static_cast<unsigned long long>(spin_ns)) {
  }
  const long long tid = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long nth = static_cast<long long>(gridDim.x) * blockDim.x;
  const bool vec = ((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src) | bytes | stride) & 15) == 0;
  for (int c = 0; c < n_chunks; ++c) {
    uint8_t* d = dst + c * stride;
    uint8_t* s = src + c * stride;
    if (vec) {
      uint4* d4 = reinterpret_cast<uint4*>(d);
      uint4* s4 = reinterpret_cast<uint4*>(s);
      for (long long i = tid; i < bytes / 16; i += nth) {
        const uint4 v = s4[i];
        if (late_read) s4[i] = d4[i];
        d4[i] = v;
      }
    } else {
      for (long long i = tid; i < bytes; i += nth) {
        const uint8_t v = s[i];
        if (late_read) s[i] = d[i];
        d[i] = v;
      }
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&g_probes_done, 1ull);
}

__global__ void __launch_bounds__(256) pdl_canary_kernel(int variant, const uint32_t* src, uint32_t* dst, int n) {
  pdl_trigger();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t early = 0;
  if (i < n && variant == 1) early = src[i];   // seeded read violation
  if (i < n && variant == 2) dst[i] = src[i];  // seeded write violation
  pdl_wait();
  if (i < n && variant == 0) dst[i] = src[i];
  if (i < n && variant == 1) dst[i] = early;
}

}  // namespace

int vlo::pdl_probe_fire(cudaStream_t st) {
  if (g_probe.mode == 0) return 0;
  const PdlProbe p = g_probe;
  g_probe = PdlProbe{};
  pdl_probe_kernel<<<kProbeCtas, 256, 0, st>>>(p.mode == VLO_PDL_LATE_READ, p.dst, p.src, p.bytes, p.n_chunks, p.stride,
                                                p.spin_ns);
  VLO_LAUNCH_CHECK();
  return 0;
}

extern "C" {

const char* vlo_last_error(void) { return last_error(); }

long long vlo_launch_count(void) { return launch_count(); }

int vlo_profile_enable(int on) {
  prof_enable(on != 0);
  return 0;
}
int vlo_profile_read(double* ms, long long* launches, double* algo_bytes, int n_classes) {
  return prof_read(ms, launches, algo_bytes, n_classes);
}

int vlo_device_supported(int device) {
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return (prop.major == 9 && prop.minor == 0) ? 1 : 0;
}

int vlo_op_gemm(int epi, int act, const void* d_x, int rows_x, const void* d_w, int rows_w, int k, void* d_out, int ld_out,
                const float* d_bias, const float* d_pos, int pos_rows, int bn, void* cuda_stream) {
  GemmCall c{};
  c.epi = epi;
  c.act = act;
  c.a = d_x;
  c.rows_a = rows_x;
  c.b = d_w;
  c.rows_b = rows_w;
  c.k = k;
  c.out = d_out;
  c.ld_out = ld_out;
  c.bias = d_bias;
  c.pos = d_pos;
  c.pos_rows = pos_rows;
  c.bn = bn > 0 ? bn : 128;
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_launch(c, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_gemm_ws(int fmt, int mode, const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out,
                   int ld_out, long long plane_stride, const float* d_bias, int act, int n_ctas, int bn, int* h_max_planes,
                   void* cuda_stream) {
  int32_t plan[3] = {0, 0, 0};
  const int rc = vlo_op_gemm_ws_tiled(fmt, mode, d_w, rows_w, d_x, rows_x, k, d_out, ld_out, plane_stride, d_bias, act,
                                      n_ctas, bn, WS_TILE_FIT, plan, cuda_stream);
  if (rc == 0 && h_max_planes) *h_max_planes = plan[2];
  return rc;
}

int vlo_op_gemm_ws_tiled(int fmt, int mode, const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out,
                         int ld_out, long long plane_stride, const float* d_bias, int act, int n_ctas, int bn, int tiling,
                         int32_t* h_plan, void* cuda_stream) {
  VLO_CHECK(tiling == WS_TILE_FIT || tiling == WS_TILE_TRUNK || tiling == WS_TILE_BESIDE_DECODER, "gemm_ws: unknown tiling");
  GemmWsCall c{};
  c.w = WeightOperand{fmt, d_w, nullptr, nullptr};
  c.mode = mode;
  c.rows_w = rows_w;
  c.x = d_x;
  c.rows_x = rows_x;
  c.k = k;
  c.out = d_out;
  c.out_elems = SIZE_MAX;  // the caller sizes d_out from the planning query
  c.ld_out = ld_out;
  c.plane_stride = plane_stride;
  c.bias = d_bias;
  c.act = act;
  c.n_ctas = n_ctas;
  c.bn = bn;
  c.tiling = tiling;
  GemmWsPlan plan{};
  if (d_out != nullptr && pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  const int rc = gemm_ws_launch(c, static_cast<cudaStream_t>(cuda_stream), &plan);
  if (rc == 0 && h_plan) {
    h_plan[0] = plan.bn;
    h_plan[1] = plan.x_tiles;
    h_plan[2] = plan.planes;
  }
  return rc;
}

int vlo_op_gemm_ws_f8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x, int rows_x, int k, float* d_out,
                      long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream) {
  VLO_CHECK(d_out == nullptr || d_scale != nullptr, "gemm_ws_f8: null row scales");
  return op_gemm_ws_partials(WeightOperand{FMT_E4M3, d_w8, d_scale, nullptr}, rows_w, d_x, nullptr, rows_x, k, d_out,
                             plane_stride, n_ctas, h_max_planes, cuda_stream);
}

int vlo_op_gemm_ws_i4(const void* d_w4, const void* d_gscale, int rows_w, const void* d_x, int rows_x, int k, float* d_out,
                      long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream) {
  VLO_CHECK(d_out == nullptr || d_gscale != nullptr, "gemm_ws_i4: null group scales");
  return op_gemm_ws_partials(WeightOperand{FMT_I4, d_w4, nullptr, static_cast<const uint16_t*>(d_gscale)}, rows_w, d_x,
                             nullptr, rows_x, k, d_out, plane_stride, n_ctas, h_max_planes, cuda_stream);
}

int vlo_op_gemm_ws_tiles_q(int fmt, const void* d_w, const void* d_scale, int rows_w, const void* d_x, int rows_x, int k,
                           void* d_out, int ld_out, int n_ctas, int32_t* h_plan, void* cuda_stream) {
  VLO_CHECK(fmt == FMT_E4M3 || fmt == FMT_I4, "gemm_ws_tiles_q: fmt 2 (e4m3 weights, fp32 row scales) or 4 (int4 weights, "
                                              "bf16 group scales)");
  VLO_CHECK(d_out == nullptr || d_scale != nullptr, "gemm_ws_tiles_q: null scales");
  GemmWsCall c{};
  c.w = fmt == FMT_E4M3 ? WeightOperand{fmt, d_w, static_cast<const float*>(d_scale), nullptr}
                        : WeightOperand{fmt, d_w, nullptr, static_cast<const uint16_t*>(d_scale)};
  c.mode = 1;
  c.rows_w = rows_w;
  c.x = d_x;
  c.rows_x = rows_x;
  c.k = k;
  c.out = d_out;
  c.ld_out = ld_out;
  c.n_ctas = n_ctas;
  GemmWsPlan plan{};
  if (d_out != nullptr && pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  const int rc = gemm_ws_launch(c, static_cast<cudaStream_t>(cuda_stream), &plan);
  if (rc == 0 && h_plan) {
    h_plan[0] = plan.bn;
    h_plan[1] = plan.x_tiles;
    h_plan[2] = plan.sk.G;
  }
  return rc;
}

int vlo_op_embed_rows_q(int fmt, const void* d_table, const void* d_scale, int vocab, int hidden, const int64_t* d_ids, int n,
                        void* d_out, void* cuda_stream) {
  VLO_CHECK(fmt == FMT_BF16 || fmt == FMT_E4M3 || fmt == FMT_I4, "embed_rows_q: fmt 1 (bf16), 2 (e4m3) or 4 (int4)");
  VLO_CHECK(d_table != nullptr && d_ids != nullptr && d_out != nullptr && (fmt == FMT_BF16 || d_scale != nullptr),
            "embed_rows_q: null argument");
  VLO_CHECK(n > 0 && vocab > 0 && hidden > 0 && hidden % 128 == 0, "embed_rows_q: n, vocab > 0, hidden a multiple of 128");
  const WeightOperand t = fmt == FMT_E4M3 ? WeightOperand{fmt, d_table, static_cast<const float*>(d_scale), nullptr}
                          : fmt == FMT_I4 ? WeightOperand{fmt, d_table, nullptr, static_cast<const uint16_t*>(d_scale)}
                                          : WeightOperand{fmt, d_table, nullptr, nullptr};
  return embed_rows_launch(t, reinterpret_cast<const long long*>(d_ids), n, vocab, hidden, d_out,
                           static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_gemm_ws_a8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x8, const float* d_xscale, int rows_x,
                      int k, float* d_out, long long plane_stride, int n_ctas, int* h_max_planes, void* cuda_stream) {
  VLO_CHECK(d_out == nullptr || (d_scale != nullptr && d_xscale != nullptr), "gemm_ws_a8: null row or token scales");
  return op_gemm_ws_partials(WeightOperand{FMT_E4M3_A8, d_w8, d_scale, nullptr}, rows_w, d_x8, d_xscale, rows_x, k, d_out,
                             plane_stride, n_ctas, h_max_planes, cuda_stream);
}

int vlo_op_gemm_vit(const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out, int ld_out,
                    const float* d_bias, int act, int n_ctas, void* cuda_stream) {
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_vit_launch(d_x, rows_x, d_w, rows_w, k, d_out, ld_out, d_bias, act, n_ctas, static_cast<cudaStream_t>(cuda_stream));
}

int64_t vlo_op_attn_ws_bytes(int n_tok, int n_heads, int head_dim, int kv_len) {
  (void)head_dim;
  // n_kv_heads is not part of this query: bound it by n_heads (G = 1 is the worst case); the identity page table of
  // the contiguous layout follows the plan's workspace
  return 2 * static_cast<int64_t>(attn_ws_bytes(n_tok, 1, n_heads, n_heads)) +
         static_cast<int64_t>(align256(sizeof(int) * kv_pages_for(kv_len)));
}

int vlo_op_attn_kvappend(const void* d_q, const void* d_k, const void* d_v, void* d_out, float* d_ws, int n_tok,
                         int n_heads, int n_kv_heads, int head_dim, int kv_len, long long kv_stride,
                         void* cuda_stream) {
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  AttnPlan plan{};
  const int* pt = nullptr;
  if (op_attn_plan(&plan, d_ws, n_tok, n_heads, n_kv_heads, head_dim, kv_len, true, &pt, st)) return -1;
  if (pdl_probe_fire(st)) return -1;
  if (attn_run(plan, d_q, d_k, d_v, static_cast<long long>(n_kv_heads) * kv_stride, pt, kKvPageTokens, kv_stride, d_out,
               n_heads, n_kv_heads, head_dim, st))
    return -1;
  VLO_CUDA(cudaStreamSynchronize(st));  // the plan lives in a per-thread buffer: finish before it can be reused
  return 0;
}

int vlo_op_attn_kvappend_paged(const void* d_q, const void* d_k_pool, const void* d_v_pool, const int32_t* d_page_table,
                               int n_pages, void* d_out, float* d_ws, int n_tok, int n_heads, int n_kv_heads,
                               int head_dim, int kv_len, void* cuda_stream) {
  VLO_CHECK(n_pages > 0 && n_kv_heads > 0, "attn_paged: sizes");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  AttnPlan plan{};
  if (op_attn_plan(&plan, d_ws, n_tok, n_heads, n_kv_heads, head_dim, kv_len, false, nullptr, st)) return -1;
  if (pdl_probe_fire(st)) return -1;
  const long long page_rows = static_cast<long long>(n_kv_heads) * kKvPageTokens;
  if (attn_run(plan, d_q, d_k_pool, d_v_pool, n_pages * page_rows, d_page_table, page_rows, kKvPageTokens, d_out, n_heads,
               n_kv_heads, head_dim, st))
    return -1;
  VLO_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int vlo_op_attn_kvappend_segments(const void* d_q, const void* d_k_pool, const void* d_v_pool, const int32_t* d_page_table,
                                  int n_pages, void* d_out, int n_segs, const int32_t* h_seg_lens, int n_heads,
                                  int n_kv_heads, int head_dim, int kv_len, void* cuda_stream) {
  VLO_CHECK(n_pages > 0 && n_kv_heads > 0 && n_heads > 0 && n_heads % n_kv_heads == 0, "attn_segments: sizes");
  VLO_CHECK(n_segs > 0 && h_seg_lens != nullptr, "attn_segments: need at least one segment");
  int n_tok = 0;
  for (int j = 0; j < n_segs; ++j) {
    VLO_CHECK(h_seg_lens[j] > 0, "attn_segments: segment lengths must be positive");
    n_tok += h_seg_lens[j];
  }
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  OpScratch ws;  // sized for the plan's segments: the caller's query of vlo_op_attn_ws_bytes does not know them
  VLO_CUDA(cudaMalloc(&ws.p, attn_ws_bytes(n_tok, 1, n_heads, n_kv_heads)));
  AttnPlan plan{};
  if (op_attn_plan(&plan, ws.p, n_tok, n_heads, n_kv_heads, head_dim, kv_len, false, nullptr, st, n_segs, h_seg_lens))
    return -1;
  if (pdl_probe_fire(st)) return -1;
  const long long page_rows = static_cast<long long>(n_kv_heads) * kKvPageTokens;
  if (attn_run(plan, d_q, d_k_pool, d_v_pool, n_pages * page_rows, d_page_table, page_rows, kKvPageTokens, d_out, n_heads,
               n_kv_heads, head_dim, st))
    return -1;
  VLO_CUDA(cudaStreamSynchronize(st));  // the workspace is freed on return
  return 0;
}

int vlo_op_attn_plan_counts(int n_segs, const int32_t* h_seg_lens, int n_heads, int n_kv_heads, int head_dim, int kv_len,
                            int32_t* h_counts) {
  VLO_CHECK(n_kv_heads > 0 && n_heads > 0 && n_heads % n_kv_heads == 0, "attn_plan_counts: sizes");
  VLO_CHECK(n_segs > 0 && h_seg_lens != nullptr && h_counts != nullptr, "attn_plan_counts: null argument");
  int n_tok = 0;
  for (int j = 0; j < n_segs; ++j) {
    VLO_CHECK(h_seg_lens[j] > 0, "attn_plan_counts: segment lengths must be positive");
    n_tok += h_seg_lens[j];
  }
  AttnSeq s{0, n_tok, kv_len, 0, n_segs, h_seg_lens};
  AttnPlan plan{};
  if (attn_plan(&plan, nullptr, nullptr, &s, 1, n_tok, n_heads, n_kv_heads, head_dim, nullptr)) return -1;
  h_counts[0] = plan.n_items;
  h_counts[1] = plan.n_clusters;
  h_counts[2] = plan.n_packs;
  h_counts[3] = plan.n_packed_items;
  return 0;
}

int vlo_op_vit_attn(const void* d_qkv, void* d_out, int n_frames, int n_tok, int hidden, void* cuda_stream) {
  VLO_CHECK(d_qkv != nullptr && d_out != nullptr, "vit_attn: null argument");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return vit_attn_launch(d_qkv, d_out, n_frames, n_tok, hidden, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_probe_attn(const void* d_kv, const float* d_q, void* d_out, int n_frames, int n_tok, int hidden,
                      void* cuda_stream) {
  VLO_CHECK(d_kv != nullptr && d_q != nullptr && d_out != nullptr, "probe_attn: null argument");
  return probe_attn_launch(d_kv, d_q, d_out, n_frames, n_tok, hidden, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_vit_tiling(int n_frames, int n_patches, int hidden, int mlp, int32_t* h_out) {
  VLO_CHECK(n_frames > 0 && n_patches > 0 && hidden > 0 && mlp > 0 && h_out != nullptr, "vit_tiling: sizes");
  const int rows = n_frames * n_patches;
  const bool beside = vit_beside_decoder(n_frames);
  // the planning query of each gemm_ws_launch vlo_vit_encode makes (mode, output features, k, tiling)
  auto query = [&](int mode, int n_out, int k, int tiling, int tok_rows, GemmWsPlan* plan) -> int {
    GemmWsCall c{};
    c.w.fmt = FMT_F16;
    c.mode = mode;
    c.rows_w = n_out;
    c.rows_x = tok_rows;
    c.k = k;
    c.tiling = tiling;
    return gemm_ws_launch(c, nullptr, plan);
  };
  GemmWsPlan qkv{}, fc1{}, out{}, fc2{}, head{};
  const int part_tiling = beside ? WS_TILE_BESIDE_DECODER : WS_TILE_TRUNK;
  if (!beside && (query(1, 3 * hidden, hidden, WS_TILE_TRUNK, rows, &qkv) || query(1, mlp, hidden, WS_TILE_TRUNK, rows, &fc1)))
    return -1;
  if (query(0, hidden, hidden, part_tiling, rows, &out) || query(0, hidden, mlp, part_tiling, rows, &fc2) ||
      query(1, hidden, hidden, WS_TILE_FIT, n_frames, &head))
    return -1;
  h_out[0] = beside ? 0 : WS_TILE_TRUNK;
  h_out[1] = beside ? kGemmBM : qkv.bn;
  h_out[2] = beside ? kGemmBM : fc1.bn;
  h_out[3] = part_tiling;
  h_out[4] = out.bn;
  h_out[5] = out.planes;
  h_out[6] = fc2.bn;
  h_out[7] = fc2.planes;
  h_out[8] = vit_bn(rows, hidden);
  h_out[9] = vit_bn(rows, 2 * hidden);
  h_out[10] = head.bn;
  return 0;
}

int vlo_op_tanh_approx(const float* d_x, float* d_y, long long n, void* cuda_stream) {
  VLO_CHECK(d_x != nullptr && d_y != nullptr && n > 0, "tanh_approx: null argument or n <= 0");
  tanh_approx_kernel<<<static_cast<unsigned>(std::min<long long>((n + 255) / 256, 4096)), 256, 0,
                       static_cast<cudaStream_t>(cuda_stream)>>>(d_x, d_y, n);
  VLO_LAUNCH_CHECK();
  return 0;
}

int vlo_op_patchify(const uint8_t* d_frames, int n_frames, int image_size, int patch_size, void* d_out, void* cuda_stream) {
  VLO_CHECK(d_frames != nullptr && d_out != nullptr, "patchify: null argument");
  VLO_CHECK(n_frames > 0 && patch_size > 0 && patch_size % 8 == 0 && image_size >= patch_size && image_size % patch_size == 0,
            "patchify: n_frames > 0, patch_size a multiple of 8 dividing image_size");
  VLO_CHECK((reinterpret_cast<uintptr_t>(d_frames) & 7) == 0 && (reinterpret_cast<uintptr_t>(d_out) & 15) == 0,
            "patchify: frames 8-byte and patches 16-byte aligned");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return patchify_launch(d_frames, d_out, n_frames, image_size, patch_size, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_vit_layernorm(const void* d_in, int in_is_f16, int rows, int C, const float* d_w, const float* d_b, void* d_out16,
                         float* d_out32, float eps, void* cuda_stream) {
  VLO_CHECK(d_in != nullptr && d_w != nullptr && d_b != nullptr && (d_out16 != nullptr || d_out32 != nullptr),
            "vit_layernorm: null argument");
  // the row is staged in shared memory without an opt-in beyond the default 48 KB
  VLO_CHECK(rows > 0 && C > 0 && C * sizeof(float) <= 48 * 1024, "vit_layernorm: rows > 0, 0 < C <= 12288");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return vit_layernorm_launch(d_in, in_is_f16 != 0, rows, C, d_w, d_b, d_out16, d_out32, eps,
                              static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_vit_fix_ln(const float* d_part, int rows, int C, int k, int bn, int n_ctas, const float* d_bias, float* d_h,
                      const float* d_ln_w, const float* d_ln_b, void* d_out16, float* d_out32, float eps, void* cuda_stream) {
  VLO_CHECK(d_part != nullptr && d_bias != nullptr && d_h != nullptr && d_ln_w != nullptr && d_ln_b != nullptr,
            "vit_fix_ln: null argument");
  VLO_CHECK(rows > 0 && C > 0 && C % 4 == 0 && C * sizeof(float) <= 48 * 1024, "vit_fix_ln: rows > 0, C a multiple of 4, <= 12288");
  VLO_CHECK(bn > 0, "vit_fix_ln: the producer's token tile bn must be given");
  auto aligned = [](const void* q, uintptr_t a) { return (reinterpret_cast<uintptr_t>(q) & (a - 1)) == 0; };
  // the kernel moves 4 channels per access: float4 for the fp32 rows and vectors, uint2 for out16
  VLO_CHECK(aligned(d_part, 16) && aligned(d_h, 16) && aligned(d_bias, 16) && aligned(d_ln_w, 16) && aligned(d_ln_b, 16) &&
                aligned(d_out32, 16) && aligned(d_out16, 8),
            "vit_fix_ln: fp32 arrays 16-byte and out16 8-byte aligned");
  GemmWsCall c{};
  c.w.fmt = FMT_F16;
  c.mode = 0;
  c.rows_w = C;
  c.rows_x = rows;
  c.k = k;
  c.n_ctas = n_ctas;
  c.bn = bn;
  GemmWsPlan plan{};
  if (gemm_ws_launch(c, nullptr, &plan)) return -1;
  VLO_CHECK(plan.planes <= kFixMaxPlanes, "the plan needs " + std::to_string(plan.planes) +
                                              " partial planes, more than the fix-up kernels unroll");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return vit_fix_ln_launch(d_part, plan, rows, C, d_bias, d_h, d_ln_w, d_ln_b, d_out16, d_out32, eps,
                           static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_vit_pool(const float* d_in, int n_frames, int grid, int C, int ph, int pw, int n_tok, int tok_off, float* d_tokens,
                    void* cuda_stream) {
  VLO_CHECK(d_in != nullptr && d_tokens != nullptr, "vit_pool: null argument");
  VLO_CHECK(n_frames > 0 && grid > 0 && C > 0 && ph > 0 && ph <= grid && pw > 0 && pw <= grid,
            "vit_pool: sizes (1 <= ph, pw <= grid)");
  VLO_CHECK(tok_off >= 0 && tok_off + ph * pw <= n_tok, "vit_pool: the pooled cells must fit in n_tok token slots");
  return pool_launch(d_in, d_tokens, n_frames, grid, C, ph, pw, n_tok, tok_off, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_cls_residual(const void* d_resid16, const void* d_mlp16, float* d_tokens, int n_frames, int C, int n_tok,
                        void* cuda_stream) {
  VLO_CHECK(d_resid16 != nullptr && d_mlp16 != nullptr && d_tokens != nullptr, "cls_residual: null argument");
  VLO_CHECK(n_frames > 0 && C > 0 && n_tok > 0, "cls_residual: sizes");
  return cls_residual_launch(d_resid16, d_mlp16, d_tokens, n_frames, C, n_tok, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_resid_rmsnorm(const float* d_part, int k, int n_ctas, void* d_h, const void* d_w, void* d_xn, void* d_xn_last,
                         const int32_t* d_last_index, int T, int H, float eps, void* cuda_stream) {
  // the row is staged in shared memory without an opt-in beyond the default 48 KB
  VLO_CHECK(T > 0 && H > 0 && H % 4 == 0 && H * sizeof(float) <= 48 * 1024, "resid_rmsnorm: H a multiple of 4, <= 12288");
  VLO_CHECK(d_last_index == nullptr || d_xn_last != nullptr, "resid_rmsnorm: last_index without xn_last");
  SkInfo sk{};
  if (d_part != nullptr && op_fix_plan(H, T, k, n_ctas, &sk)) return -1;
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return resid_rmsnorm_launch(d_part, &sk, d_h, d_w, d_xn, d_xn_last, d_last_index, T, H, eps,
                              static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_resid_rmsnorm_q8(const float* d_part, int k, int n_ctas, void* d_h, const void* d_w, void* d_xn, void* d_xn_last,
                            const int32_t* d_last_index, void* d_xq, float* d_xs, int T, int H, float eps, void* cuda_stream) {
  VLO_CHECK(T > 0 && H > 0 && H % 4 == 0 && H * sizeof(float) <= 48 * 1024, "resid_rmsnorm_q8: H a multiple of 4, <= 12288");
  VLO_CHECK(d_last_index == nullptr || d_xn_last != nullptr, "resid_rmsnorm_q8: last_index without xn_last");
  VLO_CHECK(d_xn != nullptr && d_xq != nullptr && d_xs != nullptr, "resid_rmsnorm_q8: null xn, xq or xs");
  SkInfo sk{};
  if (d_part != nullptr && op_fix_plan(H, T, k, n_ctas, &sk)) return -1;
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return resid_rmsnorm_q8_launch(d_part, &sk, d_h, d_w, d_xn, d_xn_last, d_last_index, static_cast<uint8_t*>(d_xq), d_xs, T,
                                 H, eps, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_quant_rows_e4m3(const void* d_x, int T, int K, void* d_q, float* d_s, void* cuda_stream) {
  VLO_CHECK(d_x != nullptr && d_q != nullptr && d_s != nullptr, "quant_rows_e4m3: null argument");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return quant_rows_launch(d_x, T, K, static_cast<uint8_t*>(d_q), d_s, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_qkv_rope_append(const float* d_part, int k, int n_ctas, const void* d_cos, const void* d_sin, int n_rope_pos,
                           const int32_t* h_tok_pos, const int64_t* h_tok_kvrow, int kv_head_stride, void* d_q, void* d_k,
                           void* d_v, int T, int n_heads, int n_kv_heads, void* cuda_stream) {
  VLO_CHECK(d_part != nullptr && n_heads > 0 && n_kv_heads > 0 && n_heads % n_kv_heads == 0, "qkv_rope_append: sizes");
  SkInfo sk{};
  if (op_fix_plan((n_heads + 2 * n_kv_heads) * 128, T, k, n_ctas, &sk)) return -1;
  for (int t = 0; t < T; ++t) {
    VLO_CHECK(h_tok_pos[t] >= 0 && h_tok_pos[t] < n_rope_pos,
              "qkv_rope_append: position " + std::to_string(h_tok_pos[t]) + " outside the RoPE tables");
    VLO_CHECK(h_tok_kvrow[t] >= 0, "qkv_rope_append: negative cache row");
  }
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  OpScratch tables;
  const size_t pos_bytes = align256(sizeof(int) * T);
  VLO_CUDA(cudaMalloc(&tables.p, pos_bytes + sizeof(long long) * T));
  int* d_pos = static_cast<int*>(tables.p);
  long long* d_kvrow = reinterpret_cast<long long*>(static_cast<uint8_t*>(tables.p) + pos_bytes);
  VLO_CUDA(cudaMemcpyAsync(d_pos, h_tok_pos, sizeof(int) * T, cudaMemcpyHostToDevice, st));
  VLO_CUDA(cudaMemcpyAsync(d_kvrow, h_tok_kvrow, sizeof(long long) * T, cudaMemcpyHostToDevice, st));
  if (pdl_probe_fire(st)) return -1;  // after the table uploads, which serialise the stream
  if (qkv_rope_launch(d_part, sk, d_cos, d_sin, d_pos, d_kvrow, kv_head_stride, d_q, d_k, d_v, T, n_heads, n_kv_heads, st))
    return -1;
  VLO_CUDA(cudaStreamSynchronize(st));  // the tables are freed on return
  return 0;
}

int vlo_op_gemm_prefill(int epi, const void* d_w, int rows_w, const void* d_x, int rows_x, int k, int n_ctas, void* d_out,
                        void* cuda_stream) {
  VLO_CHECK(n_ctas >= 0, "gemm_prefill: n_ctas");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_prefill_launch(epi, WeightOperand{FMT_BF16, d_w, nullptr, nullptr}, rows_w, d_x, rows_x, k, n_ctas, d_out,
                             static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_gemm_prefill_q(int fmt, int epi, const void* d_w, const float* d_scale, const void* d_gscale, int rows_w,
                          const void* d_x, const float* d_xscale, int rows_x, int k, int n_ctas, void* d_out,
                          void* cuda_stream) {
  VLO_CHECK(n_ctas >= 0, "gemm_prefill_q: n_ctas");
  VLO_CHECK(fmt == FMT_E4M3 || fmt == FMT_E4M3_A8 || fmt == FMT_I4, "gemm_prefill_q: fmt 2 (e4m3), 3 (W8A8) or 4 (int4)");
  VLO_CHECK(d_w != nullptr && d_x != nullptr, "gemm_prefill_q: null operand");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_prefill_launch(epi, WeightOperand{fmt, d_w, d_scale, static_cast<const uint16_t*>(d_gscale)}, rows_w, d_x,
                             rows_x, k, n_ctas, d_out, static_cast<cudaStream_t>(cuda_stream), nullptr, d_xscale);
}

int vlo_op_gemm_swiglu(const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_act, float* d_planes,
                       int64_t plane_elems, int32_t* d_flags, int n_flags, void* cuda_stream) {
  VLO_CHECK(plane_elems >= 0, "gemm_swiglu: plane_elems");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_wsf_launch(WeightOperand{FMT_BF16, d_w, nullptr, nullptr}, rows_w, d_x, rows_x, k, d_act, d_planes,
                         static_cast<size_t>(plane_elems), d_flags, n_flags, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_gemm_swiglu_f8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x, int rows_x, int k, void* d_act,
                          float* d_planes, int64_t plane_elems, int32_t* d_flags, int n_flags, void* cuda_stream) {
  VLO_CHECK(plane_elems >= 0, "gemm_swiglu_f8: plane_elems");
  VLO_CHECK(d_scale != nullptr, "gemm_swiglu_f8: null row scales");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_wsf_launch(WeightOperand{FMT_E4M3, d_w8, d_scale, nullptr}, rows_w, d_x, rows_x, k, d_act, d_planes,
                         static_cast<size_t>(plane_elems), d_flags, n_flags, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_gemm_swiglu_a8(const void* d_w8, const float* d_scale, int rows_w, const void* d_x8, const float* d_xscale,
                          int rows_x, int k, void* d_act, float* d_planes, int64_t plane_elems, int32_t* d_flags, int n_flags,
                          void* cuda_stream) {
  VLO_CHECK(plane_elems >= 0, "gemm_swiglu_a8: plane_elems");
  VLO_CHECK(d_scale != nullptr && d_xscale != nullptr, "gemm_swiglu_a8: null row or token scales");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_wsf_launch(WeightOperand{FMT_E4M3_A8, d_w8, d_scale, nullptr}, rows_w, d_x8, rows_x, k, d_act, d_planes,
                         static_cast<size_t>(plane_elems), d_flags, n_flags, static_cast<cudaStream_t>(cuda_stream), d_xscale);
}

int vlo_op_gemm_swiglu_i4(const void* d_w4, const void* d_gscale, int rows_w, const void* d_x, int rows_x, int k, void* d_act,
                          float* d_planes, int64_t plane_elems, int32_t* d_flags, int n_flags, void* cuda_stream) {
  VLO_CHECK(plane_elems >= 0, "gemm_swiglu_i4: plane_elems");
  VLO_CHECK(d_gscale != nullptr, "gemm_swiglu_i4: null group scales");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return gemm_wsf_launch(WeightOperand{FMT_I4, d_w4, nullptr, static_cast<const uint16_t*>(d_gscale)}, rows_w, d_x, rows_x,
                         k, d_act, d_planes, static_cast<size_t>(plane_elems), d_flags, n_flags,
                         static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_decision(const void* d_logits, int n_rows, int vocab, int interval_id, vlo_decision* d_out, void* cuda_stream) {
  VLO_CHECK(n_rows > 0 && vocab > 0 && vocab % 8 == 0, "decision: rows of a positive multiple of 8 logits");
  VLO_CHECK((reinterpret_cast<uintptr_t>(d_logits) & 15) == 0, "decision: logits must be 16-byte aligned");
  if (pdl_probe_fire(static_cast<cudaStream_t>(cuda_stream))) return -1;
  return decision_launch(d_logits, n_rows, vocab, interval_id, d_out, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_sample(const void* d_logits, int n_rows, int vocab, const vlo_sample_row* h_rows, const int32_t* h_penalty_ids,
                  int n_penalty_ids, int32_t* d_out_ids, void* d_info, void* cuda_stream) {
  VLO_CHECK(n_rows > 0 && vocab > 0 && vocab % 8 == 0, "sample: rows of a positive multiple of 8 logits");
  VLO_CHECK(d_logits != nullptr && d_out_ids != nullptr, "sample: null argument");
  VLO_CHECK((reinterpret_cast<uintptr_t>(d_logits) & 15) == 0, "sample: logits must be 16-byte aligned");
  VLO_CHECK(n_penalty_ids >= 0 && (n_penalty_ids == 0 || h_penalty_ids != nullptr), "sample: penalty ids");
  if (sample_check_rows(h_rows, n_rows, n_penalty_ids)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  const size_t rows_bytes = align256(sizeof(vlo_sample_row) * n_rows);
  uint8_t* d_par = nullptr;
  VLO_CUDA(cudaMalloc(&d_par, rows_bytes + sizeof(int32_t) * (n_penalty_ids + 1)));
  int rc = cudaMemcpy(d_par, h_rows, sizeof(vlo_sample_row) * n_rows, cudaMemcpyHostToDevice) != cudaSuccess ||
           (n_penalty_ids && cudaMemcpy(d_par + rows_bytes, h_penalty_ids, sizeof(int32_t) * n_penalty_ids,
                                        cudaMemcpyHostToDevice) != cudaSuccess)
               ? fail("sample: parameter upload failed")
               : 0;
  if (rc == 0) rc = pdl_probe_fire(st);
  if (rc == 0) rc = sample_launch(d_logits, n_rows, vocab, d_par, reinterpret_cast<const int*>(d_par + rows_bytes),
                                  d_out_ids, d_info, st);
  if (rc == 0 && cudaStreamSynchronize(st) != cudaSuccess) rc = fail("sample: kernel failed");
  cudaFree(d_par);
  return rc;
}

/* Back-to-back launches of the KV-append attention over `n_layers` separate K / V matrices (layer l at
 * d_k + l * layer_stride_rows * head_dim elements), `iters` passes: the micro-loop of vlo_bench_attn without an engine
 * (bench tools time it with one CUDA-event pair).  The plan is built and uploaded once, as in a decoder step. */
int vlo_op_attn_bench(const void* d_q, const void* d_k, const void* d_v, void* d_out, float* d_ws, int n_tok, int n_heads,
                      int n_kv_heads, int head_dim, int kv_len, long long kv_stride, int n_layers,
                      long long layer_stride_rows, int iters, int skip_merge, double* h_algo_bytes, void* cuda_stream) {
  VLO_CHECK(n_layers > 0 && iters > 0 && layer_stride_rows >= static_cast<long long>(n_kv_heads) * kv_stride, "attn_bench: sizes");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  AttnPlan plan{};
  const int* pt = nullptr;
  if (op_attn_plan(&plan, d_ws, n_tok, n_heads, n_kv_heads, head_dim, kv_len, true, &pt, st)) return -1;
  plan.skip_merge = skip_merge;
  if (h_algo_bytes) *h_algo_bytes = plan.algo_bytes;
  const size_t lstride = static_cast<size_t>(layer_stride_rows) * head_dim * 2;
  if (pdl_probe_fire(st)) return -1;
  for (int it = 0; it < iters; ++it)
    for (int l = 0; l < n_layers; ++l)
      if (attn_run(plan, d_q, static_cast<const uint8_t*>(d_k) + l * lstride, static_cast<const uint8_t*>(d_v) + l * lstride,
                   static_cast<long long>(n_kv_heads) * kv_stride, pt, kKvPageTokens, kv_stride, d_out, n_heads,
                   n_kv_heads, head_dim, st))
        return -1;
  return 0;
}

int vlo_op_pdl_arm(int mode, void* d_dst, void* d_src, long long bytes, int n_chunks, long long chunk_stride,
                   long long spin_ns) {
  VLO_CHECK(mode == VLO_PDL_LATE_WRITE || mode == VLO_PDL_LATE_READ, "pdl_arm: mode 1 (late write) or 2 (late read)");
  VLO_CHECK(d_dst != nullptr && d_src != nullptr && bytes > 0 && n_chunks > 0, "pdl_arm: null pointer or empty range");
  VLO_CHECK(n_chunks == 1 || chunk_stride >= bytes, "pdl_arm: chunks must not overlap");
  VLO_CHECK(spin_ns > 0 && spin_ns <= kProbeMaxSpinNs, "pdl_arm: spin_ns must lie in (0, 2 ms]");
  g_probe = PdlProbe{mode, static_cast<uint8_t*>(d_dst), static_cast<uint8_t*>(d_src), bytes, chunk_stride, spin_ns,
                     n_chunks};
  return 0;
}

long long vlo_op_pdl_probe_count(void) {
  unsigned long long n = 0;
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(&n, g_probes_done, sizeof(n)) != cudaSuccess) {
    fail("pdl_probe_count: " + std::string(cudaGetErrorString(cudaGetLastError())));
    return -1;
  }
  return static_cast<long long>(n);
}

int vlo_op_pdl_canary(int variant, const void* d_src, void* d_dst, int n_words, void* cuda_stream) {
  VLO_CHECK(variant >= 0 && variant <= 2 && d_src != nullptr && d_dst != nullptr && n_words > 0, "pdl_canary: arguments");
  cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
  if (pdl_probe_fire(st)) return -1;
  VLO_CUDA(launch_pdl(pdl_canary_kernel, dim3((n_words + 255) / 256), dim3(256), 0, st, variant,
                      static_cast<const uint32_t*>(d_src), static_cast<uint32_t*>(d_dst), n_words));
  return 0;
}

}  // extern "C"
