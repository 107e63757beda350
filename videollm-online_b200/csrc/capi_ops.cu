// C-ABI: library-level and kernel-level entry points (see include/vlo_b200.h).
#include "vlo_b200.h"

#include <vector>

#include "common.h"
#include "gemm.cuh"
#include "kv_pages.h"

using namespace vlo;

namespace {

// Plan one sequence of n_tok queries over kv_len keys and upload the plan into d_ws.  h_identity_pt: also upload an
// identity page table (the contiguous [n_kv_heads][kv_stride][128] layout, one "page" per 64-key block) behind the
// plan's workspace and return its device address in *d_pt.  The upload is synchronised: the staging is pageable.
int op_attn_plan(AttnPlan* plan, float* d_ws, int n_tok, int n_heads, int n_kv_heads, int head_dim, int kv_len,
                 bool identity_pt, const int** d_pt, cudaStream_t st) {
  VLO_CHECK(n_tok > 0 && kv_len >= n_tok, "attn: need 0 < n_tok <= kv_len");
  AttnSeq s{};
  s.q_tok0 = 0;
  s.q_len = n_tok;
  s.kv_len = kv_len;
  s.pt0 = 0;
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

}  // namespace

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
  return gemm_launch(c, static_cast<cudaStream_t>(cuda_stream));
}

int vlo_op_gemm_ws(int fmt, int mode, const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out,
                   int ld_out, long long plane_stride, const float* d_bias, int act, int n_ctas, int bn, int* h_max_planes,
                   void* cuda_stream) {
  GemmWsCall c{};
  c.fmt = fmt;
  c.mode = mode;
  c.w = d_w;
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
  GemmWsPlan plan{};
  const int rc = gemm_ws_launch(c, static_cast<cudaStream_t>(cuda_stream), &plan);
  if (rc == 0 && h_max_planes) *h_max_planes = plan.planes;
  return rc;
}

int vlo_op_gemm_vit(const void* d_w, int rows_w, const void* d_x, int rows_x, int k, void* d_out, int ld_out,
                    const float* d_bias, int act, int n_ctas, void* cuda_stream) {
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
  const long long page_rows = static_cast<long long>(n_kv_heads) * kKvPageTokens;
  if (attn_run(plan, d_q, d_k_pool, d_v_pool, n_pages * page_rows, d_page_table, page_rows, kKvPageTokens, d_out, n_heads,
               n_kv_heads, head_dim, st))
    return -1;
  VLO_CUDA(cudaStreamSynchronize(st));
  return 0;
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
  for (int it = 0; it < iters; ++it)
    for (int l = 0; l < n_layers; ++l)
      if (attn_run(plan, d_q, static_cast<const uint8_t*>(d_k) + l * lstride, static_cast<const uint8_t*>(d_v) + l * lstride,
                   static_cast<long long>(n_kv_heads) * kv_stride, pt, kKvPageTokens, kv_stride, d_out, n_heads,
                   n_kv_heads, head_dim, st))
        return -1;
  return 0;
}

}  // extern "C"
