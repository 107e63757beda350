// Small fused kernels around the decoder GEMMs.  Every rounding point mirrors the HF bf16 Llama
// path (HF:models/llama/modeling_llama.py) so that the only numeric difference left against the
// reference forward is the accumulation order inside the GEMMs and the attention.
#pragma once
#include <cuda_fp8.h>
#include "ptx.cuh"
#include "streamk.h"

namespace vlo {

__device__ __forceinline__ float bf16_load(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// block-wide sum for <= 1024 threads
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (warp == 0) {
    t = warp_sum(t);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// block-wide max for <= 1024 threads
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (warp == 0) {
    t = warp_max(t);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// ---------------------------------------------------------------------------------------------
// Per-token e4m3 quantization of a bf16 row X[t, :] (weights.quantize_fp8_rows applied to activation rows):
//   s[t] = fp32(max_k |X[t, k]|) / 448   (1 for an all-zero row)
//   q[t, k] = e4m3fn(clamp(fp32(X[t, k]) / s[t], +-448))   IEEE division, round to nearest even
// The saturating conversion is the clamp: a quotient past 448 can only be the rounding of amax / s.
constexpr float kE4m3Max = 448.f;
__device__ __forceinline__ float e4m3_row_scale(float amax) { return amax > 0.f ? __fdiv_rn(amax, kE4m3Max) : 1.f; }
__device__ __forceinline__ uint16_t e4m3x2(float a, float b, float s) {
  return __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(a, s), __fdiv_rn(b, s)), __NV_SATFINITE, __NV_E4M3);
}

// ---------------------------------------------------------------------------------------------
// Stream-K fix-up + residual add + RMSNorm in one pass over a token row:
//   y      = bf16(sum_s part[s][t][:])                (the Linear output, o_proj / down_proj)
//   h[t]   = bf16(h[t] + y)                           (residual, HF:...llama.py:325,331)
//   xn[t]  = w * bf16(h * rsqrt(mean(h^2) + eps))     (LlamaRMSNorm.forward, HF:...llama.py:62-67)
// part == null: no partials, plain RMSNorm of h (first layer).  `xn_last` (optional) receives
// compact copies of the rows flagged in last_index (>= 0): the final-norm rows the lm_head needs.
// grid = T rows, block = 256.
struct ResidNormParams {
  const float* part;        // stream-K planes per 128-column tile (sk), or null
  long long split_stride;
  SkInfo sk;
  __nv_bfloat16* h;         // [T, H] residual stream, updated in place
  const __nv_bfloat16* w;   // [H] norm weight
  __nv_bfloat16* xn;        // [T, H] normalised output (may be null)
  __nv_bfloat16* xn_last;   // [n_last, H] or null
  const int* last_index;    // [T] or null
  int H;
  float eps;
};

// kQ8 (resid_rmsnorm_q8_kernel): also the e4m3 row xq[t] and its scale xs[t] of the bf16 xn row, quantized as above;
// xn itself is the same as without.
template <bool kQ8>
__device__ __forceinline__ void resid_rmsnorm_body(const ResidNormParams p, uint8_t* xq, float* xs) {
  // one CTA per token row, 4 contiguous elements per thread per sweep; the plane loads of a sweep are
  // independent (predicated, fully unrolled) so they are all in flight together.
  extern __shared__ float row[];  // H floats
  __shared__ float red[32];
  const int t = blockIdx.x;
  __nv_bfloat16* h = p.h + static_cast<size_t>(t) * p.H;
  pdl_trigger();
  // Everything that does not depend on the producer kernel is fetched BEFORE the grid dependency resolves: the norm
  // weight (a static tensor that the 15 GB weight stream has long evicted from L2 - an HBM miss that used to sit on
  // the critical path after the block reduction), the stream-K plane count of this thread's first column group and
  // the last-token index (tables uploaded by the memcpy at the start of the step).
  const int i0 = threadIdx.x * 4;
  const uint2 w_pre = (i0 < p.H) ? *reinterpret_cast<const uint2*>(p.w + i0) : make_uint2(0u, 0u);
  const int ns_pre = (p.part != nullptr && i0 < p.H) ? sk_planes(i0 >> 7, p.sk) : 0;
  const int li = p.last_index ? p.last_index[t] : -1;
  pdl_wait();
  float ss = 0.f;
  for (int i = threadIdx.x * 4; i < p.H; i += blockDim.x * 4) {
    const uint2 hraw = *reinterpret_cast<const uint2*>(h + i);
    float2 v01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hraw.x));
    float2 v23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&hraw.y));
    if (p.part != nullptr) {
      const int ns = (i == i0) ? ns_pre : sk_planes(i >> 7, p.sk);
      const float* pp = p.part + static_cast<size_t>(t) * p.H + i;
      float4 a[kFixMaxPlanes];
#pragma unroll
      for (int s = 0; s < kFixMaxPlanes; ++s)
        a[s] = (s < ns) ? *reinterpret_cast<const float4*>(pp + s * p.split_stride) : make_float4(0.f, 0.f, 0.f, 0.f);
      float y0 = 0.f, y1 = 0.f, y2 = 0.f, y3 = 0.f;
#pragma unroll
      for (int s = 0; s < kFixMaxPlanes; ++s) {  // plane order: deterministic
        y0 += a[s].x; y1 += a[s].y; y2 += a[s].z; y3 += a[s].w;
      }
      v01.x = bf16_round(v01.x + bf16_round(y0));
      v01.y = bf16_round(v01.y + bf16_round(y1));
      v23.x = bf16_round(v23.x + bf16_round(y2));
      v23.y = bf16_round(v23.y + bf16_round(y3));
      uint2 o;
      *reinterpret_cast<__nv_bfloat162*>(&o.x) = __floats2bfloat162_rn(v01.x, v01.y);
      *reinterpret_cast<__nv_bfloat162*>(&o.y) = __floats2bfloat162_rn(v23.x, v23.y);
      *reinterpret_cast<uint2*>(h + i) = o;
    }
    row[i] = v01.x; row[i + 1] = v01.y; row[i + 2] = v23.x; row[i + 3] = v23.y;
    ss += v01.x * v01.x + v01.y * v01.y + v23.x * v23.x + v23.y * v23.y;
  }
  const float tot = block_sum(ss, red);
  const float rstd = rsqrtf(tot / static_cast<float>(p.H) + p.eps);
  float amax = 0.f;
  for (int i = threadIdx.x * 4; i < p.H; i += blockDim.x * 4) {
    const uint2 wraw = (i == i0) ? w_pre : *reinterpret_cast<const uint2*>(p.w + i);
    const float2 w01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wraw.x));
    const float2 w23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wraw.y));
    uint2 o;
    *reinterpret_cast<__nv_bfloat162*>(&o.x) = __floats2bfloat162_rn(bf16_round(w01.x * bf16_round(row[i] * rstd)),
                                                                     bf16_round(w01.y * bf16_round(row[i + 1] * rstd)));
    *reinterpret_cast<__nv_bfloat162*>(&o.y) = __floats2bfloat162_rn(bf16_round(w23.x * bf16_round(row[i + 2] * rstd)),
                                                                     bf16_round(w23.y * bf16_round(row[i + 3] * rstd)));
    if (p.xn) *reinterpret_cast<uint2*>(p.xn + static_cast<size_t>(t) * p.H + i) = o;
    if (li >= 0) *reinterpret_cast<uint2*>(p.xn_last + static_cast<size_t>(li) * p.H + i) = o;
    if constexpr (kQ8) {   // this thread's own row[] entries now hold the bf16 xn values
      const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&o.x));
      const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&o.y));
      row[i] = a.x; row[i + 1] = a.y; row[i + 2] = b.x; row[i + 3] = b.y;
      amax = fmaxf(fmaxf(amax, fmaxf(fabsf(a.x), fabsf(a.y))), fmaxf(fabsf(b.x), fabsf(b.y)));
    }
  }
  if constexpr (kQ8) {
    const float sc = e4m3_row_scale(block_max(amax, red));
    for (int i = threadIdx.x * 4; i < p.H; i += blockDim.x * 4)
      *reinterpret_cast<uint32_t*>(xq + static_cast<size_t>(t) * p.H + i) =
          e4m3x2(row[i], row[i + 1], sc) | (static_cast<uint32_t>(e4m3x2(row[i + 2], row[i + 3], sc)) << 16);
    if (threadIdx.x == 0) xs[t] = sc;
  }
}

__global__ void __launch_bounds__(1024) resid_rmsnorm_kernel(const ResidNormParams p) {
  resid_rmsnorm_body<false>(p, nullptr, nullptr);
}
__global__ void __launch_bounds__(1024) resid_rmsnorm_q8_kernel(const ResidNormParams p, uint8_t* xq, float* xs) {
  resid_rmsnorm_body<true>(p, xq, xs);
}

// One CTA per row of a bf16 [T, K] tensor (K % 8 == 0): e4m3 q[T, K] and fp32 s[T] by the rule above.  The row is read
// twice (amax, then the codes); the second read hits L1 / L2.
__global__ void __launch_bounds__(256) quant_rows_e4m3_kernel(const __nv_bfloat16* x, int K, uint8_t* q, float* s) {
  __shared__ float red[32];
  const int t = blockIdx.x;
  const __nv_bfloat16* xr = x + static_cast<size_t>(t) * K;
  pdl_trigger();
  pdl_wait();
  float amax = 0.f;
  for (int i = threadIdx.x * 8; i < K; i += blockDim.x * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[j]));
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
  }
  const float sc = e4m3_row_scale(block_max(amax, red));
  for (int i = threadIdx.x * 8; i < K; i += blockDim.x * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(xr + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t c[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float2 f0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[2 * j]));
      const float2 f1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[2 * j + 1]));
      c[j] = e4m3x2(f0.x, f0.y, sc) | (static_cast<uint32_t>(e4m3x2(f1.x, f1.y, sc)) << 16);
    }
    *reinterpret_cast<uint2*>(q + static_cast<size_t>(t) * K + i) = make_uint2(c[0], c[1]);
  }
  if (threadIdx.x == 0) s[t] = sc;
}

// ---------------------------------------------------------------------------------------------
// QKV stream-K fix-up + RoPE + KV-cache append (SURVEY K12/K13/K14 fused):
//   q,k,v = bf16(sum_s part)                              (HF:...llama.py:262-264)
//   q,k   = x*cos + rotate_half(x)*sin in bf16            (apply_rotary_pos_emb, :146-168)
//   K/V rows written in place at the token's position     (replaces DynamicLayer.update's
//                                                          torch.cat, HF:cache_utils.py:119-120)
// cos/sin: bf16 tables [max_pos, head_dim/2] (the two halves of HF's cos/sin are identical).
// grid = (T, n_heads + 2*n_kv_heads), block = 64 (thread d handles dims d and d+64).
struct QkvRopeParams {
  const float* part;       // [S][T][(nh + 2 nkv) * 128], stream-K planes (head hh == weight tile hh)
  long long split_stride;
  SkInfo sk;
  const __nv_bfloat16* cos_tab;
  const __nv_bfloat16* sin_tab;
  const int* tok_pos;      // [T] absolute position of the token in its stream
  const long long* tok_kvrow;  // [T] cache row of (the token's position, kv head 0): its page's row + pos % 64
  int kv_head_stride;      // rows between kv heads (64 in the page pool)
  __nv_bfloat16* q_out;    // [T, nh, 128]
  __nv_bfloat16* k_cache;  // layer base, rows of 128
  __nv_bfloat16* v_cache;
  int n_heads, n_kv_heads;
};

__global__ void __launch_bounds__(64) qkv_rope_append_kernel(const QkvRopeParams p) {
  const int t = blockIdx.x, hh = blockIdx.y, d = threadIdx.x;
  pdl_trigger();
  // Before the grid dependency resolves: token position / cache row (tables uploaded by the memcpy at the start of
  // the step), the RoPE table entries (static) and the plane count - three dependent round trips off the critical path.
  const int width = (p.n_heads + 2 * p.n_kv_heads) * 128;
  const float* pp = p.part + static_cast<size_t>(t) * width + hh * 128 + d;
  const int ns = sk_planes(hh, p.sk);
  const int pos = p.tok_pos[t];
  const long long kvrow = p.tok_kvrow[t];
  const bool rot = hh < p.n_heads + p.n_kv_heads;
  const float c = rot ? __bfloat162float(p.cos_tab[static_cast<size_t>(pos) * 64 + d]) : 1.f;
  const float s = rot ? __bfloat162float(p.sin_tab[static_cast<size_t>(pos) * 64 + d]) : 0.f;
  pdl_wait();
  float x1 = 0.f, x2 = 0.f;
  float a1[kFixMaxPlanes], a2[kFixMaxPlanes];  // all plane loads in flight together
#pragma unroll
  for (int k = 0; k < kFixMaxPlanes; ++k) {
    a1[k] = (k < ns) ? pp[k * p.split_stride] : 0.f;
    a2[k] = (k < ns) ? pp[k * p.split_stride + 64] : 0.f;
  }
#pragma unroll
  for (int k = 0; k < kFixMaxPlanes; ++k) {  // plane order: deterministic
    x1 += a1[k];
    x2 += a2[k];
  }
  x1 = bf16_round(x1);
  x2 = bf16_round(x2);
  if (rot) {
    const float o1 = bf16_round(bf16_round(x1 * c) + bf16_round(-x2 * s));
    const float o2 = bf16_round(bf16_round(x2 * c) + bf16_round(x1 * s));
    x1 = o1;
    x2 = o2;
  }
  __nv_bfloat16* dst;
  if (hh < p.n_heads) {
    dst = p.q_out + (static_cast<size_t>(t) * p.n_heads + hh) * 128;
  } else {
    const int kvh = (hh - p.n_heads) % p.n_kv_heads;
    __nv_bfloat16* base = (hh < p.n_heads + p.n_kv_heads) ? p.k_cache : p.v_cache;
    dst = base + (kvrow + static_cast<long long>(kvh) * p.kv_head_stride) * 128;
  }
  dst[d] = __float2bfloat16_rn(x1);
  dst[d + 64] = __float2bfloat16_rn(x2);
}

// ---------------------------------------------------------------------------------------------
// Token-embedding gather (K10) into rows of the packed step input.
//   ids[i] >= 0  -> dst row dst_rows[i] = table[min(id, vocab-1)]   (clamp: models/modeling_live.py:38)
//   ids[i] <  0  -> leave the row alone (it already holds a frame embedding)
__global__ void __launch_bounds__(256) embed_rows_kernel(const long long* ids, const int* dst_rows, int n,
                                                         const __nv_bfloat16* table, int vocab, int H,
                                                         __nv_bfloat16* dst) {
  const int i = blockIdx.x;
  if (i >= n) return;
  long long id = ids[i];
  if (id < 0) return;
  if (id > vocab - 1) id = vocab - 1;
  const int r = dst_rows ? dst_rows[i] : i;
  const uint4* src = reinterpret_cast<const uint4*>(table + static_cast<size_t>(id) * H);
  uint4* out = reinterpret_cast<uint4*>(dst + static_cast<size_t>(r) * H);
  for (int j = threadIdx.x; j < H / 8; j += blockDim.x) out[j] = src[j];
}

// The same gather from a quantized table [vocab, H]: the ids are taken as embed_rows_kernel takes them, and the row is
// dequantized on the way.
//   I4 = false (e4m3): codes [vocab][H] bytes, fp32 row scales; element k of row n = bf16_rn(fp32(q[n, k]) * s[n])
//   I4 = true:  codes in the engine byte order (gemm.cuh), bf16 group scales [vocab][H / 128]; element k of row n =
//               bf16_rn(q * s[n, k / 128]), q = code - 8 (the W4 of the int4 GEMMs).  In each (tile, k-block) unit the
//               row's 64 codes lie in the 16 bytes of four consumer threads (lane % 4 = 0..3) at h * 2048 + 16 t, t = 32
//               warp + lane; one thread here decodes one of those 16-byte pieces: 16 codes, columns 16 kk + 8 f + 2 (lane
//               % 4) + b.
template <bool I4>
__global__ void __launch_bounds__(256) embed_rows_q_kernel(const long long* ids, const int* dst_rows, int n,
                                                           const uint8_t* codes, const void* scale, int vocab, int H,
                                                           __nv_bfloat16* dst) {
  const int i = blockIdx.x;
  if (i >= n) return;
  long long id = ids[i];
  if (id < 0) return;
  if (id > vocab - 1) id = vocab - 1;
  const int r = dst_rows ? dst_rows[i] : i;
  __nv_bfloat16* out = dst + static_cast<size_t>(r) * H;
  if constexpr (!I4) {
    const float s = __ldg(static_cast<const float*>(scale) + id);
    const uint2* src = reinterpret_cast<const uint2*>(codes + static_cast<size_t>(id) * H);
    for (int j = threadIdx.x; j < H / 8; j += blockDim.x) {
      const uint2 v = src[j];
      uint32_t w[4];
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const uint32_t two = (p < 2 ? v.x : v.y) >> (16 * (p & 1));
        const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(two & 0xFFFF), __NV_E4M3);
        const float2 q = __half22float2(__half2(h));   // exact
        const __nv_bfloat162 b = __floats2bfloat162_rn(__fmul_rn(q.x, s), __fmul_rn(q.y, s));
        w[p] = *reinterpret_cast<const uint32_t*>(&b);
      }
      reinterpret_cast<uint4*>(out)[j] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  } else {
    const int kb = H / 64, ng = H / 128;
    const int tile = static_cast<int>(id / 128), rr = static_cast<int>(id % 128);
    const int h = rr / 64, warp = (rr % 64) / 16, e = (rr % 16) / 8, lane_hi = rr % 8;
    const uint16_t* gs = static_cast<const uint16_t*>(scale) + static_cast<size_t>(id) * ng;
    for (int j = threadIdx.x; j < kb * 4; j += blockDim.x) {
      const int kblk = j / 4, l4 = j % 4;
      const uint8_t* unit = codes + (static_cast<size_t>(tile) * kb + kblk) * 4096;
      const uint4 c = *reinterpret_cast<const uint4*>(unit + h * 2048 + (32 * warp + 4 * lane_hi + l4) * 16);
      const float s = __bfloat162float(__ushort_as_bfloat16(__ldg(gs + kblk / 2)));
      const uint32_t words[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int f = 0; f < 2; ++f) {
          const int sh = 4 * (e + 2 * f);
          const float q0 = static_cast<float>(static_cast<int>((words[kk] >> sh) & 0xF) - 8);
          const float q1 = static_cast<float>(static_cast<int>((words[kk] >> (sh + 16)) & 0xF) - 8);
          const __nv_bfloat162 b = __floats2bfloat162_rn(q0 * s, q1 * s);   // q * s is exact in fp32: one rounding
          *reinterpret_cast<__nv_bfloat162*>(out + kblk * 64 + 16 * kk + 8 * f + 2 * l4) = b;
        }
    }
  }
}

// copy packed rows (bf16) src[i] -> dst[rows[i]]
__global__ void __launch_bounds__(256) scatter_rows_kernel(const __nv_bfloat16* src, const int* rows, int n, int H,
                                                           __nv_bfloat16* dst) {
  const int i = blockIdx.x;
  if (i >= n) return;
  const uint4* s = reinterpret_cast<const uint4*>(src + static_cast<size_t>(i) * H);
  uint4* o = reinterpret_cast<uint4*>(dst + static_cast<size_t>(rows[i]) * H);
  for (int j = threadIdx.x; j < H / 8; j += blockDim.x) o[j] = s[j];
}

// ---------------------------------------------------------------------------------------------
// Speak/silent decision + greedy argmax on the device (SURVEY K19; demo/inference.py:76-81,
// models/modeling_live.py:177-179): one block per sequence over its bf16 logits row.
struct DecisionOut {  // == vlo_decision
  int argmax_id;
  int argmax_excl_id;
  float p_interval;
  float max_logit;
  float top2_margin;
  float lse;
  int argmax_prob_id;
  int reserved1;
};

__global__ void __launch_bounds__(1024) decision_kernel(const __nv_bfloat16* logits, int vocab, int interval_id,
                                                        DecisionOut* out) {
  // Two vectorised sweeps over the row (16-byte loads, 8 logits each):
  //   A: first-index max, second max and the online sum of exponentials;
  //   B: argmax of the bf16-rounded probabilities with / without the interval id.
  __shared__ float s_m1[32], s_m2[32], s_se[32], s_pa[32], s_pe[32];
  __shared__ int s_i1[32], s_ia[32], s_ie[32];
  __shared__ float s_gmax, s_gmax2, s_sum;
  __shared__ int s_gidx;
  pdl_trigger();
  pdl_wait();
  const __nv_bfloat16* x = logits + static_cast<size_t>(blockIdx.x) * vocab;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int nvec = vocab / 8;  // rows are 16-byte aligned (vocab % 8 == 0 checked by the engine); tail handled below

  // ---- sweep A
  float m1 = -INFINITY, m2 = -INFINITY, se = 0.f;
  int i1 = 0x7fffffff;
  auto take = [&](float v, int idx) {
    if (v > m1) {
      se = se * __expf(m1 - v) + 1.f;  // m1 = -inf on the first element: se = 0 * 0 + 1
      m2 = m1; m1 = v; i1 = idx;
    } else {
      se += __expf(v - m1);
      if (v > m2) m2 = v;
    }
  };
  for (int v0 = tid; v0 < nvec; v0 += 4 * blockDim.x) {  // 4 independent 16-byte loads in flight per thread
    uint4 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int vi = v0 + u * blockDim.x;
      raw[u] = vi < nvec ? *reinterpret_cast<const uint4*>(x + static_cast<size_t>(vi) * 8) : make_uint4(0xff80ff80u, 0xff80ff80u, 0xff80ff80u, 0xff80ff80u);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int vi = v0 + u * blockDim.x;
      if (vi >= nvec) break;
      const uint32_t w[4] = {raw[u].x, raw[u].y, raw[u].z, raw[u].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[k]));
        take(f.x, vi * 8 + 2 * k);
        take(f.y, vi * 8 + 2 * k + 1);
      }
    }
  }
  for (int idx = nvec * 8 + tid; idx < vocab; idx += blockDim.x) take(__bfloat162float(x[idx]), idx);
  auto merge = [&](float om1, int oi1, float om2, float ose) {
    if (om1 > m1 || (om1 == m1 && oi1 < i1)) {
      se = ose + se * __expf(m1 - om1);
      m2 = fmaxf(m1, om2); m1 = om1; i1 = oi1;
    } else if (oi1 != 0x7fffffff) {
      se += ose * __expf(om1 - m1);
      m2 = fmaxf(m2, om1);
    }
  };
  for (int o = 16; o > 0; o >>= 1) {
    const float om1 = __shfl_xor_sync(0xffffffffu, m1, o), om2 = __shfl_xor_sync(0xffffffffu, m2, o);
    const float ose = __shfl_xor_sync(0xffffffffu, se, o);
    const int oi1 = __shfl_xor_sync(0xffffffffu, i1, o);
    merge(om1, oi1, om2, ose);
  }
  if (lane == 0) { s_m1[warp] = m1; s_i1[warp] = i1; s_m2[warp] = m2; s_se[warp] = se; }
  __syncthreads();
  if (warp == 0) {
    m1 = lane < nw ? s_m1[lane] : -INFINITY;
    i1 = lane < nw ? s_i1[lane] : 0x7fffffff;
    m2 = lane < nw ? s_m2[lane] : -INFINITY;
    se = lane < nw ? s_se[lane] : 0.f;
    for (int o = 16; o > 0; o >>= 1) {
      const float om1 = __shfl_xor_sync(0xffffffffu, m1, o), om2 = __shfl_xor_sync(0xffffffffu, m2, o);
      const float ose = __shfl_xor_sync(0xffffffffu, se, o);
      const int oi1 = __shfl_xor_sync(0xffffffffu, i1, o);
      merge(om1, oi1, om2, ose);
    }
    if (lane == 0) { s_gmax = m1; s_gidx = i1; s_gmax2 = m2; s_sum = se; }
  }
  __syncthreads();
  const float gmax = s_gmax, sum = s_sum;

  // ---- sweep B: what `next_score.argmax` sees (demo/inference.py:76-79); first index wins ties
  float pa = -1.f, pe = -1.f;
  int ia = 0x7fffffff, ie = 0x7fffffff;
  auto prob = [&](float v, int idx) {
    const float pr = bf16_round(__expf(v - gmax) / sum);
    if (pr > pa) { pa = pr; ia = idx; }
    const float pz = (idx == interval_id) ? 0.f : pr;  // zero_() then argmax
    if (pz > pe) { pe = pz; ie = idx; }
  };
  for (int v0 = tid; v0 < nvec; v0 += 4 * blockDim.x) {
    uint4 raw[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int vi = v0 + u * blockDim.x;
      raw[u] = vi < nvec ? *reinterpret_cast<const uint4*>(x + static_cast<size_t>(vi) * 8) : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int vi = v0 + u * blockDim.x;
      if (vi >= nvec) break;
      const uint32_t w[4] = {raw[u].x, raw[u].y, raw[u].z, raw[u].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[k]));
        prob(f.x, vi * 8 + 2 * k);
        prob(f.y, vi * 8 + 2 * k + 1);
      }
    }
  }
  for (int idx = nvec * 8 + tid; idx < vocab; idx += blockDim.x) prob(__bfloat162float(x[idx]), idx);
  for (int o = 16; o > 0; o >>= 1) {
    const float opa = __shfl_xor_sync(0xffffffffu, pa, o), ope = __shfl_xor_sync(0xffffffffu, pe, o);
    const int oia = __shfl_xor_sync(0xffffffffu, ia, o), oie = __shfl_xor_sync(0xffffffffu, ie, o);
    if (opa > pa || (opa == pa && oia < ia)) { pa = opa; ia = oia; }
    if (ope > pe || (ope == pe && oie < ie)) { pe = ope; ie = oie; }
  }
  if (lane == 0) { s_pa[warp] = pa; s_ia[warp] = ia; s_pe[warp] = pe; s_ie[warp] = ie; }
  __syncthreads();
  if (warp == 0) {
    pa = lane < nw ? s_pa[lane] : -1.f; ia = lane < nw ? s_ia[lane] : 0x7fffffff;
    pe = lane < nw ? s_pe[lane] : -1.f; ie = lane < nw ? s_ie[lane] : 0x7fffffff;
    for (int o = 16; o > 0; o >>= 1) {
      const float opa = __shfl_xor_sync(0xffffffffu, pa, o), ope = __shfl_xor_sync(0xffffffffu, pe, o);
      const int oia = __shfl_xor_sync(0xffffffffu, ia, o), oie = __shfl_xor_sync(0xffffffffu, ie, o);
      if (opa > pa || (opa == pa && oia < ia)) { pa = opa; ia = oia; }
      if (ope > pe || (ope == pe && oie < ie)) { pe = ope; ie = oie; }
    }
    if (lane == 0) {
      DecisionOut d;
      d.argmax_id = s_gidx;
      d.argmax_excl_id = ie;
      d.p_interval = (interval_id >= 0 && interval_id < vocab)
                         ? bf16_round(__expf(__bfloat162float(x[interval_id]) - gmax) / sum)
                         : 0.f;
      d.max_logit = gmax;
      d.top2_margin = gmax - s_gmax2;
      d.lse = gmax + logf(sum);
      d.argmax_prob_id = ia;
      d.reserved1 = 0;
      out[blockIdx.x] = d;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// KV page-pool copies and fill.  One layer's K or V matrix is a plane of [page][kv_head][64][128] rows (kv_pages.h);
// planes follow each other at plane_stride elements.  A paged side is addressed through its page table, a
// contiguous side is [n_kv_heads][ld][128].
struct KvSide {
  __nv_bfloat16* base;
  const int* pt;  // page table, or null: contiguous
  long long plane_stride;
  int ld;         // contiguous rows per kv head
};
__device__ __forceinline__ long long kv_side_row(const KvSide& s, int n_kv, int h, int pos) {
  return s.pt ? (static_cast<long long>(s.pt[pos >> 6]) * n_kv + h) * 64 + (pos & 63)
              : static_cast<long long>(h) * s.ld + pos;
}

// rows [0, n_tok) of every kv head and plane: src -> dst, 16 bytes per thread.
// grid = (ceil(n_tok * 16 / 256), n_kv_heads, planes), block = 256.
__global__ void __launch_bounds__(256) kv_copy_kernel(const KvSide src, const KvSide dst, int n_kv, int n_tok) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n_tok) * 16) return;
  const int pos = static_cast<int>(i >> 4), c = static_cast<int>(i & 15), h = blockIdx.y, pl = blockIdx.z;
  const uint4* s = reinterpret_cast<const uint4*>(src.base + pl * src.plane_stride + kv_side_row(src, n_kv, h, pos) * 128);
  uint4* d = reinterpret_cast<uint4*>(dst.base + pl * dst.plane_stride + kv_side_row(dst, n_kv, h, pos) * 128);
  d[c] = s[c];
}

// KV synthetic fill (bench pre-fill): deterministic finite pseudo-random bf16 in about [-1, 1].  The value of element
// d of (position pos, kv head h) of plane pl = 2 layer + is_v hashes the LOGICAL index
// ((sid * n_kv + h) * max_kv_tokens + pos) * 128 + d with seed + pl * 1315423911 + h * 2654435761, wherever its page is.
// grid = (x, n_kv_heads, planes), block = 256.
__global__ void __launch_bounds__(256) kv_fill_kernel(const KvSide dst, int n_kv, int n_tok, int sid, int max_kv_tokens,
                                                      unsigned long long seed) {
  const int h = blockIdx.y, pl = blockIdx.z;
  const unsigned long long sd = seed + static_cast<unsigned long long>(pl) * 1315423911ull + h * 2654435761ull;
  const long long row0 = (static_cast<long long>(sid) * n_kv + h) * max_kv_tokens;
  const long long n = static_cast<long long>(n_tok) * 128;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    unsigned long long z = sd + 0x9E3779B97F4A7C15ull * static_cast<unsigned long long>(row0 * 128 + i + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    const float u = static_cast<float>(z >> 40) * (1.0f / 16777216.0f);  // [0,1)
    const int pos = static_cast<int>(i >> 7);
    dst.base[pl * dst.plane_stride + kv_side_row(dst, n_kv, h, pos) * 128 + (i & 127)] = __float2bfloat16_rn(2.f * u - 1.f);
  }
}

// The re-rotation of eight RoPE pairs (d, d + 64), d = d0 .. d0 + 7, of one key row: a holds x1 = k[d0 .. d0 + 8),
// b holds x2 = k[64 + d0 .. 64 + d0 + 8), cs = [c_0 .. c_63 | s_0 .. s_63].  On return
//   a[d] = bf16(fl(fl(x1 c_d) + fl(x2 s_d)))      b[d] = bf16(fl(fl(x2 c_d) - fl(x1 s_d)))
// every fl one fp32 round-to-nearest (no FMA contraction), so an fp32 emulation reproduces it bit for bit.  The one
// definition of the arithmetic kv_rerotate_kernel and kv_compact_kernel share.
__device__ __forceinline__ void rope_rerotate8(uint4& a, uint4& b, const float* cs, int d0) {
  float c[8], s[8];
  *reinterpret_cast<float4*>(c) = *reinterpret_cast<const float4*>(cs + d0);
  *reinterpret_cast<float4*>(c + 4) = *reinterpret_cast<const float4*>(cs + d0 + 4);
  *reinterpret_cast<float4*>(s) = *reinterpret_cast<const float4*>(cs + 64 + d0);
  *reinterpret_cast<float4*>(s + 4) = *reinterpret_cast<const float4*>(cs + 64 + d0 + 4);
  const uint32_t wa[4] = {a.x, a.y, a.z, a.w}, wb[4] = {b.x, b.y, b.z, b.w};
  uint32_t oa[4], ob[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 x1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wa[j]));
    const float2 x2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&wb[j]));
    const float c0 = c[2 * j], c1 = c[2 * j + 1], s0 = s[2 * j], s1 = s[2 * j + 1];
    const __nv_bfloat162 r1 = __floats2bfloat162_rn(__fadd_rn(__fmul_rn(x1.x, c0), __fmul_rn(x2.x, s0)),
                                                    __fadd_rn(__fmul_rn(x1.y, c1), __fmul_rn(x2.y, s1)));
    const __nv_bfloat162 r2 = __floats2bfloat162_rn(__fsub_rn(__fmul_rn(x2.x, c0), __fmul_rn(x1.x, s0)),
                                                    __fsub_rn(__fmul_rn(x2.y, c1), __fmul_rn(x1.y, s1)));
    oa[j] = *reinterpret_cast<const uint32_t*>(&r1);
    ob[j] = *reinterpret_cast<const uint32_t*>(&r2);
  }
  a = make_uint4(oa[0], oa[1], oa[2], oa[3]);
  b = make_uint4(ob[0], ob[1], ob[2], ob[3]);
}

// KV eviction: rotate the keys of positions [pos0, pos0 + n_tok) of every kv head and layer by -delta in place, so that
// a key RoPE put at position p sits at p - delta (V has no position in it and is not touched).  With the RoPE pairs
// (d, d + 64) of qkv_rope_append_kernel and cs = [c_0 .. c_63 | s_0 .. s_63], c_d = cos(delta f_d), s_d = sin(delta f_d),
// each key is rotated by rope_rerotate8.  Each thread rotates eight pairs of one row (two 16-byte loads and stores); no
// row depends on another.  K of layer l is plane 2 l.
// grid = (ceil(n_tok * 8 / 256), n_kv_heads, layers), block = 256.
__global__ void __launch_bounds__(256) kv_rerotate_kernel(const KvSide k, int n_kv, int pos0, int n_tok, const float* cs) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n_tok) * 8) return;
  const int pos = pos0 + static_cast<int>(i >> 3), d0 = static_cast<int>(i & 7) * 8, h = blockIdx.y, l = blockIdx.z;
  __nv_bfloat16* row = k.base + 2ll * l * k.plane_stride + kv_side_row(k, n_kv, h, pos) * 128;
  uint4* lo = reinterpret_cast<uint4*>(row + d0);
  uint4* hi = reinterpret_cast<uint4*>(row + 64 + d0);
  uint4 a = *lo, b = *hi;
  rope_rerotate8(a, b, cs, d0);
  *lo = a;
  *hi = b;
}

// Token-granular KV compaction (vlo_kv_compact), one batch of (destination page, plane) units.  Kept span i moves from
// cache positions [src[i], src[i] + len) to [dst[i], dst[i] + len), dst[i] <= src[i]; its keys are rotated by
// rope_rerotate8 with cs + 128 i (cos | sin of d_i = src[i] - dst[i]), its values are copied.  Unit u of the batch is
// destination page j = j0 + (u0 + u) / planes of plane (u0 + u) % planes (K of layer l is plane 2 l, V plane 2 l + 1).
//   gather (to_stage): read the sources of the unit's positions q in [q_lo, new_len) through the stream's table, rotate
//     the K rows, write them to stage[u][kv head][q % 64][128];
//   scatter: copy those stage rows to the unit's own positions, through the same table.
// A destination page j only reads source positions >= 64 j (every d_i >= 0), so the batches, run in increasing unit
// order with a batch's scatter after its gather, never overwrite a row a later batch still reads: the compaction runs in
// place, and its bits do not depend on the batching.  Positions below q_lo (spans with d_i = 0) and past new_len are not
// written.  Each thread moves eight RoPE pairs (or 16 V elements) of one row.
// grid = (ceil(n_units * n_kv * 64 * 8 / 256)), block = 256.
struct CompactSpans {
  const float* cs;   // [n][128]: cos | sin of each span's shift
  const int* src;    // [n] first source position of each span
  const int* dst;    // [n] first destination position, ascending, dst[0] = 0
  int n;
};
__global__ void __launch_bounds__(256) kv_compact_kernel(const KvSide kv, int n_kv, int planes, int j0, int u0, int n_units,
                                                         int q_lo, int new_len, const CompactSpans sp,
                                                         __nv_bfloat16* stage, int to_stage) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int per_unit = n_kv * 64 * 8;
  if (i >= static_cast<long long>(n_units) * per_unit) return;
  const int u = static_cast<int>(i / per_unit), t = static_cast<int>(i % per_unit);
  const int h = t >> 9, r = (t >> 3) & 63, d0 = (t & 7) * 8;
  const int unit = u0 + u, pl = unit % planes, q = (j0 + unit / planes) * 64 + r;
  if (q < q_lo || q >= new_len) return;
  __nv_bfloat16* st = stage + ((static_cast<long long>(u) * n_kv + h) * 64 + r) * 128;
  __nv_bfloat16* plane = kv.base + pl * kv.plane_stride;
  if (!to_stage) {
    __nv_bfloat16* row = plane + kv_side_row(kv, n_kv, h, q) * 128;
    *reinterpret_cast<uint4*>(row + d0) = *reinterpret_cast<const uint4*>(st + d0);
    *reinterpret_cast<uint4*>(row + 64 + d0) = *reinterpret_cast<const uint4*>(st + 64 + d0);
    return;
  }
  int lo = 0, hi = sp.n - 1;   // the span holding q: the last one with dst <= q
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sp.dst[mid] <= q) lo = mid;
    else hi = mid - 1;
  }
  const __nv_bfloat16* row = plane + kv_side_row(kv, n_kv, h, sp.src[lo] + q - sp.dst[lo]) * 128;
  uint4 a = *reinterpret_cast<const uint4*>(row + d0), b = *reinterpret_cast<const uint4*>(row + 64 + d0);
  if ((pl & 1) == 0) rope_rerotate8(a, b, sp.cs + 128ll * lo, d0);
  *reinterpret_cast<uint4*>(st + d0) = a;
  *reinterpret_cast<uint4*>(st + 64 + d0) = b;
}

}  // namespace vlo
