// Vision-tower kernels around the wgmma GEMMs: pixel rescale/normalise + patchify, LayerNorm,
// the 576-token non-causal self-attention, 3x3 adaptive average pool, the MAP-head probe attention
// and the final token assembly.  Dtype flow follows the reference's GPU path — fp16 autocast
// operands, fp32 LayerNorm and residual stream (models/vision_live.py:10-30 under
// models/modeling_live.py:23; HF:models/siglip/modeling_siglip.py).
#pragma once
#include <cuda.h>
#include "mma.cuh"
#include "ptx.cuh"
#include "streamk.h"

namespace vlo {

// ---------------------------------------------------------------------------------------------
// K1 + im2col: frames u8 [B,3,S,S] -> fp16 patches [B*P, 3*ps*ps], value (x/255 - .5)/.5
// (models/vision_live.py:12; column order = conv weight [C,3,ps,ps] flattened,
//  HF:...siglip.py:175-179).  One thread per 8 horizontally adjacent pixels.
__global__ void __launch_bounds__(256) patchify_kernel(const uint8_t* frames, __half* out, int B, int S, int ps) {
  pdl_trigger();
  pdl_wait();
  const int g = S / ps, P = g * g, K = 3 * ps * ps;
  const long long total = static_cast<long long>(B) * P * K / 8;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long e = idx * 8;
    const int col = static_cast<int>(e % K);
    const long long row = e / K;
    const int b = static_cast<int>(row / P), pidx = static_cast<int>(row % P);
    const int py = pidx / g, px = pidx % g;
    const int c = col / (ps * ps), iy = (col / ps) % ps, ix = col % ps;
    const uint8_t* src = frames + ((static_cast<size_t>(b) * 3 + c) * S + (py * ps + iy)) * S + px * ps + ix;
    const uint2 raw = *reinterpret_cast<const uint2*>(src);
    const uint32_t w[2] = {raw.x, raw.y};
    __half h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float x = static_cast<float>((w[j >> 2] >> ((j & 3) * 8)) & 0xff);
      const float v = (x * 0.00392156862745098f - 0.5f) / 0.5f;
      h[j] = __float2half_rn(v);
    }
    *reinterpret_cast<uint4*>(out + e) = *reinterpret_cast<const uint4*>(h);
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm over the last dim, fp32 statistics (nn.LayerNorm under autocast runs in fp32).
// in: fp32 (trunk residual stream) or fp16 (MAP head); out16 fp16, optional out32.
template <typename InT>
__global__ void __launch_bounds__(256) layernorm_kernel(const InT* in, const float* w, const float* b, __half* out16,
                                                        float* out32, int C, float eps) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float row[];
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  float s = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float v = static_cast<float>(in[r * C + i]);
    row[i] = v;
    s += v;
  }
  s = warp_sum(s);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (lane == 0) red[warp] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < nw; ++i) tot += red[i];
  const float mean = tot / C;
  __syncthreads();
  float q = 0.f;
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float d = row[i] - mean;
    q += d * d;
  }
  q = warp_sum(q);
  if (lane == 0) red[warp] = q;
  __syncthreads();
  float var = 0.f;
  for (int i = 0; i < nw; ++i) var += red[i];
  const float rstd = rsqrtf(var / C + eps);
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    const float y = (row[i] - mean) * rstd * w[i] + b[i];
    if (out16) out16[r * C + i] = __float2half_rn(y);
    if (out32) out32[r * C + i] = y;
  }
}

// Stream-K fix-up + fp32 residual add + LayerNorm in one pass over a token row:
//   y    = fp16(sum_s part[s][r][:] + bias)      (the out_proj / fc2 Linear output under fp16 autocast)
//   h[r] += y                                     (fp32 residual stream, HF:...siglip.py:353,360)
//   out  = LayerNorm(h[r])                        (the next layer_norm1 / layer_norm2 / post_layernorm)
struct VitFixLnParams {
  const float* part;  // [planes][rows][C], stream-K planes of tile (col/128) * sk_xtiles + row / sk_bn
  SkInfo sk;
  int sk_bn, sk_xtiles;
  long long split_stride;
  const float* bias;
  float* h;
  const float* ln_w;
  const float* ln_b;
  __half* out16;
  float* out32;
  int C;
  float eps;
};
__global__ void __launch_bounds__(256) vit_fix_ln_kernel(const VitFixLnParams p) {
  pdl_trigger();
  pdl_wait();
  // 4 contiguous channels per thread per sweep; the (<= kFixMaxPlanes) plane loads of a sweep are independent.
  extern __shared__ float row[];
  __shared__ float red[32];
  const size_t r = blockIdx.x;
  const int C = p.C;
  float s = 0.f;
  for (int i = threadIdx.x * 4; i < C; i += blockDim.x * 4) {
    float4 a[kFixMaxPlanes];
    const int ns = sk_planes((i >> 7) * p.sk_xtiles + static_cast<int>(r) / p.sk_bn, p.sk);
#pragma unroll
    for (int k = 0; k < kFixMaxPlanes; ++k)
      a[k] = (k < ns) ? *reinterpret_cast<const float4*>(p.part + k * p.split_stride + r * C + i)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 hv = *reinterpret_cast<const float4*>(p.h + r * C + i);
    const float4 bv = *reinterpret_cast<const float4*>(p.bias + i);
    float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < kFixMaxPlanes; ++k) {
      y.x += a[k].x; y.y += a[k].y; y.z += a[k].z; y.w += a[k].w;
    }
    float4 v;
    v.x = hv.x + fp16_round(y.x + bv.x);
    v.y = hv.y + fp16_round(y.y + bv.y);
    v.z = hv.z + fp16_round(y.z + bv.z);
    v.w = hv.w + fp16_round(y.w + bv.w);
    *reinterpret_cast<float4*>(p.h + r * C + i) = v;
    *reinterpret_cast<float4*>(row + i) = v;
    s += v.x + v.y + v.z + v.w;
  }
  s = warp_sum(s);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  if (lane == 0) red[warp] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < nw; ++i) tot += red[i];
  const float mean = tot / C;
  __syncthreads();
  float q = 0.f;
  for (int i = threadIdx.x * 4; i < C; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    const float d0 = v.x - mean, d1 = v.y - mean, d2 = v.z - mean, d3 = v.w - mean;
    q += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
  }
  q = warp_sum(q);
  if (lane == 0) red[warp] = q;
  __syncthreads();
  float var = 0.f;
  for (int i = 0; i < nw; ++i) var += red[i];
  const float rstd = rsqrtf(var / C + p.eps);
  for (int i = threadIdx.x * 4; i < C; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + i);
    const float4 w = *reinterpret_cast<const float4*>(p.ln_w + i);
    const float4 b = *reinterpret_cast<const float4*>(p.ln_b + i);
    float4 y;
    y.x = (v.x - mean) * rstd * w.x + b.x;
    y.y = (v.y - mean) * rstd * w.y + b.y;
    y.z = (v.z - mean) * rstd * w.z + b.z;
    y.w = (v.w - mean) * rstd * w.w + b.w;
    if (p.out16) {
      __half2 h01 = __floats2half2_rn(y.x, y.y), h23 = __floats2half2_rn(y.z, y.w);
      uint2 o;
      o.x = *reinterpret_cast<uint32_t*>(&h01);
      o.y = *reinterpret_cast<uint32_t*>(&h23);
      *reinterpret_cast<uint2*>(p.out16 + r * C + i) = o;
    }
    if (p.out32) *reinterpret_cast<float4*>(p.out32 + r * C + i) = y;
  }
}

// ---------------------------------------------------------------------------------------------
// ViT self-attention (K5): non-causal softmax(Q K^T / sqrt(64)) V, fp16, head_dim 64.
// qkv: [B*N, 3C] fp16 (q | k | v column blocks, head h at column h*64 inside each).
// grid = (ceil(N/64), heads, B); block = 160 (warp 0 = TMA producer, warps 1-4 = 16 query rows each).
constexpr int kVitHD = 64;
constexpr int kVitBlk = 64;
constexpr int kVitStages = 4;
constexpr int kVitTile = kVitBlk * kVitHD * 2;  // 8 KB
constexpr int kVitSmemBytes = kVitTile * (1 + 2 * kVitStages) + 1024 + 256;
constexpr int kVitThreads = 160;

__device__ __forceinline__ void mma_f16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, "
      "{%8, %9}, {%0, %1, %2, %3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_f16(float lo, float hi) {
  __half2 t = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

__global__ void __launch_bounds__(kVitThreads, 1)
vit_attn_kernel(const __grid_constant__ CUtensorMap tm_qkv, __half* out, int N, int C, float scale_log2) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* q_tile = smem;
  uint8_t* kv_tiles = smem + kVitTile;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kVitTile * (1 + 2 * kVitStages));
  uint64_t* empty_bar = full_bar + kVitStages;
  uint64_t* q_bar = empty_bar + kVitStages;

  const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nblk = (N + kVitBlk - 1) / kVitBlk;
  const int row_base = b * N;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_qkv);
    for (int i = 0; i < kVitStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 4);
    }
    mbar_init(q_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  if (warp == 0) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_bar, kVitTile);
      tma_load_2d(q_tile, &tm_qkv, q_bar, head * kVitHD, row_base + qt * kVitBlk, kEvictNormal);
      for (int i = 0; i < nblk; ++i) {
        const int s = i % kVitStages;
        const uint32_t ph = (i / kVitStages) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        mbar_arrive_expect_tx(&full_bar[s], 2 * kVitTile);
        tma_load_2d(kv_tiles + s * 2 * kVitTile, &tm_qkv, &full_bar[s], C + head * kVitHD, row_base + i * kVitBlk,
                    kEvictNormal);
        tma_load_2d(kv_tiles + s * 2 * kVitTile + kVitTile, &tm_qkv, &full_bar[s], 2 * C + head * kVitHD,
                    row_base + i * kVitBlk, kEvictNormal);
      }
    }
    return;
  }
  const int mt = warp - 1;
  const int g8 = lane >> 2, q4 = lane & 3;
  // Q fragments (16 rows x 64 dims = 4 k-steps) via ldmatrix from the swizzled tile
  uint32_t qf[4][4];
  mbar_wait(q_bar, 0);
  {
    const uint32_t qs = smem_u32(q_tile);
    const int r = mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int cg = 2 * ks + (lane >> 4);
      ldsm_x4(qs + r * 128 + ((cg ^ (r & 7)) << 4), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
    }
  }
  float o_acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float c = scale_log2;

  for (int i = 0; i < nblk; ++i) {
    const int s = i % kVitStages;
    const uint32_t ph = (i / kVitStages) & 1;
    mbar_wait(&full_bar[s], ph);
    const uint32_t sk = smem_u32(kv_tiles + s * 2 * kVitTile);
    const uint32_t sv = sk + kVitTile;
    float sc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      sc[nt][0] = sc[nt][1] = sc[nt][2] = sc[nt][3] = 0.f;
      const int krow = nt * 8 + (lane & 7);
#pragma unroll
      for (int kp = 0; kp < 2; ++kp) {
        const int cg = kp * 4 + (lane >> 3);
        uint32_t b0, b1, b2, b3;
        ldsm_x4(sk + krow * 128 + ((cg ^ (krow & 7)) << 4), b0, b1, b2, b3);
        mma_f16_16816(sc[nt], qf[2 * kp], b0, b1);
        mma_f16_16816(sc[nt], qf[2 * kp + 1], b2, b3);
      }
    }
    const int key0 = i * kVitBlk;
    if (key0 + kVitBlk > N) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int k = key0 + nt * 8 + q4 * 2;
        if (k >= N) sc[nt][0] = sc[nt][2] = -INFINITY;
        if (k + 1 >= N) sc[nt][1] = sc[nt][3] = -INFINITY;
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx0 = fmaxf(mx0, fmaxf(sc[nt][0], sc[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(sc[nt][2], sc[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m_run[0], mx0), mn1 = fmaxf(m_run[1], mx1);
    const float me0 = (mn0 == -INFINITY) ? 0.f : mn0 * c, me1 = (mn1 == -INFINITY) ? 0.f : mn1 * c;
    const float al0 = exp2f(m_run[0] * c - me0), al1 = exp2f(m_run[1] * c - me1);
    m_run[0] = mn0;
    m_run[1] = mn1;
    float ps0 = 0.f, ps1 = 0.f;
    uint32_t pf[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f(sc[nt][0] * c - me0), p1 = exp2f(sc[nt][1] * c - me0);
      const float p2 = exp2f(sc[nt][2] * c - me1), p3 = exp2f(sc[nt][3] * c - me1);
      ps0 += p0 + p1;
      ps1 += p2 + p3;
      pf[nt >> 1][(nt & 1) * 2 + 0] = pack_f16(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_f16(p2, p3);
    }
    l_run[0] = l_run[0] * al0 + ps0;
    l_run[1] = l_run[1] * al1 + ps1;
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {
      o_acc[nd][0] *= al0;
      o_acc[nd][1] *= al0;
      o_acc[nd][2] *= al1;
      o_acc[nd][3] *= al1;
    }
    // keys >= N of the last block are the next frame's first rows (or the TMA zero fill past the last frame): P is 0
    // there, but 0 * Inf and 0 * NaN are NaN, so the 4 MMA warps zero those V rows in the stage before the P V product
    // reads it.  A finite row's 0 * v adds nothing, so the bits stay those of the unmasked product.
    if (key0 + kVitBlk > N) {
      uint8_t* vst = kv_tiles + s * 2 * kVitTile + kVitTile;
      const int first = N - key0;  // rows first .. 63: 8 chunks of 16 B per row
      for (int c = mt * 32 + lane; c < (kVitBlk - first) * 8; c += 4 * 32)
        *reinterpret_cast<uint4*>(vst + (first + (c >> 3)) * 128 + (c & 7) * 16) = make_uint4(0, 0, 0, 0);
      fence_proxy_async();    // the stage's next TMA fill is ordered after these stores
      named_bar_sync<1>(4 * 32);  // the 4 MMA warps
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const int vrow = kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        const int cg = np * 2 + (lane >> 4);
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(sv + vrow * 128 + ((cg ^ (vrow & 7)) << 4), b0, b1, b2, b3);
        mma_f16_16816(o_acc[2 * np], pf[kk], b0, b1);
        mma_f16_16816(o_acc[2 * np + 1], pf[kk], b2, b3);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }
  l_run[0] += __shfl_xor_sync(0xffffffffu, l_run[0], 1);
  l_run[0] += __shfl_xor_sync(0xffffffffu, l_run[0], 2);
  l_run[1] += __shfl_xor_sync(0xffffffffu, l_run[1], 1);
  l_run[1] += __shfl_xor_sync(0xffffffffu, l_run[1], 2);
  const int r0 = qt * kVitBlk + mt * 16 + g8, r1 = r0 + 8;
  const float i0 = 1.f / l_run[0], i1 = 1.f / l_run[1];
#pragma unroll
  for (int nd = 0; nd < 8; ++nd) {
    const int col = head * kVitHD + nd * 8 + q4 * 2;
    if (r0 < N)
      *reinterpret_cast<__half2*>(out + static_cast<size_t>(row_base + r0) * C + col) =
          __floats2half2_rn(o_acc[nd][0] * i0, o_acc[nd][1] * i0);
    if (r1 < N)
      *reinterpret_cast<__half2*>(out + static_cast<size_t>(row_base + r1) * C + col) =
          __floats2half2_rn(o_acc[nd][2] * i1, o_acc[nd][3] * i1);
  }
}

// ---------------------------------------------------------------------------------------------
// K8: adaptive_avg_pool2d of the g x g token grid to ph x pw (models/vision_live.py:17-23),
// written into the token buffer after the optional CLS slot.  in: fp32 [B, g*g, C].
__global__ void __launch_bounds__(256) pool_kernel(const float* in, float* tokens, int B, int g, int C, int ph, int pw,
                                                   int n_tok, int tok_off) {
  pdl_trigger();
  pdl_wait();
  const long long total = static_cast<long long>(B) * ph * pw * C;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ch = static_cast<int>(idx % C);
    const int cell = static_cast<int>((idx / C) % (ph * pw));
    const int b = static_cast<int>(idx / (static_cast<long long>(C) * ph * pw));
    const int i = cell / pw, j = cell % pw;
    const int y0 = (i * g) / ph, y1 = ((i + 1) * g + ph - 1) / ph;
    const int x0 = (j * g) / pw, x1 = ((j + 1) * g + pw - 1) / pw;
    float s = 0.f;
    for (int y = y0; y < y1; ++y)
      for (int x = x0; x < x1; ++x) s += in[(static_cast<size_t>(b) * g * g + y * g + x) * C + ch];
    tokens[(static_cast<size_t>(b) * n_tok + tok_off + cell) * C + ch] = s / static_cast<float>((y1 - y0) * (x1 - x0));
  }
}

// ---------------------------------------------------------------------------------------------
// K7 (part): MAP-head attention of the single learned probe over the N tokens
// (SiglipMultiheadAttentionPoolingHead, HF:...siglip.py:628-651 -> nn.MultiheadAttention).
// kv: fp16 [B*N, 2C] (k | v), q: fp32 [C] (= in_proj_q(probe), rounded to fp16 on the host by pack_vision_for_engine).
// grid = (heads, B), block = 128; dynamic smem = N floats.
__global__ void __launch_bounds__(128) probe_attn_kernel(const __half* kv, const float* q, __half* out, int N, int C,
                                                         float scale) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float sc[];
  __shared__ float red[4];
  __shared__ float part[2][kVitHD];
  const int head = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const __half* kb = kv + static_cast<size_t>(b) * N * 2 * C + head * kVitHD;
  float qreg[kVitHD];
#pragma unroll
  for (int d = 0; d < kVitHD; ++d) qreg[d] = q[head * kVitHD + d] * scale;
  float mx = -INFINITY;
  for (int n = tid; n < N; n += 128) {
    const __half2* kr = reinterpret_cast<const __half2*>(kb + static_cast<size_t>(n) * 2 * C);
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < kVitHD / 2; ++d) {
      const float2 k2 = __half22float2(kr[d]);
      s += qreg[2 * d] * k2.x + qreg[2 * d + 1] * k2.y;
    }
    sc[n] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if ((tid & 31) == 0) red[tid >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int n = tid; n < N; n += 128) {
    const float e = expf(sc[n] - mx);
    sc[n] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if ((tid & 31) == 0) red[tid >> 5] = sum;
  __syncthreads();
  sum = red[0] + red[1] + red[2] + red[3];
  // weighted V: thread (half, d) sums over its half of the keys
  const int d = tid & 63, hf = tid >> 6;
  const __half* vb = kb + C + d;
  float acc = 0.f;
  int n = hf;
  for (; n + 14 < N; n += 16) {  // 8 independent loads in flight
    float x[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) x[u] = __half2float(vb[static_cast<size_t>(n + 2 * u) * 2 * C]);
#pragma unroll
    for (int u = 0; u < 8; ++u) acc += sc[n + 2 * u] * x[u];
  }
  for (; n < N; n += 2) acc += sc[n] * __half2float(vb[static_cast<size_t>(n) * 2 * C]);
  part[hf][d] = acc;
  __syncthreads();
  if (tid < kVitHD) out[static_cast<size_t>(b) * C + head * kVitHD + tid] = __float2half_rn((part[0][tid] + part[1][tid]) / sum);
}

// CLS slot of the token buffer = fp16(residual + mlp_out)  (HF:...siglip.py:647-651); then
// tokens16 = bf16(tokens32) is what the connector reads (frames.to(self.dtype),
// models/modeling_live.py:25).
__global__ void __launch_bounds__(256) cls_residual_kernel(const __half* resid, const __half* mlp, float* tokens, int B,
                                                           int C, int n_tok) {
  pdl_trigger();
  pdl_wait();
  const int total = B * C;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int b = idx / C, c = idx % C;
    const float v = __half2float(__float2half_rn(__half2float(resid[idx]) + __half2float(mlp[idx])));
    tokens[(static_cast<size_t>(b) * n_tok) * C + c] = v;
  }
}
__global__ void __launch_bounds__(256) f32_to_bf16_kernel(const float* in, __nv_bfloat16* out, long long n) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = __float2bfloat16_rn(in[i]);
}

}  // namespace vlo
