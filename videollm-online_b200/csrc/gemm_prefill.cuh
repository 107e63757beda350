// Prefill GEMM of the decoder layers (bf16 weights) for inputs longer than one step:  out[t, n] = sum_k X[t, k] * W[n, k]
// over up to max_prefill_tokens token rows, with the bits of the chunked path (gemm_ws_kernel mode 0 on each
// <= 128-token chunk, then the fix-up kernels / the gate|up finisher).
//
// The problem is tensor-bound, so the tokens ride wgmma M and each CTA computes whole 128-token x 128-feature tiles:
//   warps 0-3   warpgroup 0: wgmma m64n128k16 on token rows 0-63 of the tile
//   warps 4-7   warpgroup 1: the same on token rows 64-127
//   warp 8      TMA producer: one 16 KB X box and one 16 KB W box per 64-wide k-block, 128-byte swizzle
// Persistent, one CTA per SM: CTA c owns tiles [c * tiles / G, (c + 1) * tiles / G), tile = weight tile * m_tiles + token
// tile, so a CTA's consecutive tiles share their weight tile and re-read it from L2.
//
// Exactness.  A chunk of the chunked path has one token tile, so the stream-K plan of a weight tile (sk: units of one
// weight tile x one 64-wide k-block over G CTAs, streamk.h) depends on (N, K, G) alone.  Its k-ranges are those of the
// CTAs sk_first_cta(tile) .. in order; each partial plane is an in-order wgmma chain from zero over one range, and the
// fix-up sums the planes in plane order.  This kernel walks the same ranges: each range runs from a zeroed accumulator
// (acc), and the finished range is added into a second register set (sum) in plane order:
//   PREFILL_PLANE   sum = 0 + P0 + P1 + ...  (the fix-up kernels' order), written as ONE fp32 plane [rows_x][rows_w]
//                   that qkv_rope_append_kernel and resid_rmsnorm_kernel read through a one-plane SkInfo (G = 1): they
//                   add 0 + sum + 0 ..., which gives sum again (sum is never -0);
//   PREFILL_SWIGLU  g, u = P0 + P1 + ... (the gate|up finisher's order), then gemm_wsf's SwiGLU (swiglu_bf16, gemm.cuh)
//                   into act [rows_x][rows_w / 2].  Tile j holds gate features 64 j .. 64 j + 63 in its rows 0-63 and the
//                   matching up features in rows 64-127, so a thread holds the gate value of column group g and the up
//                   value of group g + 8 of the same token: no exchange is needed.
// One output's wgmma chain has the same bits whichever operand carries the tokens and however wide the token tile is
// (tests/test_gpu_vit_gemm.py, tests/test_gpu_frame_backlog.py); tests/test_gpu_prefill.py holds this kernel to the
// chunked path bit for bit.
//
// PDL: the first S weight boxes load before griddepcontrol.wait (the weights never depend on an earlier kernel).
#pragma once
#include <cuda.h>
#include "gemm.cuh"
#include "streamk.h"

namespace vlo {

struct GemmPrefillArgs {
  int rows_x, rows_w, k;  // X [rows_x, k] (tokens), W [rows_w, k]
  int m_tiles;            // ceil(rows_x / 128)
  int tiles;              // m_tiles * ceil(rows_w / 128)
  SkInfo sk;              // the chunked path's stream-K plan of the weight tiles (one token tile)
  float* plane;           // PREFILL_PLANE: [rows_x][rows_w]
  __nv_bfloat16* act;     // PREFILL_SWIGLU: [rows_x][rows_w / 2]
};

constexpr int kPrefillThreads = 288;
constexpr int kPrefillProducerWarp = 8;

struct GemmPrefillCfg {
  static constexpr int kBytesX = kGemmBM * kGemmBK * 2;
  static constexpr int kBytesW = kGemmBM * kGemmBK * 2;
  // 1024 B of slack to align the ring for SWIZZLE_128B, 256 B of barriers
  static constexpr int kStages = fit_stages(kBytesX + kBytesW, 1024 + 256, 6);
  static constexpr int kSmemBytes = kStages * (kBytesX + kBytesW) + 1024 + 256;
};

template <int EPI>
__global__ void __launch_bounds__(kPrefillThreads, 1)
gemm_prefill_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                    const __grid_constant__ GemmPrefillArgs p) {
  using Cfg = GemmPrefillCfg;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_x = smem;
  uint8_t* smem_w = smem + S * Cfg::kBytesX;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S * (Cfg::kBytesX + Cfg::kBytesW));
  uint64_t* empty_bar = full_bar + S;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb = p.k / kGemmBK;
  const int tile0 = static_cast<int>((static_cast<long long>(blockIdx.x) * p.tiles) / gridDim.x);
  const int tile1 = static_cast<int>((static_cast<long long>(blockIdx.x + 1) * p.tiles) / gridDim.x);
  const long long u0 = static_cast<long long>(tile0) * kb, u1 = static_cast<long long>(tile1) * kb;
  const bool producer = warp == kPrefillProducerWarp && lane == 0;

  if (producer) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_w);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();
  int pre = 0;
  if (producer) {
    for (long long u = u0; u < u1 && pre < S; ++u, ++pre) {
      const int tile = static_cast<int>(u / kb);
      const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
      const int nt = tile / p.m_tiles;
      mbar_arrive_expect_tx(&full_bar[pre], Cfg::kBytesX + Cfg::kBytesW);
      tma_load_2d(smem_w + pre * Cfg::kBytesW, &tm_w, &full_bar[pre], kblk * kGemmBK, nt * kGemmBM, kEvictNormal);
    }
  }
  // the activations are the predecessors' output
  pdl_wait();

  if (warp == kPrefillProducerWarp) {
    if (lane == 0) {
      int i = 0;
      for (long long u = u0; u < u1; ++u, ++i) {
        const int tile = static_cast<int>(u / kb);
        const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
        const int nt = tile / p.m_tiles, mt = tile - nt * p.m_tiles;
        const int s = i % S;
        if (i >= pre) {
          mbar_wait(&empty_bar[s], ((i / S) & 1) ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], Cfg::kBytesX + Cfg::kBytesW);
          tma_load_2d(smem_w + s * Cfg::kBytesW, &tm_w, &full_bar[s], kblk * kGemmBK, nt * kGemmBM, kEvictNormal);
        }
        tma_load_2d(smem_x + s * Cfg::kBytesX, &tm_x, &full_bar[s], kblk * kGemmBK, mt * kGemmBM, kEvictLast);
      }
    }
    return;
  }

  // -------------------------------------------------- consumer warpgroups
  const int wg = warp >> 2;
  // accumulator element 4 * g + r of this thread: tile row rbase + 8 * (r >> 1), column 8 * g + cq + (r & 1)
  const int rbase = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
  int i = 0;
  for (int tile = tile0; tile < tile1; ++tile) {
    const int nt = tile / p.m_tiles, mt = tile - nt * p.m_tiles;
    const long long t_u0 = static_cast<long long>(nt) * kb;  // the weight tile's first unit in the plan
    float sum[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) sum[j] = 0.f;
    // one k-range per contributing CTA of the plan, in plane order
    for (int c = sk_first_cta(nt, p.sk), j = 0; j < kb; ++c) {
      const int j_end = static_cast<int>(min(static_cast<long long>(kb), sk_lo(c + 1, p.sk) - t_u0));
      const bool first = j == 0;
      float acc[64];
#pragma unroll
      for (int q = 0; q < 64; ++q) acc[q] = 0.f;
      // one k-block of MMAs stays in flight while the next stage is awaited; a stage is released once its MMAs retire
      for (int jj = 0; j < j_end; ++j, ++jj, ++i) {
        const int s = i % S;
        mbar_wait(&full_bar[s], (i / S) & 1);
        wgmma_fence();
        const uint64_t dx = wgmma_desc_sw128(smem_u32(smem_x + s * Cfg::kBytesX + wg * (Cfg::kBytesX / 2)));
        const uint64_t dw = wgmma_desc_sw128(smem_u32(smem_w + s * Cfg::kBytesW));
#pragma unroll
        for (int kk = 0; kk < kGemmBK / 16; ++kk) Wgmma<FMT_BF16, 128>::mma(acc, dx + 2 * kk, dw + 2 * kk);
        wgmma_commit();
        wgmma_wait<1>();
        if (jj > 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % S]);
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % S]);
      if (EPI == PREFILL_SWIGLU && first) {
#pragma unroll
        for (int q = 0; q < 64; ++q) sum[q] = acc[q];
      } else {
#pragma unroll
        for (int q = 0; q < 64; ++q) sum[q] += acc[q];
      }
    }

    const int t0 = mt * kGemmBM + rbase;  // token rows t0 and t0 + 8
    if constexpr (EPI == PREFILL_PLANE) {
      const int n0 = nt * kGemmBM + cq;
      const bool vec = (p.rows_w & 1) == 0;
#pragma unroll
      for (int g = 0; g < 16; ++g) {
        const int n = n0 + 8 * g;
        if (n >= p.rows_w) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int t = t0 + 8 * h;
          if (t >= p.rows_x) continue;
          float* o = p.plane + static_cast<size_t>(t) * p.rows_w + n;
          if (vec) {
            *reinterpret_cast<float2*>(o) = make_float2(sum[4 * g + 2 * h], sum[4 * g + 2 * h + 1]);
          } else {
            o[0] = sum[4 * g + 2 * h];
            if (n + 1 < p.rows_w) o[1] = sum[4 * g + 2 * h + 1];
          }
        }
      }
    } else {
      const int I = p.rows_w / 2;
      const int f0 = nt * 64 + cq;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int t = t0 + 8 * h;
          if (t >= p.rows_x) continue;
          const float a0 = swiglu_bf16(bf16_round(sum[4 * g + 2 * h]), bf16_round(sum[4 * (g + 8) + 2 * h]));
          const float a1 = swiglu_bf16(bf16_round(sum[4 * g + 2 * h + 1]), bf16_round(sum[4 * (g + 8) + 2 * h + 1]));
          *reinterpret_cast<__nv_bfloat162*>(p.act + static_cast<size_t>(t) * I + f0 + 8 * g) = __floats2bfloat162_rn(a0, a1);
        }
      }
    }
  }
}

}  // namespace vlo
