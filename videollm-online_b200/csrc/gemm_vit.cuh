// ViT trunk GEMM for one or two frames (576 / 1152 token rows) with the fp16 epilogue of QKV and fc1:
//   out[t, n] = r16(act(r16(sum_k X[t, k] * W[n, k] + bias[n])))
//
// The problem is tensor-bound, so the tokens ride wgmma M and each CTA computes a 128-token x 128-feature tile:
//   warps 0-3   warpgroup 0: wgmma m64n128k16 on token rows 0-63 of the tile
//   warps 4-7   warpgroup 1: the same on token rows 64-127
//   warp 8      TMA producer: one 16 KB X box and one 16 KB W box per 64-wide k-block
// Both warpgroups read the shared W box, so one k-block moves 32 KB into shared memory for 2.1 MFLOP (64 FLOP/B; a
// 64-token swap-AB tile of gemm_ws_kernel moves 24 KB for 1 MFLOP).  The 3-stage ring (97 KB) leaves room on the SM for
// a decoder weight-streaming CTA, so the ViT of the next frame still runs beside the decoder step (gemm.cu checks it).
//
// Each output element is the same chain of fp32 wgmma accumulations over the whole of K, in k order, as in the
// swap-AB kernel, so the two produce the same bits (tests/test_gpu_vit_gemm.py).  out_proj and fc2 are not run here:
// their stream-K partial planes sum in an order fixed by the 64-token decomposition of gemm_ws_kernel.
//
// Persistent, one CTA per SM: CTA c owns tiles [c * tiles / G, (c + 1) * tiles / G), tile = feature tile * m_tiles +
// token tile; the producer keeps the ring full across tiles while the warpgroups run the epilogue, which writes
// straight from the accumulator registers.  Token rows past rows_x (576 = 4 x 128 + 64) are zero-filled by the TMA
// unit and never stored.
#pragma once
#include <cuda.h>
#include "gemm.cuh"

namespace vlo {

struct GemmVitArgs {
  int rows_x, rows_w, k;  // X [rows_x, k] (tokens), W [rows_w, k]
  int m_tiles;            // ceil(rows_x / 128)
  int tiles;              // m_tiles * ceil(rows_w / 128)
  __half* out;            // [rows_x][ld_out]
  int ld_out;
  const float* bias;      // [rows_w] or nullptr
  int act;
};

constexpr int kVitGemmStages = 3;
constexpr int kVitGemmThreads = 288;
constexpr int kVitGemmProducerWarp = 8;

struct GemmVitCfg {
  static constexpr int kBytesX = kGemmBM * kGemmBK * 2;
  static constexpr int kBytesW = kGemmBM * kGemmBK * 2;
  // 1024 B of slack to align the ring for SWIZZLE_128B, 256 B of barriers
  static constexpr int kSmemBytes = kVitGemmStages * (kBytesX + kBytesW) + 1024 + 256;
};

__global__ void __launch_bounds__(kVitGemmThreads, 1)
gemm_vit_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                const GemmVitArgs p) {
  using Cfg = GemmVitCfg;
  constexpr int S = kVitGemmStages;
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
  const bool producer = warp == kVitGemmProducerWarp && lane == 0;

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
  // weights never depend on an earlier kernel: the first S weight boxes load while the predecessors still run
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

  if (warp == kVitGemmProducerWarp) {
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
    float acc[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.f;
    // one k-block of MMAs stays in flight while the next stage is awaited; a stage is released once its MMAs retire
    for (int j = 0; j < kb; ++j, ++i) {
      const int s = i % S;
      mbar_wait(&full_bar[s], (i / S) & 1);
      wgmma_fence();
      const uint64_t dx = wgmma_desc_sw128(smem_u32(smem_x + s * Cfg::kBytesX + wg * (Cfg::kBytesX / 2)));
      const uint64_t dw = wgmma_desc_sw128(smem_u32(smem_w + s * Cfg::kBytesW));
#pragma unroll
      for (int kk = 0; kk < kGemmBK / 16; ++kk) Wgmma<FMT_F16, 128>::mma(acc, dx + 2 * kk, dw + 2 * kk);
      wgmma_commit();
      wgmma_wait<1>();
      if (j > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % S]);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % S]);

    const int nt = tile / p.m_tiles, mt = tile - nt * p.m_tiles;
    const int t0 = mt * kGemmBM + rbase;  // token rows t0 and t0 + 8
    const int n0 = nt * kGemmBM + cq;
#pragma unroll
    for (int g = 0; g < 16; ++g) {
      const int n = n0 + 8 * g;
      if (n >= p.rows_w) continue;
      const bool pair = n + 1 < p.rows_w;
      float b0 = 0.f, b1 = 0.f;
      if (p.bias != nullptr) {
        b0 = __ldg(p.bias + n);
        if (pair) b1 = __ldg(p.bias + n + 1);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t = t0 + 8 * h;
        if (t >= p.rows_x) continue;
        const float x0 = apply_act<FMT_F16>(r16<FMT_F16>(acc[4 * g + 2 * h] + b0), p.act);
        const float x1 = apply_act<FMT_F16>(r16<FMT_F16>(acc[4 * g + 2 * h + 1] + b1), p.act);
        __half* o = p.out + static_cast<size_t>(t) * p.ld_out + n;
        if (pair) {
          *reinterpret_cast<__half2*>(o) = __floats2half2_rn(x0, x1);
        } else {
          *o = __float2half_rn(x0);
        }
      }
    }
  }
}

}  // namespace vlo
