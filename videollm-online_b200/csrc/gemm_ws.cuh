// Persistent weight-streaming GEMM (decoder / connector / lm_head):  out[t, n] = sum_k X[t, k] * W[n, k]
//
// Same wgmma / TMA machinery as gemm.cuh, swap-AB (W rows ride the 128-row M tile, the T <= 128 tokens are
// the wgmma N dimension) and scheduled for an HBM-bound problem:
//   * ONE CTA per SM, resident for the whole GEMM: barrier init and descriptor prefetch
//     are paid once and the TMA ring never drains between work items;
//   * stream-K: the (weight tile, 64-wide k-block) units are dealt out evenly, CTA c owns the contiguous
//     unit range [c*U/G, (c+1)*U/G), so all SMs stream the same number of bytes (no wave
//     quantisation, no tail).  A CTA whose range crosses a tile boundary emits one fp32 partial per tile
//     it touches into plane (c - first_cta_of_tile); the consumer kernels (resid_rmsnorm / qkv_rope /
//     vit_fix_ln) add the planes of each tile in plane order -> deterministic;
//   * TILES mode (lm_head, connector): whole tiles per CTA, direct 16-bit epilogue, no partials;
//   * the producer warp keeps the ring full across items, so the weight stream continues while the warpgroup
//     runs the epilogue of an item;
//   * FMT_E4M3 (mode 0 only): e4m3 weight stages, upcast to bf16 by the warpgroup (wg_mainloop_f8), each partial
//     multiplied by its row's scale once before it is written;
//   * FMT_E4M3_A8 (mode 0 only): e4m3 weight and e4m3 activation stages straight into the FP8 wgmma (wg_mainloop_a8);
//     each partial is multiplied by its row's weight scale, then by its token's activation scale, before it is written;
//   * FMT_I4 (mode 0, one token tile only): 4-bit codes with per-group bf16 scales, dequantized into the wgmma A fragment in
//     registers (wg_mainloop_i4); a ring slot carries up to i4_slot_units(BN) consecutive k-blocks of one tile, the codes
//     as one bulk copy.  The units, their k order and the plane each lands in are those of the bf16 kernel.
#pragma once
#include <cuda.h>
#include "gemm.cuh"
#include "streamk.h"

namespace vlo {

struct GemmWsArgs {
  int rows_w, rows_x, k;   // W [rows_w, k], X [rows_x, k]
  int tiles;               // weight tiles x token tiles
  int x_tiles;             // ceil(rows_x / BN) token tiles (1 for the decoder); tile = w_tile * x_tiles + x_tile
  SkInfo sk;
  int mode;                // 0 = stream-K partials, 1 = whole tiles + 16-bit epilogue
  void* out;               // mode 0: fp32 [plane][rows_x][rows_w]; mode 1: 16-bit [rows_x][ld_out]
  int ld_out;
  long long plane_stride;
  const float* bias;
  int act;
  unsigned long long hint_w;  // L2 policy for the weight stream (evict-first when read once per launch)
  const float* w_scale;       // FMT_E4M3 / FMT_E4M3_A8: [rows_w] fp32 row scales, applied once to each partial
  const float* a_scale;       // FMT_E4M3_A8: [rows_x] fp32 token scales, applied after the row scale
  const uint8_t* w4;          // FMT_I4: the codes in the engine byte order (gemm.cuh)
  const uint16_t* g_scale;    // FMT_I4: bf16 [rows_w][k / 128] group scales
};

// deepest ring of at most 8 stages that fits next to the staging tile
constexpr int ws_default_stages(int bn) { return fit_stages(kGemmBM * kGemmBK * 2 + bn * kGemmBK * 2, kWgStageBytes + 1024 + 256, 8); }
// e4m3 weights: stages of half the weight bytes, so up to 16 of them (the barrier block holds 16 pairs), next to the
// staging tile and the two converted bf16 tiles
constexpr int ws_f8_default_stages(int bn) {
  return fit_stages(kF8BytesW + bn * kGemmBK * 2, kF8BytesCvt + kWgStageBytes + 1024 + 256, 16);
}

// e4m3 weights and activations: up to 16 stages of 8 KB + BN x 64 B next to the staging tile (no conversion tiles)
constexpr int ws_a8_default_stages(int bn) { return fit_stages(kA8BytesW + bn * kGemmBK, kWgStageBytes + 1024 + 256, 16); }

// int4 weights: up to 16 slots of i4_slot_units(BN) k-blocks (codes + activation boxes) next to the staging tile
constexpr int ws_i4_default_stages(int bn) {
  return fit_stages(i4_slot_units(bn) * (kI4BytesUnit + bn * kGemmBK * 2), kWgStageBytes + 1024 + 256, 16);
}

template <int BN, int STAGES = ws_default_stages(BN), int FMT = FMT_BF16>
struct GemmWsCfg {
  static constexpr int kStages = STAGES;
  // FMT_I4: per ring slot
  static constexpr int kBytesA = FMT == FMT_E4M3 ? kF8BytesW : FMT == FMT_E4M3_A8 ? kA8BytesW
                                 : FMT == FMT_I4 ? i4_slot_units(BN) * kI4BytesUnit : kGemmBM * kGemmBK * 2;
  static constexpr int kBytesB = BN * kGemmBK * (FMT == FMT_E4M3_A8 ? 1 : 2) * (FMT == FMT_I4 ? i4_slot_units(BN) : 1);
  static constexpr int kBytesCvt = FMT == FMT_E4M3 ? kF8BytesCvt : 0;
  static constexpr int kSmemBytes = kBytesCvt + kStages * (kBytesA + kBytesB) + 1024 + 256 + kWgStageBytes;
  static_assert(kSmemBytes <= kSmemOptIn, "ring + staging tile exceed the shared memory of one block");
  static_assert(kStages <= 16, "the barrier block holds 16 full / empty pairs");
};

template <int FMT, int BN, int STAGES = ws_default_stages(BN)>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_ws_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
               const GemmWsArgs p) {
  using Cfg = GemmWsCfg<BN, STAGES, FMT>;
  constexpr bool kF8 = FMT == FMT_E4M3;
  constexpr bool kA8 = FMT == FMT_E4M3_A8;
  constexpr bool kI4 = FMT == FMT_I4;
  constexpr int KU = i4_slot_units(BN);
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_cvt = smem;               // kF8: the converted bf16 weight tiles
  uint8_t* smem_a = smem + Cfg::kBytesCvt;
  uint8_t* smem_b = smem + Cfg::kBytesCvt + S * Cfg::kBytesA;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBytesCvt + S * (Cfg::kBytesA + Cfg::kBytesB));
  uint64_t* empty_bar = full_bar + S;
  float* stage = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full_bar) + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x;
  const int kb = p.sk.kb;
  long long u0, u1;
  if (p.mode == 0) {
    u0 = sk_lo(c, p.sk);
    u1 = sk_lo(c + 1, p.sk);
  } else {
    u0 = ((static_cast<long long>(c) * p.tiles) / p.sk.G) * kb;
    u1 = ((static_cast<long long>(c + 1) * p.tiles) / p.sk.G) * kb;
  }
  const bool producer = warp == kGemmProducerWarp && lane == 0;

  if (producer) {
    if constexpr (!kI4) tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_x);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Early triggering lets the next kernels of the step become resident and prefetch while this one streams.
  pdl_trigger();
  // The weight operand never depends on any earlier kernel: the producer starts streaming the first S weight
  // k-blocks right away, i.e. while the predecessors are still running.
  int pre = 0;
  if constexpr (kI4) {
    if (producer) pre = i4_prefetch_codes<BN, S, KU>(p.w4, smem_a, full_bar, u0, u1, kb, p.hint_w);
    else if (warp < kGemmProducerWarp) i4_prefetch_scales(p.g_scale, p.k / kI4Group, p.rows_w, u0, u1, kb);
  } else if (producer) {
    for (long long u = u0; u < u1 && pre < S; ++u, ++pre) {
      const int tile = static_cast<int>(u / kb);
      const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
      const int wt = tile / p.x_tiles;
      mbar_arrive_expect_tx(&full_bar[pre], Cfg::kBytesA + Cfg::kBytesB);
      tma_load_2d(smem_a + pre * Cfg::kBytesA, &tm_w, &full_bar[pre], kblk * kGemmBK, wt * kGemmBM, p.hint_w);
    }
  }
  // everything above overlapped the predecessors; their results (the activations) are needed from here on
  pdl_wait();

  if (warp == kGemmProducerWarp) {
    if constexpr (kI4) {
      if (lane == 0) i4_produce<BN, S, KU>(p.w4, &tm_x, smem_a, smem_b, full_bar, empty_bar, u0, u1, kb, pre, p.hint_w);
    } else if (lane == 0) {
      // ------------------------------------------------ TMA producer: one continuous stream of k-blocks
      int i = 0;
      for (long long u = u0; u < u1; ++u, ++i) {
        const int tile = static_cast<int>(u / kb);
        const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
        const int wt = tile / p.x_tiles, xt = tile - wt * p.x_tiles;
        const int s = i % S;
        if (i >= pre) {
          const uint32_t ph = (i / S) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], Cfg::kBytesA + Cfg::kBytesB);
          tma_load_2d(smem_a + s * Cfg::kBytesA, &tm_w, &full_bar[s], kblk * kGemmBK, wt * kGemmBM, p.hint_w);
        }
        tma_load_2d(smem_b + s * Cfg::kBytesB, &tm_x, &full_bar[s], kblk * kGemmBK, xt * BN, kEvictLast);
      }
    }
  } else {
    // -------------------------------------------------- MMA + epilogue warpgroup (warps 0-3)
    const int row = threadIdx.x;  // tile row (output feature inside the weight tile) this thread finishes
    int i = 0;
    for (long long u = u0; u < u1;) {
      const int tile = static_cast<int>(u / kb);
      const int k0 = static_cast<int>(u - static_cast<long long>(tile) * kb);
      const int nk = static_cast<int>(min(static_cast<long long>(kb - k0), u1 - u));
      u += nk;
      float acc[2][BN / 2];
      if constexpr (kF8)
        wg_mainloop_f8<BN, S>(acc, smem_cvt, smem_a, smem_b, full_bar, empty_bar, i, nk);
      else if constexpr (kA8)
        wg_mainloop_a8<BN, S>(acc, smem_a, smem_b, full_bar, empty_bar, i, nk);
      else if constexpr (kI4)
        wg_mainloop_i4<BN, S, KU>(acc, smem_a, smem_b, full_bar, empty_bar, i, tile, k0, nk, p.g_scale, p.k / kI4Group,
                                  p.rows_w);
      else
        wg_mainloop<FMT, BN, S>(acc, smem_a, smem_b, full_bar, empty_bar, i, nk);
      const int wt = tile / p.x_tiles, xt = tile - wt * p.x_tiles;
      const int n = wt * kGemmBM + row;  // output feature (row of W)
      const int t0 = xt * BN;            // first token row of this tile
      const bool n_ok = n < p.rows_w;
      float* plane = nullptr;
      float bias_n = 0.f;
      float scale_n = 0.f;
      if constexpr (kF8 || kA8) {
        if (n_ok) scale_n = __ldg(p.w_scale + n);
      }
      if (p.mode == 0) {
        const int pl = c - sk_first_cta(tile, p.sk);
        plane = reinterpret_cast<float*>(p.out) + static_cast<size_t>(pl) * p.plane_stride;
      } else if (p.bias != nullptr && n_ok) {
        bias_n = __ldg(p.bias + n);
      }
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += kWgChunk) {
        wg_sync();                            // the previous chunk's readers are done with the staging tile
        wg_stage_chunk<BN>(acc, c0, stage);
        wg_sync();
        if (!n_ok || t0 + c0 >= p.rows_x) continue;
        float v[16];
        wg_load16(stage, row, v);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int t = t0 + c0 + j;
          if (t >= p.rows_x) break;
          const float acc = v[j];
          if constexpr (kF8) {
            plane[static_cast<size_t>(t) * p.rows_w + n] = __fmul_rn(acc, scale_n);   // the one rounding of the scale
          } else if constexpr (kA8) {
            // a_scale is the quantizer's output: a plain load, after pdl_wait
            plane[static_cast<size_t>(t) * p.rows_w + n] = __fmul_rn(__fmul_rn(acc, scale_n), p.a_scale[t]);
          } else if (p.mode == 0) {
            plane[static_cast<size_t>(t) * p.rows_w + n] = acc;
          } else {
            float x = r16<FMT>(acc + bias_n);
            x = apply_act<FMT>(x, p.act);
            reinterpret_cast<uint16_t*>(p.out)[static_cast<size_t>(t) * p.ld_out + n] = to16<FMT>(x);
          }
        }
      }
    }
  }
}

}  // namespace vlo
