// Prefill GEMM of quantized decoder layers (e4m3 weights, W8A8, int4 weights) for inputs longer than one step:
//   out[t, n] = sum_k X[t, k] * W[n, k]
// over up to max_prefill_tokens token rows, with the bits of the chunked path (gemm_ws_kernel mode 0 on each <= 128-token
// chunk, then the fix-up kernels / the gate|up finisher, on the same weight format).
//
// Schedule as gemm_prefill_kernel (persistent, one CTA per SM, whole 128 x 128 tiles in weight-tile-major order, the
// chunked plan's k-ranges of each weight tile walked from a zeroed accumulator and added in plane order), but with the
// chunked kernels' operand roles: the weights ride wgmma M and the 128 tokens of a tile N.
//   warps 0-3   warpgroup 0: m64n128 on weight rows 0-63 of the tile over the shared token box
//   warps 4-7   warpgroup 1: the same on weight rows 64-127
//   warps 8-11  producer warpgroup, lane 0 of warp 8: per 64-wide k-block one weight stage (TMA box, or the 4 KB int4
//               unit as one bulk copy) and one 128-token activation box
// The producer warpgroup gives its registers to the consumers (setmaxnreg): the running sum and the accumulator of a
// range take 128 registers per thread, and the e4m3 conversion or the int4 fragments would not fit beside them in the
// 168 of an even split.
// Each warpgroup issues exactly the MMAs the chunked kernels issue on its 64-row half (gemm.cuh, wg_mainloop and
// wg_mainloop_i4):
//   FMT_E4M3     the warpgroup upcasts its half of the e4m3 stage into a SWIZZLE_128B bf16 tile of its own (exact), then
//                the bf16 chain; two tiles per warpgroup, each guarded by the warpgroup's own named barrier;
//   FMT_E4M3_A8  the FP8 chain straight from the 64-byte-swizzled stages;
//   FMT_I4       the warpgroup's 2 KB of a unit are the A fragments of its half in the engine byte order, converted in
//                registers (i4_fragment) and fed to the bf16 chain.
// A finished range is scaled as scale_partial scales a partial (fl(P * s[n]); W8A8 then fl(. * a[t]); int4: as is) before
// it is added, so
//   PREFILL_PLANE   writes sum = 0 + P0' + P1' + ... as ONE fp32 plane [rows_x][rows_w] (read through a one-plane SkInfo);
//   PREFILL_SWIGLU  g, u = P0' + P1' + ... (the first range sets the sum), then swiglu_bf16 into act [rows_x][rows_w / 2].
//                   Gate rows 0-63 and up rows 64-127 of a tile sit in different warpgroups: warpgroup 1 passes its
//                   bf16 up values to the same thread of warpgroup 0 through a 16 KB exchange tile.
// One output's wgmma chain has the same bits at every token-tile width (tests/test_gpu_fp8_activations.py,
// tests/test_gpu_int4_weights.py); tests/test_gpu_quant_prefill.py holds this kernel to the chunked path bit for bit.
//
// PDL: the first S weight stages load (and the int4 group scales are pulled into L2) before griddepcontrol.wait.
#pragma once
#include <cuda.h>
#include "gemm_prefill.cuh"
#include "gemm_ws.cuh"

namespace vlo {

struct GemmPrefillQArgs {
  GemmPrefillArgs g;
  WsWeightArgs wt;   // row scales (e4m3), token scales (W8A8), codes and group scales (int4)
};

constexpr int kPrefillQThreads = 384;
constexpr int kPrefillQConsumerRegs = 232, kPrefillQProducerRegs = 40;   // 2 x 128 x 232 + 128 x 40 <= 64 K
static_assert(2 * 128 * kPrefillQConsumerRegs + 128 * kPrefillQProducerRegs <= 65536, "register file of one SM");

template <int FMT, int EPI>
struct GemmPrefillQCfg {
  static_assert(FMT == FMT_E4M3 || FMT == FMT_E4M3_A8 || FMT == FMT_I4, "quantized weight formats only");
  static constexpr int kBytesW = FMT == FMT_I4 ? kI4BytesUnit : kGemmBM * kGemmBK;       // one k-block of a weight tile
  static constexpr int kBytesX = kGemmBM * kGemmBK * (FMT == FMT_E4M3_A8 ? 1 : 2);        // one k-block of 128 tokens
  static constexpr int kBytesHalf = 64 * kGemmBK * 2;                                      // a bf16 64-row tile, 8 KB
  static constexpr int kBytesCvt = FMT == FMT_E4M3 ? 2 * 2 * kBytesHalf : 0;              // 2 per warpgroup
  static constexpr int kBytesXch = EPI == PREFILL_SWIGLU ? 64 * kGemmBM * 2 : 0;          // bf16 up values of a tile
  // 1024 B of slack to align the ring for SWIZZLE_128B, 256 B of barriers
  static constexpr int kFixed = kBytesCvt + kBytesXch + 1024 + 256;
  static constexpr int kStages = fit_stages(kBytesW + kBytesX, kFixed, 10);
  static constexpr int kSmemBytes = kStages * (kBytesW + kBytesX) + kFixed;
  static_assert(kStages >= 4 && kStages <= 16, "the barrier block holds 16 full / empty pairs");
};

// bar.sync for the 128 threads of warpgroup wg (barrier 2 + wg; wg_sync's barrier 1 is the one-warpgroup kernels')
__device__ __forceinline__ void prefill_wg_sync(int wg) { asm volatile("bar.sync %0, 128;\n" ::"r"(2 + wg) : "memory"); }

// warpgroup thread t (0..127) converts a 64-row half of an e4m3 stage, src [64][64 B], into the bf16 tile dst [64][128 B]
// laid out as f8_tile_to_bf16_sw128 lays out a 128-row tile (16-byte chunk c of row r at chunk c ^ (r % 8))
__device__ __forceinline__ void f8_half_to_bf16_sw128(const uint8_t* src, uint8_t* dst, int t) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int idx = j * 128 + t, r = idx >> 3, c = idx & 7;
    const uint2 v = *reinterpret_cast<const uint2*>(src + r * 64 + c * 8);
    const uint4 o = make_uint4(e4m3x2_to_bf16x2(v.x), e4m3x2_to_bf16x2(v.x >> 16), e4m3x2_to_bf16x2(v.y),
                               e4m3x2_to_bf16x2(v.y >> 16));
    *reinterpret_cast<uint4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = o;
  }
}

template <int FMT, int EPI>
__global__ void __launch_bounds__(kPrefillQThreads, 1)
gemm_prefill_q_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                      const __grid_constant__ GemmPrefillQArgs p) {
  using Cfg = GemmPrefillQCfg<FMT, EPI>;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_cvt = smem;
  uint8_t* smem_w = smem + Cfg::kBytesCvt;
  uint8_t* smem_x = smem_w + S * Cfg::kBytesW;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_x + S * Cfg::kBytesX);
  uint64_t* empty_bar = full_bar + S;
  uint32_t* xch = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(full_bar) + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb = p.g.k / kGemmBK;
  const int m_tiles = p.g.m_tiles;
  const int tile0 = static_cast<int>((static_cast<long long>(blockIdx.x) * p.g.tiles) / gridDim.x);
  const int tile1 = static_cast<int>((static_cast<long long>(blockIdx.x + 1) * p.g.tiles) / gridDim.x);
  const long long u0 = static_cast<long long>(tile0) * kb, u1 = static_cast<long long>(tile1) * kb;
  const bool producer = warp == kPrefillProducerWarp && lane == 0;
  // the weight stage of k-block kblk of weight tile nt into ring slot s
  auto load_w = [&](int s, int nt, int kblk) {
    if constexpr (FMT == FMT_I4)
      bulk_load(smem_w + s * Cfg::kBytesW, p.wt.w4 + (static_cast<long long>(nt) * kb + kblk) * kI4BytesUnit, kI4BytesUnit,
                &full_bar[s], kEvictNormal);
    else
      tma_load_2d(smem_w + s * Cfg::kBytesW, &tm_w, &full_bar[s], kblk * kGemmBK, nt * kGemmBM, kEvictNormal);
  };

  if (producer) {
    if constexpr (FMT != FMT_I4) tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_x);
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
      mbar_arrive_expect_tx(&full_bar[pre], Cfg::kBytesW + Cfg::kBytesX);
      load_w(pre, tile / m_tiles, kblk);
    }
  } else if (FMT == FMT_I4 && warp < kPrefillProducerWarp && threadIdx.x < kGemmBM && tile0 < tile1) {
    // the group-scale rows of this CTA's weight tiles into L2, one 128-byte line per 64 scales
    const int ng = p.g.k / kI4Group;
    for (int nt = tile0 / m_tiles; nt <= (tile1 - 1) / m_tiles; ++nt) {
      const int n = nt * kGemmBM + static_cast<int>(threadIdx.x);
      if (n >= p.g.rows_w) break;
      for (int g = 0; g < ng; g += 64) prefetch_l2(p.wt.g_scale + static_cast<size_t>(n) * ng + g);
    }
  }
  // the activations (and W8A8's token scales) are the predecessors' output
  pdl_wait();

  if (warp >= kPrefillProducerWarp) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(kPrefillQProducerRegs));
    if (warp == kPrefillProducerWarp && lane == 0) {
      int i = 0;
      for (long long u = u0; u < u1; ++u, ++i) {
        const int tile = static_cast<int>(u / kb);
        const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
        const int nt = tile / m_tiles, mt = tile - nt * m_tiles;
        const int s = i % S;
        if (i >= pre) {
          mbar_wait(&empty_bar[s], ((i / S) & 1) ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], Cfg::kBytesW + Cfg::kBytesX);
          load_w(s, nt, kblk);
        }
        tma_load_2d(smem_x + s * Cfg::kBytesX, &tm_x, &full_bar[s], kblk * kGemmBK, mt * kGemmBM, kEvictLast);
      }
    }
    return;
  }

  // -------------------------------------------------- consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(kPrefillQConsumerRegs));
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  // accumulator element 4 * g + 2 * e + b of this thread: weight row 64 * wg + wr + 8 * e of the tile, token 8 * g + cq + b
  const int wr = 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
  auto release = [&](int pos) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[pos % S]);
  };
  int i = 0;
  for (int tile = tile0; tile < tile1; ++tile) {
    const int nt = tile / m_tiles, mt = tile - nt * m_tiles;
    const long long t_u0 = static_cast<long long>(nt) * kb;  // the weight tile's first unit in the plan
    const int n_lo = nt * kGemmBM + 64 * wg + wr;             // weight rows n_lo and n_lo + 8
    const bool ok_lo = n_lo < p.g.rows_w, ok_hi = n_lo + 8 < p.g.rows_w;
    const int t0 = mt * kGemmBM + cq;                         // tokens t0 + 8 g + b
    float s_lo = 0.f, s_hi = 0.f;                             // e4m3 row scales
    if constexpr (FMT == FMT_E4M3 || FMT == FMT_E4M3_A8) {
      if (ok_lo) s_lo = __ldg(p.wt.w_scale + n_lo);
      if (ok_hi) s_hi = __ldg(p.wt.w_scale + n_lo + 8);
    }
    const int ng = p.g.k / kI4Group;
    const uint16_t* gs_lo = p.wt.g_scale + static_cast<size_t>(n_lo) * ng;   // int4, read only for rows < rows_w
    const uint16_t* gs_hi = gs_lo + 8 * static_cast<size_t>(ng);
    float sum[64];
#pragma unroll
    for (int q = 0; q < 64; ++q) sum[q] = 0.f;
    // one k-range per contributing CTA of the plan, in plane order
    for (int c = sk_first_cta(nt, p.g.sk), j = 0; j < kb; ++c) {
      const int j_end = static_cast<int>(min(static_cast<long long>(kb), sk_lo(c + 1, p.g.sk) - t_u0));
      const bool first = j == 0;
      float acc[64];
#pragma unroll
      for (int q = 0; q < 64; ++q) acc[q] = 0.f;
      for (int jj = 0; j < j_end; ++j, ++jj, ++i) {
        const int s = i % S;
        if constexpr (FMT == FMT_I4) {
          // the scales of k-block j's group, loaded before the wait
          const uint32_t sl = bf16x2_bcast(ok_lo ? __ldg(gs_lo + j / 2) : 0);
          const uint32_t sh = bf16x2_bcast(ok_hi ? __ldg(gs_hi + j / 2) : 0);
          mbar_wait(&full_bar[s], (i / S) & 1);
          const uint4 cw = *reinterpret_cast<const uint4*>(smem_w + s * Cfg::kBytesW + wg * (kI4BytesUnit / 2) + tid * 16);
          // no MMA in flight while the A registers are written (gemm.cuh, wg_mainloop_i4); the other warpgroup's MMAs
          // keep the tensor cores busy meanwhile
          wgmma_wait<0>();
          if (jj > 0) release(i - 1);
          uint32_t a[4][4];
          i4_fragment(cw.x, sl, sh, a[0]);
          i4_fragment(cw.y, sl, sh, a[1]);
          i4_fragment(cw.z, sl, sh, a[2]);
          i4_fragment(cw.w, sl, sh, a[3]);
          wgmma_fence();
          const uint64_t dx = wgmma_desc_sw128(smem_u32(smem_x + s * Cfg::kBytesX));
#pragma unroll
          for (int kk = 0; kk < kGemmBK / 16; ++kk) WgmmaRegA<128>::mma(acc, a[kk], dx + 2 * kk);
          wgmma_commit();
        } else {
          mbar_wait(&full_bar[s], (i / S) & 1);
          if constexpr (FMT == FMT_E4M3) {
            uint8_t* cvt = smem_cvt + (2 * wg + (i & 1)) * Cfg::kBytesHalf;
            prefill_wg_sync(wg);   // every warp of the warpgroup has retired the MMAs of position i - 2, the tile's readers
            f8_half_to_bf16_sw128(smem_w + s * Cfg::kBytesW + wg * (Cfg::kBytesW / 2), cvt, tid);
            fence_proxy_async();   // the generic-proxy stores become visible to the wgmma operand reads
            prefill_wg_sync(wg);
            wgmma_fence();
            const uint64_t dw = wgmma_desc_sw128(smem_u32(cvt));
            const uint64_t dx = wgmma_desc_sw128(smem_u32(smem_x + s * Cfg::kBytesX));
#pragma unroll
            for (int kk = 0; kk < kGemmBK / 16; ++kk) Wgmma<FMT_BF16, 128>::mma(acc, dw + 2 * kk, dx + 2 * kk);
          } else {
            wgmma_fence();
            // +2 per 32 elements (32 B) along K; the second 64-row half of the weight stage starts 4 KB (+256) further
            const uint64_t dw = wgmma_desc_sw64(smem_u32(smem_w + s * Cfg::kBytesW)) + 256 * wg;
            const uint64_t dx = wgmma_desc_sw64(smem_u32(smem_x + s * Cfg::kBytesX));
#pragma unroll
            for (int kk = 0; kk < kGemmBK / 32; ++kk) WgmmaE4M3<128>::mma(acc, dw + 2 * kk, dx + 2 * kk);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (jj > 0) release(i - 1);
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      release(i - 1);
      // the range's partial, scaled as scale_partial scales it
      if constexpr (FMT == FMT_E4M3 || FMT == FMT_E4M3_A8) {
#pragma unroll
        for (int g = 0; g < 16; ++g)
#pragma unroll
          for (int b = 0; b < 2; ++b) {
            float a_t = 0.f;
            if constexpr (FMT == FMT_E4M3_A8) {
              const int t = t0 + 8 * g + b;
              if (t < p.g.rows_x) a_t = p.wt.a_scale[t];
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float& v = acc[4 * g + 2 * e + b];
              v = __fmul_rn(v, e ? s_hi : s_lo);
              if constexpr (FMT == FMT_E4M3_A8) v = __fmul_rn(v, a_t);
            }
          }
      }
      if (EPI == PREFILL_SWIGLU && first) {
#pragma unroll
        for (int q = 0; q < 64; ++q) sum[q] = acc[q];
      } else {
#pragma unroll
        for (int q = 0; q < 64; ++q) sum[q] += acc[q];
      }
    }

    if constexpr (EPI == PREFILL_PLANE) {
#pragma unroll
      for (int g = 0; g < 16; ++g)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int t = t0 + 8 * g + b;
          if (t >= p.g.rows_x) continue;
          float* o = p.g.plane + static_cast<size_t>(t) * p.g.rows_w + n_lo;
          if (ok_lo) o[0] = sum[4 * g + b];
          if (ok_hi) o[8] = sum[4 * g + 2 + b];
        }
    } else {
      // warpgroup 1 holds the up features of the gate features warpgroup 0 holds, thread for thread
      named_bar_sync<4>(256);   // warpgroup 0 has read the previous tile's up values
      if (wg == 1) {
#pragma unroll
        for (int q = 0; q < 32; ++q) {
          const __nv_bfloat162 u2 = __floats2bfloat162_rn(sum[2 * q], sum[2 * q + 1]);
          xch[q * 128 + tid] = *reinterpret_cast<const uint32_t*>(&u2);
        }
      }
      named_bar_sync<4>(256);
      if (wg == 0) {
        const int I = p.g.rows_w / 2;
        const int f = nt * 64 + wr;   // gate features f and f + 8
#pragma unroll
        for (int q = 0; q < 32; ++q) {
          const uint32_t w = xch[q * 128 + tid];
          const __nv_bfloat162 u2 = *reinterpret_cast<const __nv_bfloat162*>(&w);
          const float up[2] = {__low2float(u2), __high2float(u2)};
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int qq = 2 * q + r, g = qq >> 2, e = (qq >> 1) & 1, b = qq & 1;
            const int t = t0 + 8 * g + b;
            if (t >= p.g.rows_x) continue;
            p.g.act[static_cast<size_t>(t) * I + f + 8 * e] = __float2bfloat16_rn(swiglu_bf16(bf16_round(sum[qq]), up[r]));
          }
        }
      }
    }
  }
}

}  // namespace vlo
