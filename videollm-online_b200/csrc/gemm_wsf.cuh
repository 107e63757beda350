// Persistent stream-K weight-streaming GEMM with the SwiGLU fix-up FUSED into its epilogue (the decoder's gate|up):
//   out[t, n] = sum_k X[t, k] * W[n, k]      X = the step's <= 128 tokens (MMA-N), W rows ride MMA-M (128-row tiles)
//
// Same TMA ring / wgmma / stream-K schedule as gemm_ws.cuh (CTA c owns the contiguous unit range [c*U/G, (c+1)*U/G),
// unit = (weight tile, 64-wide k-block)), but the partial sums of a tile no longer go through a separate fix-up kernel:
//   * the FIRST contributing CTA of a tile is its finisher.  It works on the tile's k-blocks LAST (the tail of its unit
//     range), whereas every other contributor meets the tile at the very START of its range - so by the time the
//     finisher's accumulator is complete the other partials have long been published;
//   * contributors write their fp32 partial plane, fence, and bump the tile's arrival counter (flags[tile]);
//   * the finisher waits for the counter (normally already there), adds the planes in plane order to its own
//     accumulator (deterministic), resets the counter and applies SwiGLU:
//       act = bf16(bf16(silu(g)) * u)  with gate / up rows interleaved per tile (64 + 64)   (HF:...llama.py:182-184)
//     gate and up are finished by different threads: they are exchanged through a small shared-memory tile.
// Only gate|up has enough tiles to amortise the finisher tail; q|k|v, o_proj and down_proj leave fp32 planes to the
// fix-up kernels of decoder_kernels.cuh, whose rounding points this epilogue shares.
// The weight formats are those of gemm_ws_kernel, with its ring and partial scaling: for e4m3 weights every contributor,
// the finisher's own accumulator included, multiplies its fp32 partial of feature n by the row scale w_scale[n] once
// before the plane sum, and for e4m3 activations then by the token scale a_scale[t]; int4 weights run the bf16 kernel's
// units, planes and epilogue, so their output is the bf16 kernel's on W4.
// All CTAs of the grid are co-resident or become so without depending on a waiting CTA (grid <= #SMs, the PDL successor
// cannot start before every CTA of this grid has started), so the finisher's wait cannot dead-lock; it is bounded anyway.
#pragma once
#include <cuda.h>
#include "gemm_ws.cuh"
#include "streamk.h"

namespace vlo {

struct GemmWsfArgs {
  int rows_w, rows_x, k;
  SkInfo sk;
  float* planes;              // fp32 [plane - 1][rows_x][rows_w]: partials of the non-finisher contributors
  long long plane_stride;
  int* flags;                 // [tiles] arrival counters; zero between launches (the finisher resets them)
  unsigned long long hint_w;
  __nv_bfloat16* act;         // [rows_x, I]
  int I;
  WsWeightArgs wt;
};

constexpr int kWsfXchStride = 17;   // floats per feature row of the exchange tile (16 tokens + 1: conflict-free)
constexpr int kWsfXchBytes = kGemmBM * kWsfXchStride * 4;

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// p is __grid_constant__ so that its fields are read from parameter space where used: ptxas otherwise copies a struct
// this small up front, which costs the 64- and 128-token instances registers.  FMT is FMT_BF16, FMT_E4M3, FMT_E4M3_A8 or
// FMT_I4 (tm_w unused: the codes stream as bulk copies).
template <int FMT, int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wsf_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
                const __grid_constant__ GemmWsfArgs p) {
  using Cfg = GemmWsCfg<FMT, BN, STAGES, kWsfXchBytes>;
  constexpr int S = Cfg::kStages;
  const WsRing r = ws_ring<Cfg>();
  float* xch = r.tail;   // [128][17] exchange tile
  float* stage = xch + kGemmBM * kWsfXchStride;

  const float* a_scale = p.wt.a_scale;   // FMT_E4M3_A8
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x;
  const int kb = p.sk.kb;
  const long long u0 = sk_lo(c, p.sk), u1 = sk_lo(c + 1, p.sk);
  const bool producer = warp == kGemmProducerWarp && lane == 0;
  const int pre = ws_prologue<FMT, BN, S>(tm_w, tm_x, r, p, u0, u1, kb, 1, warp, producer);

  if (warp == kGemmProducerWarp) {
    if (lane == 0) ws_produce<FMT, BN, S>(tm_w, tm_x, r, p, u0, u1, kb, 1, pre);
  } else {
    // -------------------------------------------------- MMA + epilogue warpgroup: contributor or finisher per item
    const int d = threadIdx.x;            // row of the weight tile (output feature inside the tile)
    int i = 0;
    for (long long u = u0; u < u1;) {
      const int tile = static_cast<int>(u / kb);
      const int k0 = static_cast<int>(u - static_cast<long long>(tile) * kb);
      const int nk = static_cast<int>(min(static_cast<long long>(kb - k0), u1 - u));
      u += nk;
      float acc[2][BN / 2];
      ws_mainloop<FMT, BN, S>(acc, r, p, i, tile, k0, nk);
      const int pl = c - sk_first_cta(tile, p.sk);
      const int n_planes = sk_planes(tile, p.sk);
      const int n = tile * kGemmBM + d;
      const bool n_ok = n < p.rows_w;
      const float scale_n = ws_row_scale<FMT>(p.wt.w_scale, n, n_ok);
      if (pl > 0) {
        // ---- contributor: publish the partial plane, then bump the tile's arrival counter
        float* plane = p.planes + static_cast<size_t>(pl - 1) * p.plane_stride;
#pragma unroll
        for (int c0 = 0; c0 < BN; c0 += kWgChunk) {
          wg_sync();                                  // the previous chunk's readers are done with the staging tile
          wg_stage_chunk<BN>(acc, c0, stage);
          wg_sync();
          if (!n_ok || c0 >= p.rows_x) continue;
          float v[16];
          wg_load16(stage, d, v);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int t = c0 + j;
            if (t >= p.rows_x) break;
            __stcg(plane + static_cast<size_t>(t) * p.rows_w + n, scale_partial<FMT>(v[j], scale_n, a_scale, t));
          }
        }
        __threadfence();
        wg_sync();
        if (d == 0) atomicAdd(p.flags + tile, 1);
        continue;
      }
      // ---- finisher
      if (n_planes > 1) {
        if (d == 0) {
          uint32_t spins = 0;
          while (ld_acquire_gpu(p.flags + tile) < n_planes - 1) {
            __nanosleep(32);
            if (++spins > (1u << 22)) {
#if VLO_MBAR_TRACE
              printf("vlo: stream-K finisher timeout cta %d tile %d\n", c, tile);
#endif
              __trap();
            }
          }
          p.flags[tile] = 0;   // next launch starts from zero again (no other reader or writer is left)
        }
        wg_sync();
        __threadfence();
      }
#pragma unroll
      for (int c0 = 0; c0 < BN; c0 += kWgChunk) {
        if (c0 >= p.rows_x) continue;    // (uniform over the warpgroup: the barriers below stay aligned)
        wg_sync();                            // the previous chunk's readers are done with the staging tile
        wg_stage_chunk<BN>(acc, c0, stage);
        wg_sync();
        float x[16];
        wg_load16(stage, d, x);
        if constexpr (FMT == FMT_E4M3 || FMT == FMT_E4M3_A8) {
          // the finisher's own partial, before the sum; a_scale has rows_x entries
#pragma unroll
          for (int j = 0; j < 16; ++j)
            x[j] = FMT == FMT_E4M3 || c0 + j < p.rows_x ? scale_partial<FMT>(x[j], scale_n, a_scale, c0 + j) : 0.f;
        }
        for (int s2 = 1; s2 < n_planes; ++s2) {   // plane order: deterministic
          const float* plane = p.planes + static_cast<size_t>(s2 - 1) * p.plane_stride + n;
          float a[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) a[j] = (n_ok && c0 + j < p.rows_x) ? __ldcg(plane + static_cast<size_t>(c0 + j) * p.rows_w) : 0.f;
#pragma unroll
          for (int j = 0; j < 16; ++j) x[j] += a[j];
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) x[j] = bf16_round(x[j]);    // the Linear output in bf16
        // tile rows 0..63 = gate features 64*tile.., rows 64..127 = the matching up features
        if (d >= 64) {
#pragma unroll
          for (int j = 0; j < 16; ++j) xch[(d - 64) * kWsfXchStride + j] = x[j];
        }
        wg_sync();
        if (d < 64) {
          const int f = tile * 64 + d;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int t = c0 + j;
            if (t >= p.rows_x) break;
            p.act[static_cast<size_t>(t) * p.I + f] = __float2bfloat16_rn(swiglu_bf16(x[j], xch[d * kWsfXchStride + j]));
          }
        }
        wg_sync();
      }
    }
  }
}

}  // namespace vlo
