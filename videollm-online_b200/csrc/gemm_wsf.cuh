// Persistent stream-K weight-streaming GEMM with the SwiGLU fix-up FUSED into its epilogue (the decoder's gate|up, bf16):
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
// gemm_wsf_f8_kernel runs the same schedule on e4m3 weights (FMT_E4M3, gemm.cuh): every contributor, the finisher's own
// accumulator included, multiplies its fp32 partial of feature n by the row scale w_scale[n] once before the plane sum.
// gemm_wsf_a8_kernel runs it on e4m3 weights and e4m3 activations (FMT_E4M3_A8): every partial of feature n, token t is
// fl(fl(P * w_scale[n]) * a_scale[t]) before the plane sum.
// gemm_wsf_i4_kernel runs it on int4 weights (FMT_I4, gemm.cuh): the same units and planes as the bf16 kernel in the
// int4 ring slots of gemm_ws_kernel, and the bf16 kernel's epilogue, so its output is the bf16 kernel's on W4.
// All CTAs of the grid are co-resident or become so without depending on a waiting CTA (grid <= #SMs, the PDL successor
// cannot start before every CTA of this grid has started), so the finisher's wait cannot dead-lock; it is bounded anyway.
#pragma once
#include <cuda.h>
#include "gemm.cuh"
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
};

constexpr int kWsfXchStride = 17;   // floats per feature row of the exchange tile (16 tokens + 1: conflict-free)

template <int BN, int STAGES, int FMT = FMT_BF16>
struct GemmWsfCfg {
  static constexpr int kStages = STAGES;
  // FMT_I4: per ring slot
  static constexpr int kBytesA = FMT == FMT_E4M3 ? kF8BytesW : FMT == FMT_E4M3_A8 ? kA8BytesW
                                 : FMT == FMT_I4 ? i4_slot_units(BN) * kI4BytesUnit : kGemmBM * kGemmBK * 2;
  static constexpr int kBytesB = BN * kGemmBK * (FMT == FMT_E4M3_A8 ? 1 : 2) * (FMT == FMT_I4 ? i4_slot_units(BN) : 1);
  static constexpr int kBytesCvt = FMT == FMT_E4M3 ? kF8BytesCvt : 0;
  static constexpr int kXchBytes = kGemmBM * kWsfXchStride * 4;
  static constexpr int kSmemBytes = kBytesCvt + kStages * (kBytesA + kBytesB) + 1024 + 256 + kXchBytes + kWgStageBytes;
  static_assert(kSmemBytes <= kSmemOptIn, "ring + exchange + staging tiles exceed the shared memory of one block");
  static_assert(kStages <= 16, "the barrier block holds 16 full / empty pairs");
};
// deepest ring of at most 8 stages that fits next to the exchange and staging tiles
constexpr int wsf_default_stages(int bn) {
  return fit_stages(kGemmBM * kGemmBK * 2 + bn * kGemmBK * 2, 1024 + 256 + kGemmBM * kWsfXchStride * 4 + kWgStageBytes, 8);
}
// e4m3 weights: up to 16 half-size stages next to the converted bf16 tiles, the exchange and the staging tile
constexpr int wsf_f8_default_stages(int bn) {
  return fit_stages(kF8BytesW + bn * kGemmBK * 2, kF8BytesCvt + 1024 + 256 + kGemmBM * kWsfXchStride * 4 + kWgStageBytes, 16);
}
// e4m3 weights and activations: up to 16 stages next to the exchange and the staging tile
constexpr int wsf_a8_default_stages(int bn) {
  return fit_stages(kA8BytesW + bn * kGemmBK, 1024 + 256 + kGemmBM * kWsfXchStride * 4 + kWgStageBytes, 16);
}

// int4 weights: up to 16 slots of i4_slot_units(bn) k-blocks next to the exchange and the staging tile
constexpr int wsf_i4_default_stages(int bn) {
  return fit_stages(i4_slot_units(bn) * (kI4BytesUnit + bn * kGemmBK * 2), 1024 + 256 + kGemmBM * kWsfXchStride * 4 + kWgStageBytes, 16);
}

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// The body of the kernels below; FMT is FMT_BF16, FMT_E4M3, FMT_E4M3_A8 or FMT_I4 (tm_w unused: w4 and g_scale instead).  p by value: ptxas then still reads
// the fields from parameter space where used (the bf16 kernels compile to the same code as with the body inline).
template <int FMT, int BN, int STAGES>
__device__ __forceinline__ void gemm_wsf_body(const CUtensorMap& tm_w, const CUtensorMap& tm_x, const GemmWsfArgs p,
                                              const float* w_scale, const float* a_scale = nullptr,
                                              const uint8_t* w4 = nullptr, const uint16_t* g_scale = nullptr) {
  using Cfg = GemmWsfCfg<BN, STAGES, FMT>;
  constexpr bool kF8 = FMT == FMT_E4M3;
  constexpr bool kA8 = FMT == FMT_E4M3_A8;
  constexpr bool kI4 = FMT == FMT_I4;
  constexpr int KU = i4_slot_units(BN);
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* smem_cvt = smem;               // kF8: the converted bf16 weight tiles
  uint8_t* smem_a = smem + Cfg::kBytesCvt;
  uint8_t* smem_b = smem + Cfg::kBytesCvt + S * Cfg::kBytesA;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBytesCvt + S * (Cfg::kBytesA + Cfg::kBytesB));
  uint64_t* empty_bar = full_bar + S;
  float* xch = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full_bar) + 256);   // [128][17] exchange tile
  float* stage = xch + kGemmBM * kWsfXchStride;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x;
  const int kb = p.sk.kb;
  const long long u0 = sk_lo(c, p.sk), u1 = sk_lo(c + 1, p.sk);
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
  pdl_trigger();
  // the weight operand never depends on an earlier kernel: fill the ring while the predecessors are still running
  int pre = 0;
  if constexpr (kI4) {
    if (producer) pre = i4_prefetch_codes<BN, S, KU>(w4, smem_a, full_bar, u0, u1, kb, p.hint_w);
    else if (warp < kGemmProducerWarp) i4_prefetch_scales(g_scale, p.k / kI4Group, p.rows_w, u0, u1, kb);
  } else if (producer) {
    for (long long u = u0; u < u1 && pre < S; ++u, ++pre) {
      const int tile = static_cast<int>(u / kb);
      const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
      mbar_arrive_expect_tx(&full_bar[pre], Cfg::kBytesA + Cfg::kBytesB);
      tma_load_2d(smem_a + pre * Cfg::kBytesA, &tm_w, &full_bar[pre], kblk * kGemmBK, tile * kGemmBM, p.hint_w);
    }
  }
  pdl_wait();

  if (warp == kGemmProducerWarp) {
    if constexpr (kI4) {
      if (lane == 0) i4_produce<BN, S, KU>(w4, &tm_x, smem_a, smem_b, full_bar, empty_bar, u0, u1, kb, pre, p.hint_w);
    } else if (lane == 0) {
      // ------------------------------------------------ TMA producer: one continuous stream of k-blocks
      int i = 0;
      for (long long u = u0; u < u1; ++u, ++i) {
        const int tile = static_cast<int>(u / kb);
        const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
        const int s = i % S;
        if (i >= pre) {
          const uint32_t ph = (i / S) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          mbar_arrive_expect_tx(&full_bar[s], Cfg::kBytesA + Cfg::kBytesB);
          tma_load_2d(smem_a + s * Cfg::kBytesA, &tm_w, &full_bar[s], kblk * kGemmBK, tile * kGemmBM, p.hint_w);
        }
        tma_load_2d(smem_b + s * Cfg::kBytesB, &tm_x, &full_bar[s], kblk * kGemmBK, 0, kEvictLast);
      }
    }
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
      if constexpr (kF8)
        wg_mainloop_f8<BN, S>(acc, smem_cvt, smem_a, smem_b, full_bar, empty_bar, i, nk);
      else if constexpr (kA8)
        wg_mainloop_a8<BN, S>(acc, smem_a, smem_b, full_bar, empty_bar, i, nk);
      else if constexpr (kI4)
        wg_mainloop_i4<BN, S, KU>(acc, smem_a, smem_b, full_bar, empty_bar, i, tile, k0, nk, g_scale, p.k / kI4Group,
                                  p.rows_w);
      else
        wg_mainloop<FMT_BF16, BN, S>(acc, smem_a, smem_b, full_bar, empty_bar, i, nk);
      const int pl = c - sk_first_cta(tile, p.sk);
      const int n_planes = sk_planes(tile, p.sk);
      const int n = tile * kGemmBM + d;
      const bool n_ok = n < p.rows_w;
      float scale_n = 0.f;
      if constexpr (kF8 || kA8) {
        if (n_ok) scale_n = __ldg(w_scale + n);
      }
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
            if constexpr (kF8)
              __stcg(plane + static_cast<size_t>(t) * p.rows_w + n, __fmul_rn(v[j], scale_n));
            else if constexpr (kA8)
              __stcg(plane + static_cast<size_t>(t) * p.rows_w + n, __fmul_rn(__fmul_rn(v[j], scale_n), a_scale[t]));
            else
              __stcg(plane + static_cast<size_t>(t) * p.rows_w + n, v[j]);
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
        if constexpr (kF8) {
#pragma unroll
          for (int j = 0; j < 16; ++j) x[j] = __fmul_rn(x[j], scale_n);   // the finisher's own partial, before the sum
        }
        if constexpr (kA8) {
#pragma unroll
          for (int j = 0; j < 16; ++j) x[j] = c0 + j < p.rows_x ? __fmul_rn(__fmul_rn(x[j], scale_n), a_scale[c0 + j]) : 0.f;
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

// p is __grid_constant__ so that its fields are read from parameter space where used: ptxas otherwise copies a struct
// this small up front, which costs the 64- and 128-token instances registers.
template <int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wsf_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
                const __grid_constant__ GemmWsfArgs p) {
  gemm_wsf_body<FMT_BF16, BN, STAGES>(tm_w, tm_x, p, nullptr);
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wsf_f8_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
                   const __grid_constant__ GemmWsfArgs p, const float* __restrict__ w_scale) {
  gemm_wsf_body<FMT_E4M3, BN, STAGES>(tm_w, tm_x, p, w_scale);
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wsf_a8_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
                   const __grid_constant__ GemmWsfArgs p, const float* __restrict__ w_scale, const float* a_scale) {
  gemm_wsf_body<FMT_E4M3_A8, BN, STAGES>(tm_w, tm_x, p, w_scale, a_scale);
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wsf_i4_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ GemmWsfArgs p,
                   const uint8_t* __restrict__ w4, const uint16_t* __restrict__ g_scale) {
  gemm_wsf_body<FMT_I4, BN, STAGES>(tm_x, tm_x, p, nullptr, nullptr, w4, g_scale);
}

}  // namespace vlo
