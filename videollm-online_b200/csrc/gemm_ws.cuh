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
//   * FMT_E4M3 and FMT_I4 also run whole tiles (the vocabulary matrices), in gemm_ws_tiles_kernel instances of their own
//     so that the instances the layers run keep their code (gemm.cuh, ws_tiles_own_instances);
//   * FMT_E4M3 (mode 0 only in gemm_ws_kernel): e4m3 weight stages, upcast to bf16 by the warpgroup (wg_mainloop), each
//     partial multiplied by its row's scale once before it is written;
//   * FMT_E4M3_A8 (mode 0 only): e4m3 weight and e4m3 activation stages straight into the FP8 wgmma (wg_mainloop);
//     each partial is multiplied by its row's weight scale, then by its token's activation scale, before it is written;
//   * FMT_I4 (mode 0 only in gemm_ws_kernel, one token tile only): 4-bit codes with per-group bf16 scales, dequantized
//     into the wgmma A fragment in registers (wg_mainloop_i4); a ring slot carries up to i4_slot_units(BN) consecutive k-blocks of one tile, the codes
//     as one bulk copy.  The units, their k order and the plane each lands in are those of the bf16 kernel.
#pragma once
#include <cuda.h>
#include "gemm.cuh"
#include "streamk.h"

namespace vlo {

// The weight side of a weight-streaming launch beyond the TMA map of 16-bit and e4m3 weights
struct WsWeightArgs {
  const float* w_scale;       // FMT_E4M3 / FMT_E4M3_A8: [rows_w] fp32 row scales, applied once to each partial
  const float* a_scale;       // FMT_E4M3_A8: [rows_x] fp32 token scales, applied after the row scale
  const uint8_t* w4;          // FMT_I4: the codes in the engine byte order (gemm.cuh)
  const uint16_t* g_scale;    // FMT_I4: bf16 [rows_w][k / 128] group scales
};

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
  WsWeightArgs wt;
};

// ---- the front half of the weight-streaming kernels (this file and gemm_wsf.cuh).  A CTA owns the units [u0, u1) of
// its plan; unit u is k-block u % kb of tile u / kb, and tile t multiplies weight tile t / x_tiles by token tile
// t % x_tiles (the fused kernel passes x_tiles = 1).  Args is GemmWsArgs or GemmWsfArgs: the helpers read the fields
// both have (rows_w, k, hint_w, wt) where they use them, as the kernel bodies did.

// Shared memory: [conversion tiles][S weight slots][S activation slots][barriers, 256 B][the kernel's own tiles at tail]
struct WsRing {
  uint8_t *cvt, *a, *b;
  uint64_t *full_bar, *empty_bar;
  float* tail;
};
template <class Cfg>
__device__ __forceinline__ WsRing ws_ring() {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  constexpr int S = Cfg::kStages;
  WsRing r;
  r.cvt = smem;   // FMT_E4M3: the converted bf16 weight tiles
  r.a = smem + Cfg::kBytesCvt;
  r.b = smem + Cfg::kBytesCvt + S * Cfg::kBytesA;
  r.full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBytesCvt + S * (Cfg::kBytesA + Cfg::kBytesB));
  r.empty_bar = r.full_bar + S;
  r.tail = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(r.full_bar) + 256);
  return r;
}

// Barrier init and the PDL trigger, then the weight prefetch, then pdl_wait.  The weight operand never depends on an
// earlier kernel: the producer fills the first S slots with weights (and the consumer warps pull the int4 group scales
// into L2) while the predecessors are still running.  Returns the number of slots the producer has filled.
template <int FMT, int BN, int S, class Args>
__device__ __forceinline__ int ws_prologue(const CUtensorMap& tm_w, const CUtensorMap& tm_x, const WsRing& r, const Args& p,
                                           long long u0, long long u1, int kb, int x_tiles, int warp, bool producer) {
  constexpr int kBytesA = ws_slot_bytes_w(FMT, BN), kBytesB = ws_slot_bytes_x(FMT, BN);
  if (producer) {
    if constexpr (FMT != FMT_I4) tma_prefetch_desc(&tm_w);
    tma_prefetch_desc(&tm_x);
    for (int s = 0; s < S; ++s) {
      mbar_init(&r.full_bar[s], 1);
      mbar_init(&r.empty_bar[s], 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // Early triggering lets the next kernels of the step become resident and prefetch while this one streams.
  pdl_trigger();
  int pre = 0;
  if constexpr (FMT == FMT_I4) {
    if (producer) pre = i4_prefetch_codes<BN, S, i4_slot_units(BN)>(p.wt.w4, r.a, r.full_bar, u0, u1, kb, p.hint_w);
    else if (warp < kGemmProducerWarp) i4_prefetch_scales(p.wt.g_scale, p.k / kI4Group, p.rows_w, u0, u1, kb);
  } else if (producer) {
    for (long long u = u0; u < u1 && pre < S; ++u, ++pre) {
      const int tile = static_cast<int>(u / kb);
      const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
      const int wt = tile / x_tiles;
      mbar_arrive_expect_tx(&r.full_bar[pre], kBytesA + kBytesB);
      tma_load_2d(r.a + pre * kBytesA, &tm_w, &r.full_bar[pre], kblk * kGemmBK, wt * kGemmBM, p.hint_w);
    }
  }
  // everything above overlapped the predecessors; their results (the activations) are needed from here on
  pdl_wait();
  return pre;
}

// The producer (lane 0 of the producer warp): one continuous stream of ring slots; the first `pre` slots only still
// need their activation boxes.
template <int FMT, int BN, int S, class Args>
__device__ __forceinline__ void ws_produce(const CUtensorMap& tm_w, const CUtensorMap& tm_x, const WsRing& r, const Args& p,
                                           long long u0, long long u1, int kb, int x_tiles, int pre) {
  constexpr int kBytesA = ws_slot_bytes_w(FMT, BN), kBytesB = ws_slot_bytes_x(FMT, BN);
  if constexpr (FMT == FMT_I4) {
    i4_produce<BN, S, i4_slot_units(BN)>(p.wt.w4, &tm_x, r.a, r.b, r.full_bar, r.empty_bar, u0, u1, kb, pre, p.hint_w);
  } else {
    int i = 0;
    for (long long u = u0; u < u1; ++u, ++i) {
      const int tile = static_cast<int>(u / kb);
      const int kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
      const int wt = tile / x_tiles, xt = tile - wt * x_tiles;
      const int s = i % S;
      if (i >= pre) {
        const uint32_t ph = (i / S) & 1;
        mbar_wait(&r.empty_bar[s], ph ^ 1);
        mbar_arrive_expect_tx(&r.full_bar[s], kBytesA + kBytesB);
        tma_load_2d(r.a + s * kBytesA, &tm_w, &r.full_bar[s], kblk * kGemmBK, wt * kGemmBM, p.hint_w);
      }
      tma_load_2d(r.b + s * kBytesB, &tm_x, &r.full_bar[s], kblk * kGemmBK, xt * BN, kEvictLast);
    }
  }
}

// The warpgroup's main loop over the nk k-blocks k0 .. of tile `tile`, in the format's ring slots
template <int FMT, int BN, int S, class Args>
__device__ __forceinline__ void ws_mainloop(float (&acc)[2][BN / 2], const WsRing& r, const Args& p, int& i, int tile,
                                            int k0, int nk) {
  if constexpr (FMT == FMT_I4)
    wg_mainloop_i4<BN, S, i4_slot_units(BN)>(acc, r.a, r.b, r.full_bar, r.empty_bar, i, tile, k0, nk, p.wt.g_scale,
                                             p.k / kI4Group, p.rows_w);
  else
    wg_mainloop<FMT, BN, S>(acc, r.a, r.b, r.full_bar, r.empty_bar, i, nk, r.cvt);
}

// The scaling of a partial of weight row n and token t before it is written or summed: once by the row scale for e4m3
// weights, then by the token scale for e4m3 activations (a_scale is the quantizer's output: a plain load, after
// pdl_wait); the other formats' partials are the accumulators
template <int FMT>
__device__ __forceinline__ float scale_partial(float v, float scale_n, const float* a_scale, int t) {
  if constexpr (FMT == FMT_E4M3) return __fmul_rn(v, scale_n);
  if constexpr (FMT == FMT_E4M3_A8) return __fmul_rn(__fmul_rn(v, scale_n), a_scale[t]);
  return v;
}
// the row scale of feature n (e4m3 weights; 0 for the others and for rows past rows_w)
template <int FMT>
__device__ __forceinline__ float ws_row_scale(const float* w_scale, int n, bool n_ok) {
  float scale_n = 0.f;
  if constexpr (FMT == FMT_E4M3 || FMT == FMT_E4M3_A8) {
    if (n_ok) scale_n = __ldg(w_scale + n);
  }
  return scale_n;
}

// The body of both kernels.  TILES = false: the runtime mode of p (the instances the layers run); TILES = true: whole
// tiles of e4m3 or int4 weights with the bf16 store (ws_tiles_own_instances, gemm.cuh).
template <int FMT, int BN, int STAGES, bool TILES>
__device__ __forceinline__ void gemm_ws_body(const CUtensorMap& tm_w, const CUtensorMap& tm_x, const GemmWsArgs& p) {
  static_assert(!TILES || ws_tiles_own_instances(FMT), "whole-tile instances of their own: e4m3 and int4 weights");
  using Cfg = GemmWsCfg<FMT, BN, STAGES>;
  constexpr int S = Cfg::kStages;
  const WsRing r = ws_ring<Cfg>();
  float* stage = r.tail;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x;
  const int kb = p.sk.kb;
  long long u0, u1;
  if (!TILES && p.mode == 0) {
    u0 = sk_lo(c, p.sk);
    u1 = sk_lo(c + 1, p.sk);
  } else {
    u0 = ((static_cast<long long>(c) * p.tiles) / p.sk.G) * kb;
    u1 = ((static_cast<long long>(c + 1) * p.tiles) / p.sk.G) * kb;
  }
  const bool producer = warp == kGemmProducerWarp && lane == 0;
  const int pre = ws_prologue<FMT, BN, S>(tm_w, tm_x, r, p, u0, u1, kb, p.x_tiles, warp, producer);

  if (warp == kGemmProducerWarp) {
    if (lane == 0) ws_produce<FMT, BN, S>(tm_w, tm_x, r, p, u0, u1, kb, p.x_tiles, pre);
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
      ws_mainloop<FMT, BN, S>(acc, r, p, i, tile, k0, nk);
      const int wt = tile / p.x_tiles, xt = tile - wt * p.x_tiles;
      const int n = wt * kGemmBM + row;  // output feature (row of W)
      const int t0 = xt * BN;            // first token row of this tile
      const bool n_ok = n < p.rows_w;
      float* plane = nullptr;
      float bias_n = 0.f;
      const float scale_n = ws_row_scale<FMT>(p.wt.w_scale, n, n_ok);
      if (!TILES && p.mode == 0) {
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
          if (TILES) {   // bf16(acc) for int4, bf16(fl(acc * s[n])) for e4m3
            reinterpret_cast<uint16_t*>(p.out)[static_cast<size_t>(t) * p.ld_out + n] =
                to16<FMT_BF16>(scale_partial<FMT>(v[j], scale_n, nullptr, t));
          } else if (FMT == FMT_E4M3 || FMT == FMT_E4M3_A8 || p.mode == 0) {   // e4m3 formats run mode 0 only here
            plane[static_cast<size_t>(t) * p.rows_w + n] = scale_partial<FMT>(v[j], scale_n, p.wt.a_scale, t);
          } else {
            float x = r16<FMT>(v[j] + bias_n);
            x = apply_act<FMT>(x, p.act);
            reinterpret_cast<uint16_t*>(p.out)[static_cast<size_t>(t) * p.ld_out + n] = to16<FMT>(x);
          }
        }
      }
    }
  }
}

template <int FMT, int BN, int STAGES = ws_default_stages(FMT, BN)>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_ws_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
               const GemmWsArgs p) {
  gemm_ws_body<FMT, BN, STAGES, false>(tm_w, tm_x, p);
}

// whole tiles of e4m3 or int4 weights (p.mode is ignored)
template <int FMT, int BN, int STAGES = ws_default_stages(FMT, BN)>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_ws_tiles_kernel(const __grid_constant__ CUtensorMap tm_w, const __grid_constant__ CUtensorMap tm_x,
                     const GemmWsArgs p) {
  gemm_ws_body<FMT, BN, STAGES, true>(tm_w, tm_x, p);
}

}  // namespace vlo
