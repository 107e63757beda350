// wgmma / TMA GEMM for sm_90a:   C[i, j] = sum_k A[i, k] * B[j, k]
//
// Both operands are K-major ("TN"): A = activations [rows_a, K], B = weights [rows_b, K], fp16, fp32
// accumulation in registers.  One CTA computes one 128 x BN tile of out[rows_a, rows_b]:
//   warps 0-3  one warpgroup: wgmma.mma_async m64nBNk16 on both 64-row halves of the
//              tile, then the epilogue (accumulators -> shared staging tile -> global)
//   warp 4     TMA producer   (cp.async.bulk.tensor, 128B-swizzled boxes)
// connected by an mbarrier full/empty ring.  It runs the ViT patch embed (EPI_PATCH32) and the MAP-head K/V
// projection (EPI_STORE16).  The persistent kernels (gemm_ws.cuh, gemm_wsf.cuh, gemm_vit.cuh) build on the tile
// constants and helpers defined here.
//
// Replaces, for the hot path, the cuBLAS/cuDNN GEMMs reached from
//   HF:models/llama/modeling_llama.py:262-264,288,182-184,487  (q/k/v/o, MLP, lm_head)
//   HF:models/siglip/modeling_siglip.py:175-179,285-287,309,323-327 (patch embed, attn, MLP)
//   models/live_llama/modeling_live_llama.py:18-22 (connector)
#pragma once
#include <cuda.h>
#include <cuda_fp8.h>
#include "ptx.cuh"
#include "wgmma.cuh"

namespace vlo {

enum GemmEpi : int {
  EPI_STORE16 = 1,  // out16 = r16(act(r16(acc + bias)))
  EPI_PATCH32 = 3,  // out32  = r16(acc + bias) + pos[out_row % pos_rows]     (ViT patch embed)
};
enum GemmAct : int { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_GELU_ERF_PY = 2 };
// FMT_E4M3: e4m3 weights with one fp32 scale per weight row, bf16 activations; the consumer upcasts each weight k-block
// to bf16 exactly and runs the bf16 wgmma chain (weight-streaming kernels: stream-K partials, and whole tiles in
// instances of their own)
// FMT_E4M3_A8: e4m3 weights (row scales) x e4m3 activations (token scales), multiplied by the FP8 wgmma (QGMMA) on
// SWIZZLE_64B stages; each partial is scaled once in the epilogue (weight-streaming kernels, stream-K partials only)
// FMT_I4: 4-bit weight codes with one bf16 scale per 128 k of a row, bf16 activations; the consumer dequantizes the
// codes into the wgmma A fragment in registers and runs the bf16 wgmma chain (weight-streaming kernels: stream-K
// partials, and whole tiles in instances of their own)
enum GemmFmt : int { FMT_F16 = 0, FMT_BF16 = 1, FMT_E4M3 = 2, FMT_E4M3_A8 = 3, FMT_I4 = 4 };
// epilogues of the prefill GEMM (gemm_prefill.cuh): one fp32 plane for the fix-up kernels, or gate|up + SwiGLU
enum PrefillEpi : int { PREFILL_PLANE = 0, PREFILL_SWIGLU = 1 };

struct GemmArgs {
  int rows_a, rows_b, k;
  void* out;
  int ld_out;  // row stride of the output, elements
  const float* bias;  // per output column (feature) or nullptr
  const float* pos;   // EPI_PATCH32: [pos_rows, ld_out] fp32
  int pos_rows;
  int act;
};

constexpr int kGemmBM = 128;
constexpr int kGemmBK = 64;  // one 128-byte swizzle atom of 16-bit elements
constexpr int kGemmThreads = 160;  // warps 0-3: MMA + epilogue warpgroup; warp 4: TMA producer
constexpr int kGemmProducerWarp = 4;
constexpr int kSmemOptIn = 232448;  // 227 KB: the per-block dynamic shared memory limit of sm_90

// fp32 staging tile the accumulators pass through on their way to the epilogue, 16 columns at a time: [128][16 + 4].
// 10 KB whatever the tile width, so the small-tile ViT configuration still fits on an SM beside a decoder CTA (gemm.cu).
constexpr int kWgChunk = 16;
constexpr int kWgStageLd = kWgChunk + 4;
constexpr int kWgStageBytes = kGemmBM * kWgStageLd * 4;
// deepest ring (<= cap stages of `per_stage` bytes) that fits next to `fixed` bytes in one block
constexpr int fit_stages(int per_stage, int fixed, int cap) {
  return (kSmemOptIn - fixed) / per_stage < cap ? (kSmemOptIn - fixed) / per_stage : cap;
}

template <int BN>
struct GemmCfg {
  static constexpr int kBytesA = kGemmBM * kGemmBK * 2;
  static constexpr int kBytesB = BN * kGemmBK * 2;
  // 1024 B of slack so the tile ring can be aligned for SWIZZLE_128B, 256 B of barriers, 1 KB bias tile
  static constexpr int kFixed = kWgStageBytes + 1024 + 256 + 1024;
  static constexpr int kStages = fit_stages(kBytesA + kBytesB, kFixed, BN <= 64 ? 8 : 6);
  static constexpr int kSmemBytes = kStages * (kBytesA + kBytesB) + kFixed;
};

__device__ __forceinline__ void wg_sync() { asm volatile("bar.sync 1, 128;\n" ::: "memory"); }  // the MMA warpgroup

// ---- the weight formats of the weight-streaming kernels (gemm_ws.cuh, gemm_wsf.cuh)
// FMT_E4M3: a weight stage is a 128 x 64-byte TMA box without swizzle.  Every finite e4m3 value is a bf16 value, so the
// upcast is exact; the MMAs then read a bf16 tile laid out as a SWIZZLE_128B TMA box would leave it and issue the same
// wgmma chain as FMT_BF16, so the fp32 accumulators are those of the bf16 kernel on the upcast weights.
// FMT_E4M3_A8: a weight stage is a 128 x 64-byte TMA box and an activation stage a BN x 64-byte box, both with the 64-byte
// swizzle the FP8 wgmma descriptor reads directly: no conversion, no generic-proxy stores, no warpgroup barrier.
// FMT_I4: W4[n, k] = bf16_rn(q * s), q = code - 8 in [-8, 7], s = gscale[n, k / 128] (bf16).  Engine byte order of the
// codes: one 4 KB block per (128-row tile, 64-wide k-block) unit, the units of a tile in k order and the tiles in row
// order, so the unit range of a stream-K CTA is one contiguous byte range.  Inside a unit, thread t of the warpgroup owns
// 16 bytes per 64-row half h at byte h * 2048 + t * 16: the four 32-bit words of its m64k16 A fragments for the k16 steps
// kk = 0..3.  The word of step kk holds, for row r = 64h + 16(t/32) + (t%32)/4 and column c = 16kk + 2(t%4), the code of
// element (r + 8e, c + 8f + b) in bits 4(e + 2f) + 16b .. +3, so (word >> 4p) & 0x000F000F is the pair of fragment
// register p.
constexpr int kF8BytesCvt = 2 * kGemmBM * kGemmBK * 2;  // two bf16 tiles: k-block j converts while the MMAs of j - 1 run
constexpr int kI4BytesUnit = kGemmBM * kGemmBK / 2;     // 4 KB of codes per unit
constexpr int kI4Group = 128;                           // k per scale
// An int4 ring slot carries up to this many consecutive k-blocks of one tile (8-16 KB of codes), split at multiples of
// it, so a slot never spans more than units / 2 scale groups.
constexpr int i4_slot_units(int bn) { return bn <= 32 ? 4 : 2; }

// k-blocks per ring slot, the weight and activation bytes of one slot, the conversion tiles and the deepest ring of a
// format at token-tile width bn.  16-bit weights stop at 8 stages; the others have smaller stages and go up to the 16
// full / empty barrier pairs of the barrier block.
constexpr int ws_slot_units(int fmt, int bn) { return fmt == FMT_I4 ? i4_slot_units(bn) : 1; }
constexpr int ws_slot_bytes_w(int fmt, int bn) {
  return fmt == FMT_I4 ? i4_slot_units(bn) * kI4BytesUnit : kGemmBM * kGemmBK * (fmt == FMT_E4M3 || fmt == FMT_E4M3_A8 ? 1 : 2);
}
constexpr int ws_slot_bytes_x(int fmt, int bn) { return ws_slot_units(fmt, bn) * bn * kGemmBK * (fmt == FMT_E4M3_A8 ? 1 : 2); }
constexpr int ws_cvt_bytes(int fmt) { return fmt == FMT_E4M3 ? kF8BytesCvt : 0; }
constexpr int ws_max_stages(int fmt) { return fmt == FMT_F16 || fmt == FMT_BF16 ? 8 : 16; }
// shared memory besides the ring: conversion tiles, 1024 B of alignment slack, 256 B of barriers, the staging tile and
// `extra` bytes of the kernel's own (the fused kernel's exchange tile)
constexpr int ws_fixed_bytes(int fmt, int extra) { return ws_cvt_bytes(fmt) + 1024 + 256 + extra + kWgStageBytes; }
// the deepest ring that fits
constexpr int ws_default_stages(int fmt, int bn, int extra = 0) {
  return fit_stages(ws_slot_bytes_w(fmt, bn) + ws_slot_bytes_x(fmt, bn), ws_fixed_bytes(fmt, extra), ws_max_stages(fmt));
}

// Whole tiles (mode 1) with the 16-bit store: every format but FMT_E4M3_A8.  The 16-bit formats run it in the
// instances the layers run (a runtime mode); e4m3 and int4 weights run it in instances of their own
// (gemm_ws_tiles_kernel: the vocabulary matrices of engines whose layers take those forms), which store bf16(acc) for
// int4 and bf16(fl(acc * s[n])) for e4m3, with no bias and no activation.  One CTA covers all of K for each of its
// tiles, so a logits row depends on no other row and on no token tile.  int4: at most 128 token rows (one token tile).
constexpr bool ws_tiles_own_instances(int fmt) { return fmt == FMT_E4M3 || fmt == FMT_I4; }

template <int FMT, int BN, int STAGES, int EXTRA = 0>
struct GemmWsCfg {
  static constexpr int kStages = STAGES;
  static constexpr int kBytesA = ws_slot_bytes_w(FMT, BN);
  static constexpr int kBytesB = ws_slot_bytes_x(FMT, BN);
  static constexpr int kBytesCvt = ws_cvt_bytes(FMT);
  static constexpr int kSmemBytes = kStages * (kBytesA + kBytesB) + ws_fixed_bytes(FMT, EXTRA);
  static_assert(kSmemBytes <= kSmemOptIn, "ring + staging tiles exceed the shared memory of one block");
  static_assert(kStages <= 16, "the barrier block holds 16 full / empty pairs");
};

// What the host needs of a format: the get_tmap kind (a GemmFmt) of the weight and activation maps (-1: the int4 codes
// stream as bulk copies) and the HBM bytes of one weight, one activation, one weight row's scale, one token's scale and
// one 128-k group's scale.
struct WsFmtInfo {
  int w_map, x_map;
  double w_elem, x_elem;
  int row_scale, tok_scale, group_scale;
};
constexpr WsFmtInfo kWsFmtInfo[] = {
    {FMT_F16, FMT_F16, 2.0, 2.0, 0, 0, 0},              // FMT_F16
    {FMT_BF16, FMT_BF16, 2.0, 2.0, 0, 0, 0},            // FMT_BF16
    {FMT_E4M3, FMT_BF16, 1.0, 2.0, 4, 0, 0},            // FMT_E4M3
    {FMT_E4M3_A8, FMT_E4M3_A8, 1.0, 1.0, 4, 4, 0},      // FMT_E4M3_A8
    {-1, FMT_BF16, 0.5, 2.0, 0, 0, 2},                  // FMT_I4
};
// the weight and activation bytes a weight-streaming GEMM of W [rows_w, k] by X [rows_x, k] reads (profiler, benches)
inline double ws_in_bytes(int fmt, int rows_w, int rows_x, int k) {
  const WsFmtInfo& f = kWsFmtInfo[fmt];
  return (k * f.w_elem + f.row_scale + f.group_scale * (k / kI4Group)) * rows_w + (k * f.x_elem + f.tok_scale) * rows_x;
}

__device__ __forceinline__ uint32_t e4m3x2_to_bf16x2(uint32_t two) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(two & 0xFFFF), __NV_E4M3);
  const __nv_bfloat162 b = __float22bfloat162_rn(__half22float2(__half2(h)));   // e4m3 -> f16 -> f32 -> bf16: all exact
  return *reinterpret_cast<const uint32_t*>(&b);
}

// the warpgroup converts one e4m3 stage src [128][64 B] into the bf16 tile dst [128][128 B], 16-byte chunk c of row r at
// chunk c ^ (r % 8).  Thread t converts chunks j * 128 + t: a warp reads 256 and writes 512 contiguous bytes per j.
__device__ __forceinline__ void f8_tile_to_bf16_sw128(const uint8_t* src, uint8_t* dst) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int idx = j * 128 + static_cast<int>(threadIdx.x), r = idx >> 3, c = idx & 7;
    const uint2 v = *reinterpret_cast<const uint2*>(src + r * 64 + c * 8);
    const uint4 o = make_uint4(e4m3x2_to_bf16x2(v.x), e4m3x2_to_bf16x2(v.x >> 16), e4m3x2_to_bf16x2(v.y),
                               e4m3x2_to_bf16x2(v.y >> 16));
    *reinterpret_cast<uint4*>(dst + r * 128 + ((c ^ (r & 7)) << 4)) = o;
  }
}

template <int BN>
__device__ __forceinline__ void wg_zero(float (&acc)[2][BN / 2]) {
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[h][j] = 0.f;
}

// after the last k-block: retire every MMA and give the last stage (ring position i - 1) back to the producer
template <int BN, int S>
__device__ __forceinline__ void wg_drain(float (&acc)[2][BN / 2], uint64_t* empty_bar, int i, int nk) {
  wgmma_wait<0>();
  wgmma_fence_regs(acc[0]);
  wgmma_fence_regs(acc[1]);
  if (nk > 0) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty_bar[(i - 1) % S]);
  }
}

// The warpgroup's part of the ring protocol: accumulate the nk k-blocks at ring positions i, i+1, ... into acc
// (zeroed first; acc[h] is the 64-row half h of the 128 x BN tile).  A stage goes back to the producer (one arrival per
// warp, empty barriers count 4) once the MMAs reading it have retired; one k-block of MMAs stays in flight.
// FMT_E4M3 converts k-block j into the bf16 tile j % 2 of smem_cvt first, then multiplies exactly as FMT_BF16 does.  The
// barrier before a conversion makes every warp's MMAs of k-block j - 2 (the tile's last readers) retired: each warp has
// passed wgmma_wait<1> of iteration j - 1 by then.  FMT_E4M3_A8 issues two k32 FP8 MMAs per 64-wide k-block on each
// 64-row half, in k order.
template <int FMT, int BN, int S>
__device__ __forceinline__ void wg_mainloop(float (&acc)[2][BN / 2], const uint8_t* smem_a, const uint8_t* smem_b,
                                            uint64_t* full_bar, uint64_t* empty_bar, int& i, int nk,
                                            uint8_t* smem_cvt = nullptr) {
  constexpr int kBytesA = ws_slot_bytes_w(FMT, BN), kBytesB = ws_slot_bytes_x(FMT, BN);
  const int lane = threadIdx.x & 31;
  wg_zero<BN>(acc);
  for (int j = 0; j < nk; ++j, ++i) {
    const int s = i % S;
    uint8_t* cvt = smem_cvt + (j & 1) * (kF8BytesCvt / 2);   // FMT_E4M3
    mbar_wait(&full_bar[s], (i / S) & 1);
    if constexpr (FMT == FMT_E4M3) {
      if (j >= 2) wg_sync();
      f8_tile_to_bf16_sw128(smem_a + s * kBytesA, cvt);
      fence_proxy_async();   // the generic-proxy stores become visible to the wgmma operand reads
      wg_sync();
      wgmma_fence();
      const uint64_t da = wgmma_desc_sw128(smem_u32(cvt));
      const uint64_t db = wgmma_desc_sw128(smem_u32(smem_b + s * kBytesB));
#pragma unroll
      for (int kk = 0; kk < kGemmBK / 16; ++kk) {
        Wgmma<FMT_BF16, BN>::mma(acc[0], da + 2 * kk, db + 2 * kk);
        Wgmma<FMT_BF16, BN>::mma(acc[1], da + 512 + 2 * kk, db + 2 * kk);
      }
    } else if constexpr (FMT == FMT_E4M3_A8) {
      wgmma_fence();
      const uint64_t da = wgmma_desc_sw64(smem_u32(smem_a + s * kBytesA));
      const uint64_t db = wgmma_desc_sw64(smem_u32(smem_b + s * kBytesB));
#pragma unroll
      for (int kk = 0; kk < kGemmBK / 32; ++kk) {
        // +2 per 32 elements (32 B) along K; the second 64-row half of A starts 4 KB (+256) further
        WgmmaE4M3<BN>::mma(acc[0], da + 2 * kk, db + 2 * kk);
        WgmmaE4M3<BN>::mma(acc[1], da + 256 + 2 * kk, db + 2 * kk);
      }
    } else {
      wgmma_fence();
      const uint64_t da = wgmma_desc_sw128(smem_u32(smem_a + s * kBytesA));
      const uint64_t db = wgmma_desc_sw128(smem_u32(smem_b + s * kBytesB));
#pragma unroll
      for (int kk = 0; kk < kGemmBK / 16; ++kk) {
        // +2 per 16 elements (32 B) along K; the second 64-row half of A starts 8 KB (+512) further
        Wgmma<FMT, BN>::mma(acc[0], da + 2 * kk, db + 2 * kk);
        Wgmma<FMT, BN>::mma(acc[1], da + 512 + 2 * kk, db + 2 * kk);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (j > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % S]);
    }
  }
  wg_drain<BN, S>(acc, empty_bar, i, nk);
}

// ---- int4 weights (FMT_I4): the byte order of the codes is described above

// the slot that starts at unit u of the range [u, u1): its tile, first k-block and unit count
template <int KU>
__device__ __forceinline__ int i4_slot(long long u, long long u1, int kb, int& tile, int& kblk) {
  tile = static_cast<int>(u / kb);
  kblk = static_cast<int>(u - static_cast<long long>(tile) * kb);
  return static_cast<int>(min(static_cast<long long>(min(KU - kblk % KU, kb - kblk)), u1 - u));
}

// producer, before griddepcontrol.wait: the codes of the first S slots of [u0, u1) (they depend on no earlier kernel).
// Returns the number of slots issued.
template <int BN, int S, int KU>
__device__ __forceinline__ int i4_prefetch_codes(const uint8_t* w4, uint8_t* smem_a, uint64_t* full_bar, long long u0,
                                                 long long u1, int kb, uint64_t hint) {
  int pre = 0;
  for (long long u = u0; u < u1 && pre < S; ++pre) {
    int tile, kblk;
    const int n = i4_slot<KU>(u, u1, kb, tile, kblk);
    mbar_arrive_expect_tx(&full_bar[pre], n * (kI4BytesUnit + BN * kGemmBK * 2));
    bulk_load(smem_a + pre * KU * kI4BytesUnit, w4 + u * kI4BytesUnit, n * kI4BytesUnit, &full_bar[pre], hint);
    u += n;
  }
  return pre;
}

// producer: the whole slot stream of [u0, u1); slots below `pre` only still need their activation boxes
template <int BN, int S, int KU>
__device__ __forceinline__ void i4_produce(const uint8_t* w4, const CUtensorMap* tm_x, uint8_t* smem_a, uint8_t* smem_b,
                                           uint64_t* full_bar, uint64_t* empty_bar, long long u0, long long u1, int kb,
                                           int pre, uint64_t hint) {
  int i = 0;
  for (long long u = u0; u < u1; ++i) {
    int tile, kblk;
    const int n = i4_slot<KU>(u, u1, kb, tile, kblk);
    const int s = i % S;
    if (i >= pre) {
      mbar_wait(&empty_bar[s], ((i / S) & 1) ^ 1);
      mbar_arrive_expect_tx(&full_bar[s], n * (kI4BytesUnit + BN * kGemmBK * 2));
      bulk_load(smem_a + s * KU * kI4BytesUnit, w4 + u * kI4BytesUnit, n * kI4BytesUnit, &full_bar[s], hint);
    }
    for (int j = 0; j < n; ++j)
      tma_load_2d(smem_b + (s * KU + j) * BN * kGemmBK * 2, tm_x, &full_bar[s], (kblk + j) * kGemmBK, 0, kEvictLast);
    u += n;
  }
}

// consumer threads, before griddepcontrol.wait: pull the scale rows of their fragment rows over [u0, u1) into L2
__device__ __forceinline__ void i4_prefetch_scales(const uint16_t* gs, int ng, int rows_w, long long u0, long long u1, int kb) {
  if (u0 >= u1) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int t_lo = static_cast<int>(u0 / kb), t_hi = static_cast<int>((u1 - 1) / kb);
  for (int t = t_lo; t <= t_hi; ++t) {
    const int g0 = t == t_lo ? static_cast<int>(u0 - static_cast<long long>(t) * kb) / 2 : 0;
    const int g1 = t == t_hi ? static_cast<int>(u1 - 1 - static_cast<long long>(t) * kb) / 2 : ng - 1;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int n = t * kGemmBM + 64 * (r >> 1) + 16 * warp + (lane >> 2) + 8 * (r & 1);
      if (n >= rows_w) continue;
      const uint16_t* row = gs + static_cast<size_t>(n) * ng;
      for (int g = g0; g < g1; g += 64) prefetch_l2(row + g);   // one 128-B line per 64 scales
      prefetch_l2(row + g1);
    }
  }
}

__device__ __forceinline__ uint32_t bf16x2_bcast(uint16_t s) { return static_cast<uint32_t>(s) * 0x10001u; }

// four codes pairs of `word` -> the bf16x2 registers of one A fragment: (128 + code) by OR into the mantissa of 128,
// minus 136 = q exactly, times the row's scale = bf16_rn(q * s) (the product is exact in fp32; one rounding)
__device__ __forceinline__ void i4_fragment(uint32_t word, uint32_t s_lo, uint32_t s_hi, uint32_t (&a)[4]) {
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const uint32_t v = ((word >> (4 * p)) & 0x000F000Fu) | 0x43004300u;
    __nv_bfloat162 q = __hsub2(*reinterpret_cast<const __nv_bfloat162*>(&v), __floats2bfloat162_rn(136.f, 136.f));
    const uint32_t s = (p & 1) ? s_hi : s_lo;
    q = __hmul2(q, *reinterpret_cast<const __nv_bfloat162*>(&s));
    a[p] = *reinterpret_cast<const uint32_t*>(&q);
  }
}

// wg_mainloop for int4 weights over the nk k-blocks k0 .. of one tile, in the producer's slots (ring position i counts
// slots).  The codes go shared -> registers -> A fragments; each k-block issues the bf16 kernel's chain (kk = 0..3, half 0
// then half 1) with A from registers, so the fp32 accumulators are those of the bf16 kernel on W4.  The shared loads of
// a k-block's codes overlap the previous k-block's MMAs; its conversion waits for them.  A slot goes back to the producer
// once the MMAs of its last k-block retire (they read its activation boxes).
template <int BN, int S, int KU>
__device__ __forceinline__ void wg_mainloop_i4(float (&acc)[2][BN / 2], const uint8_t* smem_a, const uint8_t* smem_b,
                                               uint64_t* full_bar, uint64_t* empty_bar, int& i, int tile, int k0, int nk,
                                               const uint16_t* gs, int ng, int rows_w) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  wg_zero<BN>(acc);
  int rows[4];   // fragment rows: half h = r >> 1, +8 for r & 1
#pragma unroll
  for (int r = 0; r < 4; ++r) rows[r] = tile * kGemmBM + 64 * (r >> 1) + 16 * warp + (lane >> 2) + 8 * (r & 1);
  bool first = true;
  for (int kblk = k0; kblk < k0 + nk; ++i) {
    const int n = min(KU - kblk % KU, k0 + nk - kblk);
    const int s = i % S;
    // the scales of the (at most KU / 2) groups of the slot's KU-aligned window, loaded before the wait
    const int gw = (kblk - kblk % KU) / 2;
    uint32_t sc[KU / 2][4];
#pragma unroll
    for (int g = 0; g < KU / 2; ++g)
#pragma unroll
      for (int r = 0; r < 4; ++r)
        sc[g][r] = bf16x2_bcast(rows[r] < rows_w && gw + g < ng ? __ldg(gs + static_cast<size_t>(rows[r]) * ng + gw + g) : 0);
    mbar_wait(&full_bar[s], (i / S) & 1);
#pragma unroll
    for (int j = 0; j < KU; ++j) {
      if (j >= n) break;
      const int gsel = ((kblk + j) % KU) / 2;   // group of this k-block inside the window
      uint32_t s_r[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        s_r[r] = sc[0][r];
#pragma unroll
        for (int g = 1; g < KU / 2; ++g)
          if (gsel == g) s_r[r] = sc[g][r];
      }
      const uint8_t* unit = smem_a + (s * KU + j) * kI4BytesUnit + threadIdx.x * 16;
      const uint4 c0 = *reinterpret_cast<const uint4*>(unit);
      const uint4 c1 = *reinterpret_cast<const uint4*>(unit + kI4BytesUnit / 2);
      // no MMA in flight while the A registers are written: left to itself, ptxas serializes every wgmma of the loop
      // behind these writes (C7513), which measured 27 % slower than this one wait per k-block (DESIGN.md section 5)
      wgmma_wait<0>();
      uint32_t a[2][4][4];
      i4_fragment(c0.x, s_r[0], s_r[1], a[0][0]);
      i4_fragment(c0.y, s_r[0], s_r[1], a[0][1]);
      i4_fragment(c0.z, s_r[0], s_r[1], a[0][2]);
      i4_fragment(c0.w, s_r[0], s_r[1], a[0][3]);
      i4_fragment(c1.x, s_r[2], s_r[3], a[1][0]);
      i4_fragment(c1.y, s_r[2], s_r[3], a[1][1]);
      i4_fragment(c1.z, s_r[2], s_r[3], a[1][2]);
      i4_fragment(c1.w, s_r[2], s_r[3], a[1][3]);
      wgmma_fence();
      const uint64_t db = wgmma_desc_sw128(smem_u32(smem_b + (s * KU + j) * BN * kGemmBK * 2));
#pragma unroll
      for (int kk = 0; kk < kGemmBK / 16; ++kk) {
        WgmmaRegA<BN>::mma(acc[0], a[0][kk], db + 2 * kk);
        WgmmaRegA<BN>::mma(acc[1], a[1][kk], db + 2 * kk);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (j == 0 && !first) {   // every MMA of the previous slot has retired
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % S]);
      }
    }
    first = false;
    kblk += n;
  }
  wg_drain<BN, S>(acc, empty_bar, i, nk);
}

// columns c0 .. c0 + 15 of the accumulators -> staging tile (row r of the tile at stage[r * kWgStageLd]); c0 must be a
// compile-time constant after unrolling, so that acc stays in registers
template <int BN>
__device__ __forceinline__ void wg_stage_chunk(const float (&acc)[2][BN / 2], int c0, float* stage) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = 64 * h + 16 * warp + (lane >> 2);
#pragma unroll
    for (int c = 0; c < kWgChunk / 8; ++c) {
      const int g = c0 / 8 + c;  // 8-column group of the accumulator fragment
      const int col = 8 * c + 2 * (lane & 3);
      *reinterpret_cast<float2*>(stage + row * kWgStageLd + col) = make_float2(acc[h][4 * g], acc[h][4 * g + 1]);
      *reinterpret_cast<float2*>(stage + (row + 8) * kWgStageLd + col) = make_float2(acc[h][4 * g + 2], acc[h][4 * g + 3]);
    }
  }
}
// the staged 16 columns of tile row `row`
__device__ __forceinline__ void wg_load16(const float* stage, int row, float (&v)[16]) {
  const float4* p = reinterpret_cast<const float4*>(stage + row * kWgStageLd);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 t = p[j];
    v[4 * j] = t.x;
    v[4 * j + 1] = t.y;
    v[4 * j + 2] = t.z;
    v[4 * j + 3] = t.w;
  }
}

template <int FMT>
__device__ __forceinline__ float r16(float x) {
  return FMT == FMT_BF16 ? bf16_round(x) : fp16_round(x);
}
template <int FMT>
__device__ __forceinline__ uint16_t to16(float x) {
  if (FMT == FMT_BF16) return __bfloat16_as_ushort(__float2bfloat16_rn(x));
  return __half_as_ushort(__float2half_rn(x));
}

// LlamaMLP's act_fn(gate) * up on bf16 values g, u (HF:...llama.py:182-184): bf16(silu(g)) * u in fp32, which the caller
// rounds to bf16 once.  The gate|up finisher (gemm_wsf.cuh) and the prefill GEMM (gemm_prefill.cuh) share it.
__device__ __forceinline__ float swiglu_bf16(float g, float u) { return bf16_round(g / (1.0f + expf(-g))) * u; }

// MUFU.TANH (PTX ISA: maximum relative error 2^-10.987 over the entire range); vlo_op_tanh_approx exposes it to tests
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Activations evaluated the way the reference evaluates them on 16-bit tensors.
template <int FMT>
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ACT_GELU_TANH) {
    // F.gelu(x, approximate='tanh'), HF:activations.py ("gelu_pytorch_tanh"); fp32 math on
    // the 16-bit input, one rounding at the end.
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    const float inner = k0 * (v + k1 * v * v * v);
    const float th = tanh_approx(inner);  // |err| ~ 2^-11, below fp16 output resolution
    return r16<FMT>(0.5f * v * (1.0f + th));
  }
  if (act == ACT_GELU_ERF_PY) {
    // GELUActivation(use_gelu_python=True): x * 0.5 * (1 + erf(x / sqrt(2))) evaluated as four
    // separate 16-bit tensor ops (HF:activations.py:78-86 as instantiated at
    // models/live_llama/modeling_live_llama.py:20) -> one rounding per op.
    float t1 = r16<FMT>(v * 0.5f);
    float t2 = r16<FMT>(v / 1.4142135623730951f);
    float t3 = r16<FMT>(erff(t2));
    float t4 = r16<FMT>(1.0f + t3);
    return r16<FMT>(t1 * t4);
  }
  return v;
}

template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
               const GemmArgs p) {
  using Cfg = GemmCfg<BN>;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + S * Cfg::kBytesA;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S * (Cfg::kBytesA + Cfg::kBytesB));
  uint64_t* empty_bar = full_bar + S;
  float* s_bias = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(full_bar) + 256);
  float* stage = s_bias + 256;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_tile = blockIdx.x, n_tile = blockIdx.y;
  const int nkb = p.k / kGemmBK;

  if (warp == kGemmProducerWarp && lane == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  if (warp == kGemmProducerWarp) {
    if (lane == 0) {
      // ------------------------------------------------ TMA producer
      for (int i = 0; i < nkb; ++i) {
        const int s = i % S;
        const uint32_t ph = (i / S) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        mbar_arrive_expect_tx(&full_bar[s], Cfg::kBytesA + Cfg::kBytesB);
        const int kc = i * kGemmBK;
        tma_load_2d(smem_a + s * Cfg::kBytesA, &tm_a, &full_bar[s], kc, m_tile * kGemmBM, kEvictNormal);
        tma_load_2d(smem_b + s * Cfg::kBytesB, &tm_b, &full_bar[s], kc, n_tile * BN, kEvictNormal);
      }
    }
  } else {
    // -------------------------------------------------- MMA + epilogue warpgroup (warps 0-3)
    // per-column bias of this tile -> shared memory
    for (int j = threadIdx.x; j < BN; j += 128) {
      const int col = n_tile * BN + j;
      s_bias[j] = (p.bias != nullptr && col < p.rows_b) ? __ldg(p.bias + col) : 0.f;
    }
    float acc[2][BN / 2];
    int i = 0;
    wg_mainloop<FMT_F16, BN, S>(acc, smem_a, smem_b, full_bar, empty_bar, i, nkb);
    const int row = threadIdx.x;  // tile row this thread finishes
    const int a_row = m_tile * kGemmBM + row;
    const bool a_ok = a_row < p.rows_a;

#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += kWgChunk) {
      wg_sync();                      // the previous chunk's readers are done with the staging tile
      wg_stage_chunk<BN>(acc, c0, stage);
      wg_sync();
      const int b0 = n_tile * BN + c0;
      if (!a_ok || b0 >= p.rows_b) continue;
      float v[16];
      wg_load16(stage, row, v);
      // out[row = a, feature = b]; this thread owns 16 consecutive features of one row.
      const int nvalid = min(16, p.rows_b - b0);
      float x[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float acc = r16<FMT_F16>(v[j] + s_bias[c0 + j]);
        if (EPI == EPI_STORE16) acc = apply_act<FMT_F16>(acc, p.act);
        x[j] = acc;
      }
      const size_t idx = static_cast<size_t>(a_row) * p.ld_out + b0;
      const bool vec_ok = (nvalid == 16) && ((p.ld_out & 7) == 0);
      if (EPI == EPI_STORE16) {
        uint16_t* o = reinterpret_cast<uint16_t*>(p.out) + idx;
        if (vec_ok) {
          uint32_t w[8];
#pragma unroll
          for (int j = 0; j < 8; ++j)
            w[j] = static_cast<uint32_t>(to16<FMT_F16>(x[2 * j])) |
                   (static_cast<uint32_t>(to16<FMT_F16>(x[2 * j + 1])) << 16);
          reinterpret_cast<uint4*>(o)[0] = make_uint4(w[0], w[1], w[2], w[3]);
          reinterpret_cast<uint4*>(o)[1] = make_uint4(w[4], w[5], w[6], w[7]);
        } else {
          for (int j = 0; j < nvalid; ++j) o[j] = to16<FMT_F16>(x[j]);
        }
      } else {
        float* o = reinterpret_cast<float*>(p.out) + idx;
        const float* pe = p.pos + static_cast<size_t>(a_row % p.pos_rows) * p.ld_out + b0;
        if (vec_ok) {
#pragma unroll
          for (int j = 0; j < 16; j += 4) {
            const float4 pp = __ldg(reinterpret_cast<const float4*>(pe + j));
            reinterpret_cast<float4*>(o + j)[0] = make_float4(x[j] + pp.x, x[j + 1] + pp.y, x[j + 2] + pp.z, x[j + 3] + pp.w);
          }
        } else {
          for (int j = 0; j < nvalid; ++j) o[j] = x[j] + __ldg(pe + j);
        }
      }
    }
  }
}

}  // namespace vlo
