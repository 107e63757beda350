// Stream-K decomposition shared by the weight-streaming GEMM (producer of fp32 partial planes) and the
// fix-up kernels that consume them.  Units = (128-row weight tile, 64-wide k-block); CTA c of G owns the
// contiguous unit range [floor(c*U/G), floor((c+1)*U/G)).  A tile's partials live in planes
// 0..sk_planes(tile)-1, plane index = contributing CTA - first contributing CTA.
#pragma once
#include <cuda_runtime.h>

namespace vlo {

// The fix-up kernels unroll their plane loads to this many planes; the engine rejects plans that need more.
constexpr int kFixMaxPlanes = 8;

struct SkInfo {
  long long U;  // total units = tiles * kb
  int kb;       // k-blocks per tile
  int G;        // CTAs in the grid
};

__host__ __device__ inline long long sk_lo(int c, const SkInfo& s) { return (static_cast<long long>(c) * s.U) / s.G; }
// the CTA whose unit range contains `unit`
__host__ __device__ inline int sk_owner(long long unit, const SkInfo& s) {
  int c = static_cast<int>((unit * s.G) / s.U);
  if (c >= s.G) c = s.G - 1;
  while (sk_lo(c + 1, s) <= unit) ++c;
  while (c > 0 && sk_lo(c, s) > unit) --c;
  return c;
}
__host__ __device__ inline int sk_first_cta(int tile, const SkInfo& s) {
  return sk_owner(static_cast<long long>(tile) * s.kb, s);
}
__host__ __device__ inline int sk_planes(int tile, const SkInfo& s) {
  return sk_owner(static_cast<long long>(tile + 1) * s.kb - 1, s) - sk_first_cta(tile, s) + 1;
}

}  // namespace vlo
