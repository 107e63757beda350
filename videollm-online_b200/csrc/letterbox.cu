// letterbox_kernel: native camera frames (packed RGB / BGR, each of its own size) -> the uint8 [B, 3, R, R] RGB canvases
// vlo_vit_encode reads, by the integer INTER_CUBIC arithmetic include/vlo_b200.h defines for vlo_letterbox.
//
// One thread per canvas pixel, all three channels.  INTER_CUBIC has no antialiasing: an output pixel reads a 4 x 4
// window, and at the downscales of camera frames (x1.67 for 640 x 480, x5 for 1920 x 1080) the windows of neighbouring
// output lines share few source lines, so the horizontal sums are formed in registers rather than staged in shared
// memory.  Integer sums are exact in any order: the bits do not depend on how the work is split.
#include <algorithm>
#include <cmath>

#include "common.h"
#include "ptx.cuh"
#include "vlo_b200.h"

namespace vlo {
namespace {

constexpr int kLetterboxThreads = 256;
constexpr int kLetterboxMaxSide = 8192;

struct LetterboxGeom {
  int sw, sh, x0, y0;
};

// passed by value (kernel parameter space): no staging copy, no device table
struct LetterboxBatch {
  vlo_letterbox_frame f[kLetterboxMaxFrames];
  LetterboxGeom g[kLetterboxMaxFrames];
  uint8_t* out;
  int R;
};
static_assert(sizeof(LetterboxBatch) <= 4000, "the kernel parameters of one launch must fit in 4 KB");

// video_ingest.letterbox_geometry: Python's round() of a correctly rounded double quotient is nearbyint() here
LetterboxGeom letterbox_geometry(int w, int h, int R) {
  LetterboxGeom g{};
  if (w > h) {
    g.sw = R;
    g.sh = static_cast<int>(std::nearbyint(static_cast<double>(h) * R / w / 2.0)) * 2;
  } else {
    g.sh = R;
    g.sw = static_cast<int>(std::nearbyint(static_cast<double>(w) * R / h / 2.0)) * 2;
  }
  g.sw = std::max(2, std::min(g.sw, R));
  g.sh = std::max(2, std::min(g.sh, R));
  g.x0 = (R - g.sw) / 2;
  g.y0 = (R - g.sh) / 2;
  return g;
}

__global__ void __launch_bounds__(kLetterboxThreads) letterbox_kernel(const __grid_constant__ LetterboxBatch p) {
  pdl_trigger();
  const int b = blockIdx.y, R = p.R;
  const vlo_letterbox_frame& f = p.f[b];
  const LetterboxGeom& g = p.g[b];
  const int pix = blockIdx.x * kLetterboxThreads + threadIdx.x;
  const int y = pix / R, x = pix - y * R;
  const int dx = x - g.x0, dy = y - g.y0;
  const bool inside = dx >= 0 && dx < g.sw && dy >= 0 && dy < g.sh;
  // the canvas may still be read by the previous pass's patchify_kernel: nothing is read or written before the wait
  pdl_wait();
  if (pix >= R * R) return;
  int out[3] = {0, 0, 0};
  if (inside) {
    const int4* tx = reinterpret_cast<const int4*>(f.d_taps) + 2 * (static_cast<long long>(f.x_taps) + dx);
    const int4* ty = reinterpret_cast<const int4*>(f.d_taps) + 2 * (static_cast<long long>(f.y_taps) + dy);
    const int4 xi = __ldg(tx), xw = __ldg(tx + 1), yi = __ldg(ty), yw = __ldg(ty + 1);
    const int cx[4] = {xi.x, xi.y, xi.z, xi.w}, wx[4] = {xw.x, xw.y, xw.z, xw.w};
    const int cy[4] = {yi.x, yi.y, yi.z, yi.w}, wy[4] = {yw.x, yw.y, yw.z, yw.w};
    int col[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) col[j] = 3 * min(max(cx[j], 0), f.width - 1);   // a bad table cannot read outside the image
    int v[3] = {0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint8_t* row = f.d_pixels + static_cast<size_t>(min(max(cy[k], 0), f.height - 1)) * f.width * 3;
      int h[3] = {0, 0, 0};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int c = 0; c < 3; ++c) h[c] += static_cast<int>(__ldg(row + col[j] + c)) * wx[j];
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) v[c] += h[c] * wy[k];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = min(max((v[c] + (1 << 21)) >> 22, 0), 255);
  }
  uint8_t* dst = p.out + static_cast<size_t>(b) * 3 * R * R + pix;
  const size_t plane = static_cast<size_t>(R) * R;
  dst[0] = static_cast<uint8_t>(out[f.bgr ? 2 : 0]);
  dst[plane] = static_cast<uint8_t>(out[1]);
  dst[2 * plane] = static_cast<uint8_t>(out[f.bgr ? 0 : 2]);
}

}  // namespace

int letterbox_launch(const vlo_letterbox_frame* frames, int n, int R, uint8_t* out, cudaStream_t st) {
  VLO_CHECK(frames != nullptr && out != nullptr, "letterbox: null frames or output");
  VLO_CHECK(R > 0, "letterbox: image_size must be positive");
  for (int i = 0; i < n; ++i) {
    const vlo_letterbox_frame& f = frames[i];
    const std::string at = "letterbox: frame " + std::to_string(i) + ": ";
    VLO_CHECK(f.d_pixels != nullptr && f.d_taps != nullptr, at + "null pixels or taps");
    VLO_CHECK(f.width >= 1 && f.width <= kLetterboxMaxSide && f.height >= 1 && f.height <= kLetterboxMaxSide,
              at + "width and height must lie in [1, 8192]");
    VLO_CHECK(f.bgr == 0 || f.bgr == 1, at + "bgr must be 0 or 1");
    VLO_CHECK(reinterpret_cast<uintptr_t>(f.d_taps) % 16 == 0, at + "the tap tables must be 16-byte aligned");
    VLO_CHECK(f.x_taps >= 0 && f.y_taps >= 0, at + "tap table offsets must be >= 0");
  }
  for (int b0 = 0; b0 < n; b0 += kLetterboxMaxFrames) {
    const int nb = std::min(kLetterboxMaxFrames, n - b0);
    LetterboxBatch p{};
    for (int i = 0; i < nb; ++i) {
      p.f[i] = frames[b0 + i];
      p.g[i] = letterbox_geometry(p.f[i].width, p.f[i].height, R);
    }
    p.out = out + static_cast<size_t>(b0) * 3 * R * R;
    p.R = R;
    const dim3 grid((R * R + kLetterboxThreads - 1) / kLetterboxThreads, nb);
    VLO_CUDA(launch_pdl(letterbox_kernel, grid, dim3(kLetterboxThreads), 0, st, p));
    count_launch();
  }
  return 0;
}

}  // namespace vlo
