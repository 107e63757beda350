// letterbox_kernel: native camera frames (packed RGB / BGR, NV12, I420 or YUYV, each of its own size) -> the uint8
// [B, 3, R, R] RGB canvases vlo_vit_encode reads, by the integer INTER_CUBIC arithmetic include/vlo_b200.h defines for
// vlo_letterbox, with vlo_letterbox_planes' YUV -> RGB conversion of every tap.
//
// One thread per canvas pixel, all three channels.  INTER_CUBIC has no antialiasing: an output pixel reads a 4 x 4
// window, and at the downscales of camera frames (x1.67 for 640 x 480, x5 for 1920 x 1080) the windows of neighbouring
// output lines share few source lines, so the horizontal sums are formed in registers rather than staged in shared
// memory.  Integer sums are exact in any order: the bits do not depend on how the work is split.
//
// The source-pixel fetch is a template parameter (SrcPacked, SrcNv12, SrcI420, SrcYuyv); the tap sums, the bars and the
// canvas writes are shared.  A frame's format is uniform over its blocks (grid y = frame), so one launch takes frames of
// every format and the branch on it does not diverge.  The YUV conversion clamps each tap to [0, 255] before the cubic
// sums, as cvtColor does before a resize, so it cannot be folded in after the horizontal pass.
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

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

// passed by value (kernel parameter space): no staging copy, no device table.  80 B per frame, so 48 frames fit the
// 4 KB parameter space every CUDA 12 driver takes (the 32 KB space of CUDA >= 12.1 drivers is not relied on).
struct LetterboxBatch {
  vlo_frame_planes f[kLetterboxMaxFrames];
  LetterboxGeom g[kLetterboxMaxFrames];
  uint8_t* out;
  int R;
};
static_assert(sizeof(vlo_frame_planes) == 64, "vlo_frame_planes layout (include/vlo_b200.h, _lib.VloFramePlanes)");
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

// OpenCV's fixed-point BT.601 limited-range YUV -> RGB (cvtColor COLOR_YUV2RGB_NV12 / _I420 / _YUYV); every sum fits int32
__device__ __forceinline__ void yuv_to_rgb(int Y, int U, int V, int (&c)[3]) {
  const int y = max(Y - 16, 0) * 1220542 + (1 << 19), u = U - 128, v = V - 128;
  c[0] = min(max((y + 1673527 * v) >> 20, 0), 255);
  c[1] = min(max((y - 852492 * v - 409993 * u) >> 20, 0), 255);
  c[2] = min(max((y + 2116026 * u) >> 20, 0), 255);
}

// Source rows: built once per tap row y (clamped to the frame), then rgb(x) of a column x clamped to the frame.  The
// chroma of (x, y) is sample (x/2, y/2) or pair x/2: with even sides it lies inside the plane's row bytes.
struct SrcPacked {   // RGB or BGR in source order; the canvas write swaps BGR
  const uint8_t* p;
  __device__ SrcPacked(const vlo_frame_planes& f, int y) : p(f.d_planes[0] + static_cast<size_t>(y) * f.pitch[0]) {}
  __device__ void rgb(int x, int (&c)[3]) const {
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = __ldg(p + 3 * x + k);
  }
};
struct SrcNv12 {
  const uint8_t *py, *puv;
  __device__ SrcNv12(const vlo_frame_planes& f, int y)
      : py(f.d_planes[0] + static_cast<size_t>(y) * f.pitch[0]), puv(f.d_planes[1] + static_cast<size_t>(y >> 1) * f.pitch[1]) {}
  __device__ void rgb(int x, int (&c)[3]) const {
    const uint8_t* uv = puv + (x & ~1);
    yuv_to_rgb(__ldg(py + x), __ldg(uv), __ldg(uv + 1), c);
  }
};
struct SrcI420 {
  const uint8_t *py, *pu, *pv;
  __device__ SrcI420(const vlo_frame_planes& f, int y)
      : py(f.d_planes[0] + static_cast<size_t>(y) * f.pitch[0]), pu(f.d_planes[1] + static_cast<size_t>(y >> 1) * f.pitch[1]),
        pv(f.d_planes[2] + static_cast<size_t>(y >> 1) * f.pitch[2]) {}
  __device__ void rgb(int x, int (&c)[3]) const { yuv_to_rgb(__ldg(py + x), __ldg(pu + (x >> 1)), __ldg(pv + (x >> 1)), c); }
};
struct SrcYuyv {
  const uint8_t* p;
  __device__ SrcYuyv(const vlo_frame_planes& f, int y) : p(f.d_planes[0] + static_cast<size_t>(y) * f.pitch[0]) {}
  __device__ void rgb(int x, int (&c)[3]) const {
    const uint8_t* pair = p + 2 * (x & ~1);
    yuv_to_rgb(__ldg(pair + 2 * (x & 1)), __ldg(pair + 1), __ldg(pair + 3), c);
  }
};

// the scaled pixel (dx, dy) of frame f, channels in source order (packed) or RGB (YUV)
template <class Src>
__device__ __forceinline__ void cubic_pixel(const vlo_frame_planes& f, int dx, int dy, int (&out)[3]) {
  const int4* tx = reinterpret_cast<const int4*>(f.d_taps) + 2 * (static_cast<long long>(f.x_taps) + dx);
  const int4* ty = reinterpret_cast<const int4*>(f.d_taps) + 2 * (static_cast<long long>(f.y_taps) + dy);
  const int4 xi = __ldg(tx), xw = __ldg(tx + 1), yi = __ldg(ty), yw = __ldg(ty + 1);
  const int cx[4] = {xi.x, xi.y, xi.z, xi.w}, wx[4] = {xw.x, xw.y, xw.z, xw.w};
  const int cy[4] = {yi.x, yi.y, yi.z, yi.w}, wy[4] = {yw.x, yw.y, yw.z, yw.w};
  int col[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) col[j] = min(max(cx[j], 0), f.width - 1);   // a bad table cannot read outside the image
  int v[3] = {0, 0, 0};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const Src row(f, min(max(cy[k], 0), f.height - 1));
    int h[3] = {0, 0, 0};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int s[3];
      row.rgb(col[j], s);
#pragma unroll
      for (int c = 0; c < 3; ++c) h[c] += s[c] * wx[j];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] += h[c] * wy[k];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = min(max((v[c] + (1 << 21)) >> 22, 0), 255);
}

__global__ void __launch_bounds__(kLetterboxThreads) letterbox_kernel(const __grid_constant__ LetterboxBatch p) {
  pdl_trigger();
  const int b = blockIdx.y, R = p.R;
  const vlo_frame_planes& f = p.f[b];
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
    switch (f.format) {
      case VLO_PIX_NV12: cubic_pixel<SrcNv12>(f, dx, dy, out); break;
      case VLO_PIX_I420: cubic_pixel<SrcI420>(f, dx, dy, out); break;
      case VLO_PIX_YUYV: cubic_pixel<SrcYuyv>(f, dx, dy, out); break;
      default: cubic_pixel<SrcPacked>(f, dx, dy, out); break;
    }
  }
  const bool bgr = f.format == VLO_PIX_BGR24;
  uint8_t* dst = p.out + static_cast<size_t>(b) * 3 * R * R + pix;
  const size_t plane = static_cast<size_t>(R) * R;
  dst[0] = static_cast<uint8_t>(out[bgr ? 2 : 0]);
  dst[plane] = static_cast<uint8_t>(out[1]);
  dst[2 * plane] = static_cast<uint8_t>(out[bgr ? 0 : 2]);
}

// planes a format reads, and the row bytes of each (0: not read)
int format_planes(int format, int w, long long (&row)[3]) {
  row[0] = row[1] = row[2] = 0;
  switch (format) {
    case VLO_PIX_RGB24: case VLO_PIX_BGR24: row[0] = 3LL * w; return 1;
    case VLO_PIX_NV12: row[0] = w; row[1] = w; return 2;
    case VLO_PIX_I420: row[0] = w; row[1] = row[2] = w / 2; return 3;
    case VLO_PIX_YUYV: row[0] = 2LL * w; return 1;
    default: return 0;
  }
}

}  // namespace

int letterbox_planes_launch(const vlo_frame_planes* frames, int n, int R, uint8_t* out, cudaStream_t st) {
  VLO_CHECK(frames != nullptr && out != nullptr, "letterbox: null frames or output");
  VLO_CHECK(R > 0, "letterbox: image_size must be positive");
  for (int i = 0; i < n; ++i) {
    const vlo_frame_planes& f = frames[i];
    const std::string at = "letterbox: frame " + std::to_string(i) + ": ";
    long long row[3];
    const int np = format_planes(f.format, f.width, row);
    VLO_CHECK(np > 0, at + "unknown pixel format " + std::to_string(f.format));
    const bool yuv = f.format != VLO_PIX_RGB24 && f.format != VLO_PIX_BGR24;
    const int lo = yuv ? 2 : 1;
    VLO_CHECK(f.width >= lo && f.width <= kLetterboxMaxSide && f.height >= lo && f.height <= kLetterboxMaxSide,
              at + "width and height must lie in [" + std::to_string(lo) + ", 8192]");
    VLO_CHECK(!yuv || f.width % 2 == 0, at + "a YUV frame's width must be even");
    VLO_CHECK(!(f.format == VLO_PIX_NV12 || f.format == VLO_PIX_I420) || f.height % 2 == 0,
              at + "a 4:2:0 frame's height must be even");
    for (int q = 0; q < np; ++q) {
      VLO_CHECK(f.d_planes[q] != nullptr, at + "null plane " + std::to_string(q));
      VLO_CHECK(f.pitch[q] >= row[q], at + "plane " + std::to_string(q) + ": pitch " + std::to_string(f.pitch[q]) +
                                          " is below its " + std::to_string(row[q]) + " row bytes");
    }
    VLO_CHECK(f.d_taps != nullptr, at + "null taps");
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

int letterbox_launch(const vlo_letterbox_frame* frames, int n, int R, uint8_t* out, cudaStream_t st) {
  VLO_CHECK(frames != nullptr && out != nullptr, "letterbox: null frames or output");
  std::vector<vlo_frame_planes> planes(std::max(n, 0));
  for (int i = 0; i < n; ++i) {
    const vlo_letterbox_frame& f = frames[i];
    const std::string at = "letterbox: frame " + std::to_string(i) + ": ";
    VLO_CHECK(f.d_pixels != nullptr && f.d_taps != nullptr, at + "null pixels or taps");
    VLO_CHECK(f.width >= 1 && f.width <= kLetterboxMaxSide && f.height >= 1 && f.height <= kLetterboxMaxSide,
              at + "width and height must lie in [1, 8192]");
    VLO_CHECK(f.bgr == 0 || f.bgr == 1, at + "bgr must be 0 or 1");
    vlo_frame_planes& q = planes[i];
    q = vlo_frame_planes{};
    q.d_planes[0] = f.d_pixels;
    q.pitch[0] = 3 * f.width;
    q.d_taps = f.d_taps;
    q.format = f.bgr ? VLO_PIX_BGR24 : VLO_PIX_RGB24;
    q.width = f.width;
    q.height = f.height;
    q.x_taps = f.x_taps;
    q.y_taps = f.y_taps;
  }
  return letterbox_planes_launch(planes.data(), n, R, out, st);
}

}  // namespace vlo
