"""numpy restatements of vlo_letterbox_planes' YUV formats (include/vlo_b200.h): OpenCV's integer BT.601 limited-range
YUV -> RGB of one frame, and the kernel's fused path (each tap converted, then the two integer passes of
tests/letterbox_reference.py).  The CPU tests hold them to cv2.cvtColor and to letterbox_reference of cvtColor's RGB; the
GPU tests hold the kernel to them."""
import numpy as np

from videollm_online_b200.video_ingest import cubic_taps, letterbox_geometry, raw_frame_shape

FORMATS = ("nv12", "yuv420p", "yuyv422")


def cv2_code(pixel_format: str) -> int:
    import cv2
    return {"nv12": cv2.COLOR_YUV2RGB_NV12, "yuv420p": cv2.COLOR_YUV2RGB_I420,
            "yuyv422": cv2.COLOR_YUV2RGB_YUYV}[pixel_format]


def yuv_noise(width: int, height: int, pixel_format: str, seed: int) -> np.ndarray:
    """a uniformly random frame in the raw layout of video_ingest.raw_frame_shape"""
    shape = raw_frame_shape(width, height, pixel_format)
    return np.random.default_rng(seed).integers(0, 256, shape, dtype=np.uint8)


def planes(frame: np.ndarray, pixel_format: str):
    """(Y [H, W], U, V, chroma rows per luma row): U and V at chroma resolution ([H/2, W/2], or [H, W/2] for YUYV)"""
    if pixel_format == "yuyv422":
        return frame[:, :, 0], frame[:, 0::2, 1], frame[:, 1::2, 1], 1
    H, W = frame.shape[0] // 3 * 2, frame.shape[1]
    flat = frame.reshape(-1)
    Y = flat[:W * H].reshape(H, W)
    if pixel_format == "nv12":
        uv = flat[W * H:].reshape(H // 2, W // 2, 2)
        return Y, uv[..., 0], uv[..., 1], 2
    q = (W // 2) * (H // 2)
    return Y, flat[W * H:W * H + q].reshape(H // 2, W // 2), flat[W * H + q:].reshape(H // 2, W // 2), 2


def yuv_to_rgb(Y, U, V) -> np.ndarray:
    """the integer formula of vlo_letterbox_planes, elementwise: uint8 [..., 3] RGB"""
    y = np.maximum(Y.astype(np.int64) - 16, 0) * 1220542 + (1 << 19)
    u, v = U.astype(np.int64) - 128, V.astype(np.int64) - 128
    rgb = [(y + 1673527 * v) >> 20, (y - 852492 * v - 409993 * u) >> 20, (y + 2116026 * u) >> 20]
    return np.clip(np.stack(rgb, -1), 0, 255).astype(np.uint8)


def frame_to_rgb(frame: np.ndarray, pixel_format: str) -> np.ndarray:
    """the whole frame converted: uint8 [H, W, 3], chroma taken nearest"""
    Y, U, V, sub = planes(frame, pixel_format)
    H, W = Y.shape
    r, c = np.arange(H)[:, None] // sub, np.arange(W)[None, :] // 2
    return yuv_to_rgb(Y, U[r, c], V[r, c])


def letterbox_yuv_reference(frame: np.ndarray, pixel_format: str, resolution: int) -> np.ndarray:
    """the kernel's path: every tap (iy_k, ix_j) of a scaled pixel converted on its own, then h = sum_j rgb wx_j,
    v = sum_k h_k wy_k, (v + 2^21) >> 22 clamped, inside letterbox_geometry's bars -> uint8 [3, R, R] RGB"""
    Y, U, V, sub = planes(frame, pixel_format)
    H, W = Y.shape
    sw, sh, x0, y0 = letterbox_geometry(W, H, resolution)
    tx, ty = cubic_taps(W, sw), cubic_taps(H, sh)
    iy, ix = ty[:, :4][:, :, None, None], tx[:, :4][None, None, :, :]                  # [sh, 4, 1, 1], [1, 1, sw, 4]
    rgb = yuv_to_rgb(Y[iy, ix], U[iy // sub, ix // 2], V[iy // sub, ix // 2]).astype(np.int64)   # [sh, 4, sw, 4, 3]
    h = (rgb * tx[None, None, :, 4:, None]).sum(3)                                  # [sh, 4, sw, 3]
    v = (h * ty[:, 4:, None, None]).sum(1)                                          # [sh, sw, 3]
    assert np.abs(v).max(initial=0) < 2 ** 31
    canvas = np.zeros((resolution, resolution, 3), dtype=np.uint8)
    canvas[y0:y0 + sh, x0:x0 + sw] = np.clip((v + (1 << 21)) >> 22, 0, 255)
    return np.ascontiguousarray(canvas.transpose(2, 0, 1))
