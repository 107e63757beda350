"""numpy restatement of vlo_letterbox (include/vlo_b200.h): the two integer passes over video_ingest's tap tables, and the
black bars of letterbox_geometry.  The GPU tests hold the kernel to it bit for bit; the CPU tests hold it to OpenCV's
INTER_CUBIC (at most 1 per value) and to an exact copy at the canvas size."""
import numpy as np

from videollm_online_b200.video_ingest import cubic_taps, letterbox_geometry


def resize_reference(frame: np.ndarray, sw: int, sh: int) -> np.ndarray:
    """uint8 HWC frame -> uint8 [sh, sw, C]: h = sum_j src[y][ix_j] wx_j, v = sum_k h[iy_k] wy_k, (v + 2^21) >> 22
    clamped to [0, 255].  int64 here; the kernel's int32 holds every sum (|v| < 1.6e9)."""
    H, W = frame.shape[:2]
    tx, ty = cubic_taps(W, sw), cubic_taps(H, sh)
    src = frame.astype(np.int64)
    rows = src[ty[:, :4]]                                            # [sh, 4, W, C]
    h = (rows[:, :, tx[:, :4], :] * tx[None, None, :, 4:, None]).sum(3)   # [sh, 4, sw, C]
    v = (h * ty[:, 4:, None, None]).sum(1)                          # [sh, sw, C]
    assert np.abs(v).max(initial=0) < 2 ** 31
    return np.clip((v + (1 << 21)) >> 22, 0, 255).astype(np.uint8)


def letterbox_reference(frame: np.ndarray, resolution: int, bgr: bool = False) -> np.ndarray:
    """uint8 HWC frame (RGB, or BGR with bgr) -> the uint8 [3, R, R] RGB canvas vlo_letterbox writes"""
    H, W = frame.shape[:2]
    sw, sh, x0, y0 = letterbox_geometry(W, H, resolution)
    canvas = np.zeros((resolution, resolution, 3), dtype=np.uint8)
    canvas[y0:y0 + sh, x0:x0 + sw] = resize_reference(frame, sw, sh)
    if bgr:
        canvas = canvas[:, :, ::-1]
    return np.ascontiguousarray(canvas.transpose(2, 0, 1))
