"""YUV camera frames on the host: the numpy restatement of vlo_letterbox_planes' conversion against cv2.cvtColor, its fused
letterbox against letterbox_reference of cvtColor's RGB, the host checks of video_ingest.frame_layout, and the raw-stream
reader behind `cli --live_raw`."""
import io

import numpy as np
import pytest
import torch

from letterbox_reference import letterbox_reference
from videollm_online_b200._lib import VloError
from videollm_online_b200.video_ingest import (MAX_FRAME_SIDE, FrameRing, frame_layout, iter_raw_frames, parse_raw_spec,
                                               raw_frame_shape)
from yuv_reference import FORMATS, cv2_code, frame_to_rgb, letterbox_yuv_reference, yuv_noise

cv2 = pytest.importorskip("cv2")
R = 384
SIZES = [(2, 2), (4, 6), (6, 2), (62, 34), (640, 480), (1280, 720), (1920, 1080), (1080, 1920), (8192, 2)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("W,H", SIZES)
def test_conversion_equals_cvtcolor_on_noise(fmt, W, H):
    f = yuv_noise(W, H, fmt, W * 13 + H)
    np.testing.assert_array_equal(frame_to_rgb(f, fmt), cv2.cvtColor(f, cv2_code(fmt)))


@pytest.mark.parametrize("fmt", FORMATS)
def test_conversion_equals_cvtcolor_over_every_luma_and_the_chroma_extremes(fmt):
    """every Y value against U, V in {0, 128, 255}: the clamps at both ends and the black / white points"""
    chroma = [(u, v) for u in (0, 128, 255) for v in (0, 128, 255)]
    W, H = 256 * 2, 2 * len(chroma)   # luma pairs share a chroma sample: each Y value twice along a row
    Y = np.repeat(np.arange(256, dtype=np.uint8), 2)[None, :].repeat(H, 0)
    U = np.array([u for u, _ in chroma], dtype=np.uint8)[:, None].repeat(W // 2, 1)   # one chroma row per pair of lines
    V = np.array([v for _, v in chroma], dtype=np.uint8)[:, None].repeat(W // 2, 1)
    if fmt == "nv12":
        f = np.concatenate([Y.reshape(-1), np.stack([U, V], -1).reshape(-1)]).reshape(H * 3 // 2, W)
    elif fmt == "yuv420p":
        f = np.concatenate([Y.reshape(-1), U.reshape(-1), V.reshape(-1)]).reshape(H * 3 // 2, W)
    else:
        f = np.empty((H, W, 2), dtype=np.uint8)
        f[..., 0] = Y
        f[:, 0::2, 1] = U.repeat(2, 0)
        f[:, 1::2, 1] = V.repeat(2, 0)
    want = cv2.cvtColor(f, cv2_code(fmt))
    np.testing.assert_array_equal(frame_to_rgb(f, fmt), want)
    assert want.min() == 0 and want.max() == 255


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("W,H", [(2, 2), (384, 384), (640, 480), (1920, 1080), (1080, 1920), (62, 34), (8192, 2)])
def test_fused_letterbox_equals_letterbox_of_cvtcolor(fmt, W, H):
    """per-tap conversion then the integer passes == letterbox_reference(cv2.cvtColor(frame)), bit for bit"""
    f = yuv_noise(W, H, fmt, W + 7 * H)
    want = letterbox_reference(cv2.cvtColor(f, cv2_code(fmt)), R)
    np.testing.assert_array_equal(letterbox_yuv_reference(f, fmt, R), want)


def test_canvas_size_frame_is_its_conversion():
    f = yuv_noise(R, R, "nv12", 3)
    np.testing.assert_array_equal(letterbox_yuv_reference(f, "nv12", R), cv2.cvtColor(f, cv2_code("nv12")).transpose(2, 0, 1))


# ------------------------------------------------------------------------------------------------ host checks
def _t(shape, dtype=torch.uint8):
    return torch.zeros(shape, dtype=dtype)


def test_layout_of_each_format():
    W, H = 640, 480
    assert frame_layout(_t((H * 3 // 2, W)), "nv12")[:3] == (W, H, 2)
    assert frame_layout(_t((H * 3 // 2, W)), "nv12")[4] == [(0, 0, W), (0, W * H, W)]
    assert frame_layout(_t((H * 3 // 2, W)), "yuv420p")[4] == [(0, 0, W), (0, W * H, W // 2), (0, W * H * 5 // 4, W // 2)]
    assert frame_layout(_t((H, W, 2)), "yuyv422")[:3] == (W, H, 4)
    assert frame_layout(_t((H, W, 2)), "yuyv422")[4] == [(0, 0, 2 * W)]
    assert frame_layout(_t((H, W, 3)), None, bgr=True)[:3] == (W, H, 1)
    assert frame_layout(_t((1, 1, 3)))[:3] == (1, 1, 0)
    for fmt in FORMATS:
        assert tuple(frame_layout(_t(raw_frame_shape(W, H, fmt)), fmt)[3][0].shape) == raw_frame_shape(W, H, fmt)
    assert frame_layout(_t(raw_frame_shape(2, MAX_FRAME_SIDE, "nv12")), "nv12")[:2] == (2, MAX_FRAME_SIDE)
    assert frame_layout(_t(raw_frame_shape(MAX_FRAME_SIDE, 2, "yuyv422")), "yuyv422")[:2] == (MAX_FRAME_SIDE, 2)


BAD = {
    "odd width nv12": (lambda: _t((6, 5)), "nv12", False),
    "odd width i420": (lambda: _t((6, 7)), "yuv420p", False),
    "odd width yuyv": (lambda: _t((4, 5, 2)), "yuyv422", False),
    "odd height nv12 rows": (lambda: _t((7, 4)), "nv12", False),
    "odd height i420 rows": (lambda: _t((4, 4)), "yuv420p", False),
    "1 line yuyv": (lambda: _t((1, 4, 2)), "yuyv422", False),
    "width 8194 nv12": (lambda: _t((3, 8194)), "nv12", False),
    "height 8194 i420": (lambda: _t((8194 * 3 // 2, 4)), "yuv420p", False),
    "width 8194 yuyv": (lambda: _t((2, 8194, 2)), "yuyv422", False),
    "height 0 nv12": (lambda: _t((0, 4)), "nv12", False),
    "3-D nv12": (lambda: _t((6, 4, 1)), "nv12", False),
    "yuyv with 3 channels": (lambda: _t((4, 4, 3)), "yuyv422", False),
    "yuyv 2-D": (lambda: _t((4, 8)), "yuyv422", False),
    "float nv12": (lambda: _t((6, 4), torch.float32), "nv12", False),
    "int16 yuyv": (lambda: _t((4, 4, 2), torch.int16), "yuyv422", False),
    "numpy frame": (lambda: np.zeros((6, 4), np.uint8), "nv12", False),
    "cpu planes": (lambda: (_t((4, 4)), _t((2, 4))), "nv12", False),
    "planes for yuyv": (lambda: (_t((4, 8)),), "yuyv422", False),
    "planes for rgb": (lambda: (_t((4, 4)), _t((2, 4))), None, False),
    "unknown format": (lambda: _t((6, 4)), "nv21", False),
    "alias": (lambda: _t((6, 4)), "NV12", False),
    "i420 alias": (lambda: _t((6, 4)), "i420", False),
    "rgb24 name": (lambda: _t((4, 4, 3)), "rgb24", False),
    "bgr with nv12": (lambda: _t((6, 4)), "nv12", True),
    "bgr with yuyv": (lambda: _t((4, 4, 2)), "yuyv422", True),
    "rgb 4 channels": (lambda: _t((4, 4, 4)), None, False),
    "rgb width 8193": (lambda: _t((4, 8193, 3)), None, False),
}


@pytest.mark.parametrize("case", list(BAD))
def test_frame_layout_rejects(case):
    make, fmt, bgr = BAD[case]
    with pytest.raises(ValueError):
        frame_layout(make(), fmt, bgr)


def test_frame_ring_checks_every_frame_before_any_device_work():
    """push refuses a bad frame (VloError) before it touches the engine or a stream: here neither exists"""
    ring = FrameRing(engine=None, stream=None)
    good = _t((6, 4))
    for fmt, frames in [("nv12", [good, _t((6, 5))]), ("nv21", [good]), (None, [good])]:
        with pytest.raises(VloError):
            ring.push(frames, pixel_format=fmt)
    with pytest.raises(VloError):
        ring.push([good], bgr=True, pixel_format="nv12")
    assert ring.size(0) == 0 and not ring._pushes


# ------------------------------------------------------------------------------------------------ raw stream
class _Pipe(io.RawIOBase):
    """a pipe that hands out at most `chunk` bytes per read"""

    def __init__(self, data: bytes, chunk: int):
        self.data, self.pos, self.chunk = data, 0, chunk

    def readable(self):
        return True

    def readinto(self, b):
        n = min(len(b), self.chunk, len(self.data) - self.pos)
        b[:n] = self.data[self.pos:self.pos + n]
        self.pos += n
        return n


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("chunk", [1 << 20, 1000, 7])
def test_raw_reader_splits_frames_and_drops_a_truncated_tail(fmt, chunk):
    W, H = 64, 48
    frames = [yuv_noise(W, H, fmt, k) for k in range(3)]
    data = b"".join(f.tobytes() for f in frames)
    got = list(iter_raw_frames(_Pipe(data, chunk), W, H, fmt))
    assert len(got) == 3 and all(np.array_equal(a, b) and a.shape == raw_frame_shape(W, H, fmt) for a, b in zip(got, frames))
    with pytest.warns(UserWarning, match="dropped"):
        got = list(iter_raw_frames(_Pipe(data + frames[0].tobytes()[:-1], chunk), W, H, fmt))
    assert len(got) == 3 and np.array_equal(got[-1], frames[-1])
    assert list(iter_raw_frames(io.BytesIO(b""), W, H, fmt)) == []
    # the frames are what frame_layout takes for the format
    assert frame_layout(torch.from_numpy(got[0]), fmt)[:2] == (W, H)


def test_raw_spec():
    assert parse_raw_spec("1920x1080:nv12") == (1920, 1080, "nv12")
    assert parse_raw_spec("640x480:yuyv422") == (640, 480, "yuyv422")
    assert parse_raw_spec("2x2:yuv420p") == (2, 2, "yuv420p")
    for bad in ("1920x1080", "1920:nv12", "1920x1080:rgb24", "1921x1080:nv12", "640x481:yuv420p", "8194x2:nv12",
                "axb:nv12", "1920x1080:nv12:x"):
        with pytest.raises(ValueError):
            parse_raw_spec(bad)
