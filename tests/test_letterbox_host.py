"""The integer INTER_CUBIC letterbox that vlo_letterbox runs, on the host: video_ingest's tap tables and the numpy
restatement of the kernel's two passes (tests/letterbox_reference.py) against OpenCV's INTER_CUBIC, the geometry and
bars of letterbox_geometry, the size limits of the tap builder, and the native-size decode the live CLI pushes."""
import pathlib

import numpy as np
import pytest

from letterbox_reference import letterbox_reference, resize_reference
from videollm_online_b200.video_ingest import (MAX_FRAME_SIDE, cubic_taps, iter_video_frames, letterbox_geometry,
                                               letterbox_taps, read_video_resampled)

cv2 = pytest.importorskip("cv2")
GOLDEN = pathlib.Path(__file__).resolve().parent / "golden"
R = 384
SIZES = [(1920, 1080), (1280, 720), (640, 480), (1080, 1920), (192, 144), (385, 383), (4000, 10), (10, 4000)]


def _noise(W, H, seed):
    return np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8)


@pytest.mark.parametrize("W,H", SIZES)
def test_reference_tracks_opencv_inter_cubic(W, H):
    """uniform noise, the hardest case for a 1-LSB bound: at most 1 away from cv2.resize(INTER_CUBIC) per value"""
    f = _noise(W, H, W * 7 + H)
    sw, sh, _, _ = letterbox_geometry(W, H, R)
    got = resize_reference(f, sw, sh).astype(np.int16)
    want = cv2.resize(f, (sw, sh), interpolation=cv2.INTER_CUBIC).astype(np.int16)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1


def test_reference_tracks_opencv_on_demo_frames():
    """the demo clips' 192 x 144 frames, as decoded"""
    for name in ("demo_cooking", "demo_bicycle"):
        for k, f in enumerate(iter_video_frames(str(GOLDEN / f"{name}.mp4"), fps=2)):
            if k >= 6:
                break
            H, W = f.shape[:2]
            sw, sh, _, _ = letterbox_geometry(W, H, R)
            d = np.abs(resize_reference(f, sw, sh).astype(np.int16) -
                       cv2.resize(f, (sw, sh), interpolation=cv2.INTER_CUBIC).astype(np.int16))
            assert d.max() <= 1


def test_canvas_size_is_copied_unchanged():
    f = _noise(R, R, 1)
    np.testing.assert_array_equal(letterbox_reference(f, R), f.transpose(2, 0, 1))
    taps = cubic_taps(R, R)
    assert (taps[:, 4:] == [0, 2048, 0, 0]).all() and (taps[:, 1] == np.arange(R)).all()


@pytest.mark.parametrize("W,H", SIZES + [(383, 385), (97, 61), (8192, 33)])
@pytest.mark.parametrize("bgr", [False, True])
def test_bars_are_zero_and_geometry_is_letterbox_geometry(W, H, bgr):
    f = _noise(W, H, 3)
    out = letterbox_reference(f, R, bgr=bgr)
    sw, sh, x0, y0 = letterbox_geometry(W, H, R)
    assert out.shape == (3, R, R) and out.dtype == np.uint8
    inner = np.zeros((R, R), dtype=bool)
    inner[y0:y0 + sh, x0:x0 + sw] = True
    assert not out[:, ~inner].any()
    small = resize_reference(f, sw, sh)
    np.testing.assert_array_equal(out[:, y0:y0 + sh, x0:x0 + sw], small.transpose(2, 0, 1)[::-1 if bgr else 1])


def test_tap_tables_layout():
    """the horizontal table (sw rows) then the vertical one (sh rows); indices clamped to the frame; weights sum to 2048
    up to the rounding of each (OpenCV's tables have the same property)"""
    W, H = 1280, 720
    sw, sh, _, _ = letterbox_geometry(W, H, R)
    t = letterbox_taps(W, H, R)
    assert t.dtype == np.int32 and t.shape == (sw + sh, 8)
    np.testing.assert_array_equal(t[:sw], cubic_taps(W, sw))
    np.testing.assert_array_equal(t[sw:], cubic_taps(H, sh))
    assert t[:sw, :4].min() >= 0 and t[:sw, :4].max() <= W - 1 and t[sw:, :4].max() <= H - 1
    assert np.abs(t[:, 4:].sum(1) - 2048).max() <= 2


@pytest.mark.parametrize("W,H", [(0, 480), (640, 0), (MAX_FRAME_SIDE + 1, 480), (640, MAX_FRAME_SIDE + 1), (-1, 5)])
def test_tap_builder_rejects_sizes_outside_the_limits(W, H):
    with pytest.raises(ValueError):
        letterbox_taps(W, H, R)


def test_tap_builder_takes_the_limits():
    assert letterbox_taps(MAX_FRAME_SIDE, 1, R).shape == (R + 2, 8)
    assert letterbox_taps(1, MAX_FRAME_SIDE, R).shape == (2 + R, 8)
    with pytest.raises(ValueError):
        cubic_taps(0, 4)


def test_native_decode_is_what_read_video_resampled_letterboxes():
    """iter_video_frames (what `cli --live` pushes) yields the native frames read_video_resampled converts, one per
    output frame"""
    path = str(GOLDEN / "demo_cooking.mp4")
    native = list(iter_video_frames(path, fps=2))
    clip = read_video_resampled(path, fps=2, resolution=R)
    assert len(native) == clip.shape[0] and native[0].shape[2] == 3 and native[0].shape[:2] != (R, R)
    for k in (0, len(native) // 2, len(native) - 1):
        f = native[k]
        H, W = f.shape[:2]
        sw, sh, x0, y0 = letterbox_geometry(W, H, R)
        canvas = np.zeros((R, R, 3), dtype=np.uint8)
        canvas[y0:y0 + sh, x0:x0 + sw] = cv2.resize(f, (sw, sh), interpolation=cv2.INTER_CUBIC)
        np.testing.assert_array_equal(clip[k].numpy(), cv2.cvtColor(canvas, cv2.COLOR_BGR2RGB).transpose(2, 0, 1))
