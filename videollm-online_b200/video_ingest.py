"""Video ingest for the streaming demo (SURVEY 8(f).2): decode -> frame-rate resample -> letterbox to a square.

The reference preprocesses a clip once with an external ffmpeg binary (`ffmpeg_once`, data/utils.py:51-66, called
from demo/cli.py:15-20: `-r <fps>` and `scale` of the longer side to `resolution` followed by a centred `pad` to
`resolution x resolution` in black) and then decodes the cached file with `torchvision.io.read_video`
(demo/inference.py:111-115).  Neither the ffmpeg binary nor a torchvision video decoder exists in this image, so the
same geometry and sampling rule are applied here in one pass with OpenCV:

  * output frame k shows the source frame whose timestamp is nearest to k / fps (ffmpeg's fps conversion with its
    default rounding), for k < round(duration * fps);
  * the longer side is scaled to `resolution` with a bicubic filter (ffmpeg_once's `-sws_flags bicubic`), the shorter
    side to the nearest EVEN size that keeps the aspect ratio (ffmpeg's `-2`), and the result is centred on a black
    square ((ow-iw)/2, (oh-ih)/2 rounded down).

Not bit-identical to libswscale's bicubic taps (documented; the frames then go through the same uint8 -> ViT path).
`read_video_resampled` runs on the host: it returns a uint8 [T, 3, R, R] CPU tensor in RGB that `LiveInfer.load_video`
moves to the GPU.

Live frames (`push_frames`) are letterboxed on the device instead (`Engine.letterbox`, vlo_letterbox): `cubic_taps` builds
the integer INTER_CUBIC tap tables the kernel reads, and `FrameRing` holds a session's pushed frames until they are
encoded.  Frames may come as packed RGB / BGR or, named by ffmpeg's `-pix_fmt`, as NV12, I420 (`yuv420p`) or YUYV
(`yuyv422`), converted to RGB on the device (vlo_letterbox_planes); `frame_layout` checks them on the host, and
`iter_raw_frames` splits a raw byte stream of them (ffmpeg `-f rawvideo`) into frames.
"""
from __future__ import annotations

import collections
import warnings
from typing import BinaryIO, Iterator, Optional, Tuple

import numpy as np
import torch

from ._lib import VloError

MAX_FRAME_SIDE = 8192   # widest / tallest native frame vlo_letterbox takes
TAP_BITS = 11           # integer tap weights are round(w * 2^11), OpenCV's INTER_RESIZE_COEF_BITS
# pixel_format (ffmpeg's -pix_fmt names) -> vlo_frame_planes.format; None is packed RGB (0) or BGR (1), chosen by bgr
PIXEL_FORMATS = {"nv12": 2, "yuv420p": 3, "yuyv422": 4}


def letterbox_geometry(width: int, height: int, resolution: int) -> Tuple[int, int, int, int]:
    """(scaled_w, scaled_h, x0, y0) of ffmpeg_once's scale + pad filter chain."""
    if width > height:
        sw = resolution
        sh = int(round(height * resolution / width / 2.0)) * 2
    else:
        sh = resolution
        sw = int(round(width * resolution / height / 2.0)) * 2
    sw, sh = max(2, min(sw, resolution)), max(2, min(sh, resolution))
    return sw, sh, (resolution - sw) // 2, (resolution - sh) // 2


def cubic_taps(n_in: int, n_out: int) -> np.ndarray:
    """int32 [n_out, 8] tap table of one axis for vlo_letterbox: per output coordinate d the source indices
    clamp(s - 1 + k, 0, n_in - 1) then the weights round_half_even(w_k * 2048), k = 0..3, with
      f = fp32((d + 0.5) * (n_in / n_out) - 0.5)   (in fp64, rounded once),  s = floor(f),  t = f - s   (fp32)
    and OpenCV's cubic weights of A = -0.75, every operation rounded in fp32:
      w0 = ((A(t+1) - 5A)(t+1) + 8A)(t+1) - 4A,  w1 = ((A+2)t - (A+3))t t + 1,  w2 = w1 at 1 - t,  w3 = 1 - w0 - w1 - w2.
    Raises ValueError unless 1 <= n_in <= MAX_FRAME_SIDE and n_out >= 1."""
    if not (1 <= n_in <= MAX_FRAME_SIDE) or n_out < 1:
        raise ValueError(f"cubic_taps: a side of {n_in} pixels is outside [1, {MAX_FRAME_SIDE}] (or {n_out} outputs)")
    f32 = np.float32
    d = np.arange(n_out, dtype=np.float64)
    f = ((d + 0.5) * (n_in / n_out) - 0.5).astype(f32)
    s = np.floor(f)
    t = f - s
    A, one = f32(-0.75), f32(1)
    x = t + one
    w0 = ((A * x - f32(5) * A) * x + f32(8) * A) * x - f32(4) * A
    w1 = ((A + f32(2)) * t - (A + f32(3))) * t * t + one
    u = one - t
    w2 = ((A + f32(2)) * u - (A + f32(3))) * u * u + one
    w3 = one - w0 - w1 - w2
    w = np.stack([w0, w1, w2, w3], 1)
    assert w.dtype == np.float32
    iw = np.rint(w * f32(1 << TAP_BITS)).astype(np.int32)
    idx = np.clip(s.astype(np.int64)[:, None] - 1 + np.arange(4)[None, :], 0, n_in - 1).astype(np.int32)
    return np.ascontiguousarray(np.concatenate([idx, iw], 1))


def letterbox_taps(width: int, height: int, resolution: int) -> np.ndarray:
    """The tap tables of a width x height frame letterboxed to resolution^2, as one int32 array: the horizontal table
    (sw rows of 8) then the vertical one (sh rows), (sw, sh) from letterbox_geometry.  Raises ValueError unless both
    sides lie in [1, MAX_FRAME_SIDE]."""
    for side in (width, height):
        if not (isinstance(side, int) and 1 <= side <= MAX_FRAME_SIDE):
            raise ValueError(f"letterbox: a frame side of {side!r} pixels is outside [1, {MAX_FRAME_SIDE}]")
    sw, sh, _, _ = letterbox_geometry(width, height, resolution)
    return np.concatenate([cubic_taps(width, sw), cubic_taps(height, sh)], 0)


def raw_frame_shape(width: int, height: int, pixel_format: str) -> Tuple[int, ...]:
    """The uint8 shape of one width x height frame in pixel_format as one tensor (the layout of ffmpeg's rawvideo and of
    cv2): [H * 3 / 2, W] for the 4:2:0 formats (the Y plane, then the chroma planes packed), [H, W, 2] for YUYV."""
    if pixel_format not in PIXEL_FORMATS:
        raise ValueError(f"unknown pixel format {pixel_format!r}; one of {sorted(PIXEL_FORMATS)} (or None: RGB / BGR)")
    return (height, width, 2) if pixel_format == "yuyv422" else (height * 3 // 2, width)


def _check_sides(width: int, height: int, pixel_format: Optional[str]):
    lo = 1 if pixel_format is None else 2
    if not (lo <= width <= MAX_FRAME_SIDE and lo <= height <= MAX_FRAME_SIDE):
        raise ValueError(f"a {width} x {height} frame; both sides must lie in [{lo}, {MAX_FRAME_SIDE}]")
    if pixel_format is not None and width % 2:
        raise ValueError(f"a {pixel_format} frame {width} pixels wide; the width must be even")
    if pixel_format in ("nv12", "yuv420p") and height % 2:
        raise ValueError(f"a {pixel_format} frame {height} lines high; the height must be even")


def frame_layout(frame, pixel_format: Optional[str] = None, bgr: bool = False):
    """Check one frame of `push_frames` / `Engine.letterbox` on the host, before any device work, and return
    (width, height, vlo_frame_planes.format, parts, planes): the frame's tensors and, per plane, (index into parts, byte
    offset, pitch).  Raises ValueError on anything vlo_letterbox_planes would refuse.  A frame is
      pixel_format None               uint8 [H, W, 3] packed RGB (BGR with bgr=True), 1 <= W, H <= 8192, CPU or device;
      "nv12", "yuv420p" (I420)        uint8 [H * 3 / 2, W], the planes one after the other (raw_frame_shape), CPU or
                                      device; or, on the device only, a tuple of 2-D uint8 planes (Y [H, W] and UV
                                      [H / 2, W] for NV12; Y, U [H / 2, W / 2] and V for I420) whose rows may be padded
                                      (stride(1) == 1, stride(0) >= the row bytes): a decoder's surface, read in place;
      "yuyv422"                       uint8 [H, W, 2] (pairs Y0 U Y1 V), CPU or device.
    The YUV formats take 2 <= W, H <= 8192 with W even, and H even for the 4:2:0 formats.  The offsets and pitches of a
    single tensor are those of its contiguous copy, which is what Engine.letterbox reads."""
    if pixel_format is not None and pixel_format not in PIXEL_FORMATS:
        raise ValueError(f"unknown pixel format {pixel_format!r}; one of {sorted(PIXEL_FORMATS)} (or None: RGB / BGR)")
    if pixel_format is not None and bgr:
        raise ValueError(f"bgr=True names a packed RGB order; it does not combine with pixel_format={pixel_format!r}")
    if isinstance(frame, (tuple, list)):
        if pixel_format not in ("nv12", "yuv420p"):
            raise ValueError(f"frames as separate planes are NV12 or yuv420p; got a tuple with pixel_format={pixel_format!r}")
        n = 2 if pixel_format == "nv12" else 3
        if len(frame) != n or not all(isinstance(p, torch.Tensor) for p in frame):
            raise ValueError(f"a {pixel_format} frame as planes is a tuple of {n} tensors")
        for p in frame:
            if p.dtype != torch.uint8 or p.dim() != 2 or p.device.type != "cuda":
                raise ValueError(f"{pixel_format} planes must be 2-D uint8 device tensors, got {p.dtype} "
                                 f"{tuple(p.shape)} on {p.device}")
        H, W = int(frame[0].shape[0]), int(frame[0].shape[1])
        _check_sides(W, H, pixel_format)
        want = [(H, W), (H // 2, W)] if n == 2 else [(H, W), (H // 2, W // 2), (H // 2, W // 2)]
        planes = []
        for k, (p, shape) in enumerate(zip(frame, want)):
            if tuple(p.shape) != shape:
                raise ValueError(f"{pixel_format} plane {k} of a {W} x {H} frame must be {list(shape)}, got {list(p.shape)}")
            pitch = p.stride(0)
            if p.stride(1) != 1 or pitch < shape[1] or pitch >= 2 ** 31:
                raise ValueError(f"{pixel_format} plane {k}: rows must be unit-stride with a pitch in [{shape[1]}, 2^31), "
                                 f"got strides {p.stride()}")
            planes.append((k, 0, pitch))
        return W, H, PIXEL_FORMATS[pixel_format], tuple(frame), planes
    if not isinstance(frame, torch.Tensor) or frame.dtype != torch.uint8:
        raise ValueError(f"frames must be uint8 tensors, got {getattr(frame, 'dtype', type(frame))}")
    shape = tuple(frame.shape)
    if pixel_format is None:
        if len(shape) != 3 or shape[2] != 3:
            raise ValueError(f"packed RGB / BGR frames are uint8 HWC tensors with 3 channels, got {list(shape)}")
        H, W = shape[:2]
        _check_sides(W, H, None)
        return W, H, int(bool(bgr)), (frame,), [(0, 0, 3 * W)]
    if pixel_format == "yuyv422":
        if len(shape) != 3 or shape[2] != 2:
            raise ValueError(f"yuyv422 frames are uint8 [H, W, 2] tensors, got {list(shape)}")
        H, W = shape[:2]
        _check_sides(W, H, pixel_format)
        return W, H, PIXEL_FORMATS[pixel_format], (frame,), [(0, 0, 2 * W)]
    if len(shape) != 2 or shape[0] % 3:
        raise ValueError(f"{pixel_format} frames are uint8 [H * 3 / 2, W] tensors (or a tuple of device planes), "
                         f"got {list(shape)}")
    H, W = shape[0] // 3 * 2, shape[1]
    _check_sides(W, H, pixel_format)
    if pixel_format == "nv12":
        planes = [(0, 0, W), (0, W * H, W)]
    else:
        planes = [(0, 0, W), (0, W * H, W // 2), (0, W * H + (W // 2) * (H // 2), W // 2)]
    return W, H, PIXEL_FORMATS[pixel_format], (frame,), planes


def parse_raw_spec(spec: str) -> Tuple[int, int, str]:
    """`WxH:FORMAT` (cli --live_raw, e.g. 1920x1080:nv12) -> (width, height, pixel_format); ValueError if malformed or
    outside frame_layout's limits."""
    try:
        size, pixel_format = spec.split(":")
        width, height = (int(v) for v in size.lower().split("x"))
    except ValueError:
        raise ValueError(f"a raw video spec is WxH:FORMAT, e.g. 1920x1080:nv12; got {spec!r}") from None
    raw_frame_shape(width, height, pixel_format)
    _check_sides(width, height, pixel_format)
    return width, height, pixel_format


def iter_raw_frames(stream: BinaryIO, width: int, height: int, pixel_format: str) -> Iterator[np.ndarray]:
    """Split a raw video byte stream (ffmpeg `-f rawvideo -pix_fmt <pixel_format>`, a pipe or a file) into frames of
    raw_frame_shape, yielded as uint8 arrays as they arrive.  A stream that ends inside a frame drops that frame with a
    warning."""
    shape = raw_frame_shape(width, height, pixel_format)
    _check_sides(width, height, pixel_format)
    n = int(np.prod(shape))
    while True:
        buf = bytearray(n)
        view, got = memoryview(buf), 0
        while got < n:   # a pipe returns what it has: read until the frame is whole or the stream ends
            k = stream.readinto(view[got:])
            if not k:
                break
            got += k
        if got < n:
            if got:
                warnings.warn(f"raw video ended {got} bytes into a {n}-byte {pixel_format} frame; that frame is dropped")
            return
        yield np.frombuffer(buf, dtype=np.uint8).reshape(shape)


class FrameRing:
    """The frames pushed into a session, indexed as the session indexes a loaded clip (`video[r:r2]`, `video[i]`,
    `video.size(0)`): frame `first + j` is the j-th frame pushed.  Each push letterboxes its native frames on `stream`
    (Engine.letterbox, the session's encode-ahead stream) and records one event; reading frames makes the reading stream
    wait on the events of their pushes, so they may be encoded on any stream, and the reading stream never waits for a
    native-frame copy otherwise.  A frame is released when it is read (the session encodes each frame once): the
    canvases of a push are dropped once all of them have been read, after which their memory is reused only behind the
    work already enqueued on the streams that read them.  So the ring holds the frames pushed and not yet encoded."""

    def __init__(self, engine, stream: torch.cuda.Stream, first: int = 0):
        self.engine, self.stream = engine, stream
        self.first = self.end = int(first)
        self._pushes = collections.deque()   # [first index, canvases [n, 3, R, R], event, unread indices]

    def push(self, frames, bgr: bool = False, pixel_format: Optional[str] = None):
        """Letterbox `frames` (as frame_layout takes them: HWC uint8 tensors or, in pixel_format, YUV frames or device
        planes; CPU or CUDA, any sizes) into the ring, as the next frames.  Every frame is checked before any device work.
        CUDA frames may still be being written on the caller's current stream: `stream` reads them only after the work
        enqueued there so far, and their memory is not reused before that read, even if the caller drops them at once."""
        frames = list(frames)
        if not frames:
            return
        try:
            parts = [frame_layout(f, pixel_format, bgr)[3] for f in frames]
        except ValueError as e:
            raise VloError(f"push_frames: {e}") from None
        on_device = [t for ts in parts for t in ts if t.device == self.engine.device]
        if on_device:
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream(self.engine.device))
            self.stream.wait_event(ready)
            for f in on_device:
                f.record_stream(self.stream)
        with torch.cuda.stream(self.stream):
            canvases = self.engine.letterbox(frames, bgr=bgr, pixel_format=pixel_format)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        self._pushes.append([self.end, canvases, ev, set(range(self.end, self.end + len(frames)))])
        self.end += len(frames)

    def size(self, dim: int = 0) -> int:
        if dim != 0:
            raise IndexError("FrameRing.size: only dim 0 (frames pushed, counted from frame 0)")
        return self.end

    def __len__(self) -> int:
        return self.end

    def __getitem__(self, key):
        if isinstance(key, slice):
            start, stop, step = key.indices(self.end)
            if step != 1:
                raise IndexError("FrameRing: only contiguous slices")
            if key.stop is not None and key.stop > self.end:   # never fewer frames than asked for
                raise IndexError(f"FrameRing: frames up to {key.stop - 1} asked for, {self.end} pushed")
            idx = range(start, max(start, stop))
        else:
            i = int(key)
            idx = range(i, i + 1)
        owners = []
        for i in idx:
            p = next((p for p in self._pushes if i in p[3]), None)
            if p is None:
                what = "not pushed yet" if i >= self.end else "already encoded and released" if i >= self.first else \
                    "before the first frame pushed into this session"
                raise IndexError(f"FrameRing: frame {i} is {what}")
            owners.append(p)
        cur = torch.cuda.current_stream(self.engine.device)
        parts = []   # [push, first, end): runs of consecutive frames of one push
        for i, p in zip(idx, owners):
            if not any(q[0] is p for q in parts):
                cur.wait_event(p[2])
                p[1].record_stream(cur)
            j = i - p[0]
            if parts and parts[-1][0] is p and parts[-1][2] == j:
                parts[-1][2] = j + 1
            else:
                parts.append([p, j, j + 1])
            p[3].discard(i)   # released: a push whose frames have all been read is dropped below
        self._pushes = collections.deque(p for p in self._pushes if p[3])
        out = [p[1][a:b] for p, a, b in parts]
        out = out[0] if len(out) == 1 else torch.cat(out) if out else self._empty()
        return out if isinstance(key, slice) else out[0]

    def check_pushed(self, frame_idx: int):
        """Raise IndexError unless frame `frame_idx` has been pushed: a session checks before it changes any state."""
        if frame_idx >= self.end:
            raise IndexError(f"frame {frame_idx} is not pushed yet ({self.end} frames pushed): push_frames before "
                             f"input_video_stream reaches it")

    def _empty(self):
        R = self.engine.cfg.frame_resolution
        return torch.empty(0, 3, R, R, dtype=torch.uint8, device=self.engine.device)


def resample_indices(n_src: int, src_fps: float, fps: float) -> list:
    """Source frame index shown by every output frame of a constant-frame-rate conversion to `fps`."""
    if n_src <= 0 or src_fps <= 0 or fps <= 0:
        return []
    n_out = max(1, int(round(n_src / src_fps * fps)))
    return [min(n_src - 1, int(round(k / fps * src_fps))) for k in range(n_out)]


def iter_video_frames(path: str, fps: Optional[float] = None) -> Iterator[np.ndarray]:
    """Decode `path` with OpenCV and yield its frames at their native size (uint8 HWC, BGR), converted to `fps` frames/s
    by `resample_indices` (a source frame shown by several output frames is yielded once per output frame, as the same
    array).  Streaming: only the frames the output keeps are decoded to pixels."""
    try:
        import cv2
    except Exception as e:  # pragma: no cover
        raise RuntimeError(f"no video decoder available for {path}: {e}")

    def count_frames() -> int:
        cap = cv2.VideoCapture(path)
        n = 0
        while cap.grab():
            n += 1
        cap.release()
        return n

    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        raise RuntimeError(f"could not open video {path}")
    src_fps = float(cap.get(cv2.CAP_PROP_FPS) or 0.0)
    n_src = int(cap.get(cv2.CAP_PROP_FRAME_COUNT) or 0)
    if n_src <= 0:                       # container without a frame count: one extra demux pass
        n_src = count_frames()
    if n_src <= 0:
        cap.release()
        raise RuntimeError(f"could not decode any frame from {path}")
    wanted = resample_indices(n_src, src_fps, float(fps)) if (fps is not None and src_fps > 0) else list(range(n_src))

    k, i, last = 0, 0, None
    try:
        while k < len(wanted):
            if wanted[k] > i:                # skip without decoding to pixels
                if not cap.grab():
                    break
                i += 1
                continue
            ok, fr = cap.read()              # source frame i is wanted (possibly several times: fps above the source rate)
            if not ok:
                break
            last = fr
            while k < len(wanted) and wanted[k] == i:
                yield fr
                k += 1
            i += 1
    finally:
        cap.release()
    if last is None:
        raise RuntimeError(f"could not decode any frame from {path}")
    while k < len(wanted):               # the container over-reported its length: hold the last frame (ffmpeg -r pads the same way)
        yield last
        k += 1


def read_video_resampled(path: str, fps: Optional[float] = None, resolution: Optional[int] = None) -> torch.Tensor:
    """Decode `path`; optionally convert to `fps` frames/s and letterbox to `resolution`.  uint8 [T,3,H,W], RGB.
    Streaming: only the frames the output keeps are converted and held (a 107 s 1440x1080 clip is 3204 source frames =
    15 GB decoded, but 214 frames of 384x384 at 2 FPS)."""
    def convert(fr):
        import cv2
        h, w = fr.shape[:2]
        if resolution is not None and (h != resolution or w != resolution):
            sw, sh, x0, y0 = letterbox_geometry(w, h, resolution)
            small = cv2.resize(fr, (sw, sh), interpolation=cv2.INTER_CUBIC)
            canvas = np.zeros((resolution, resolution, 3), dtype=small.dtype)
            canvas[y0:y0 + sh, x0:x0 + sw] = small
            fr = canvas
        return torch.from_numpy(cv2.cvtColor(fr, cv2.COLOR_BGR2RGB)).permute(2, 0, 1).contiguous()

    out, src, last = [], None, None
    for fr in iter_video_frames(path, fps):
        if fr is not src:                # a repeated source frame is converted once
            src, last = fr, convert(fr)
        out.append(last)
    return torch.stack(out).contiguous()
