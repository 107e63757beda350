"""YUV camera frames (NV12, I420, YUYV) letterboxed on the device: vlo_letterbox_planes against letterbox_reference of
cv2.cvtColor's RGB bit for bit, its argument checks, and sessions pushed YUV frames against the same sessions pushed
cvtColor's RGB frames.

  A. The kernel: every format at sizes from 2 x 2 to 3840 x 2160 and 8192 x 2, from CPU and device frames; padded planes
     (pitches not a multiple of 16, padding filled with 0xFF) read in place, as separate plane tensors and through the C
     interface; batches mixing formats, sizes and packed RGB / BGR in one launch against solo launches; a batch larger
     than one launch takes, split.  Outputs are pre-filled, so a byte the kernel does not write shows.
  B. Each bad argument: a non-zero return, a message, and the canvas left as it was.
  C. LiveInfer and StreamScheduler: the conversation, every decision row and the KV cache of sessions pushed NV12 (CPU),
     I420, YUYV or NV12 device planes equal those of the sessions pushed cvtColor's RGB of the same frames."""
import ctypes as C

import numpy as np
import pytest
import torch

from letterbox_reference import letterbox_reference
from yuv_reference import FORMATS, cv2_code, yuv_noise

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

R = 384
SIZES = [(2, 2), (384, 384), (640, 480), (1920, 1080), (1080, 1920), (3840, 2160), (8192, 2)]
MAX_BATCH = 56   # more than the 48 frames one launch takes
CODE = {"nv12": 2, "yuv420p": 3, "yuyv422": 4}


def _want(f, fmt):
    return torch.from_numpy(letterbox_reference(cv2.cvtColor(f, cv2_code(fmt)), R))


@pytest.fixture(scope="module")
def eng():
    from videollm_online_b200 import tiny_config
    from videollm_online_b200.engine import Engine
    e = Engine(tiny_config(frame_resolution=R), "cuda:0", max_vit_batch=MAX_BATCH)
    yield e
    e.close()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _pitched(plane: np.ndarray, pitch: int, fill: int = 0xFF, offset: int = 3) -> torch.Tensor:
    """a 2-D device view of `plane` with rows `pitch` bytes apart, `offset` bytes into a buffer filled with `fill`"""
    rows, n = plane.shape
    buf = torch.full((offset + rows * pitch + 64,), fill, dtype=torch.uint8, device="cuda")
    view = buf[offset:offset + rows * pitch].view(rows, pitch)[:, :n]
    view.copy_(torch.from_numpy(np.ascontiguousarray(plane)))
    return view


def _planes_420(f: np.ndarray, fmt: str, pitch_pad: int, fill: int = 0xFF):
    """the device planes of a raw 4:2:0 frame, each row padded by pitch_pad bytes"""
    from yuv_reference import planes
    Y, U, V, _ = planes(f, fmt)
    H, W = Y.shape
    if fmt == "nv12":
        return (_pitched(Y, W + pitch_pad, fill), _pitched(np.stack([U, V], -1).reshape(H // 2, W), W + pitch_pad, fill))
    return tuple(_pitched(p, p.shape[1] + pitch_pad, fill) for p in (Y, U, V))


def _desc(eng, d, fmt_code, W, H, ptrs, pitches, keep):
    taps, sw = eng._letterbox_taps(W, H)
    keep.append(taps)
    for q in range(3):
        d.d_planes[q] = ptrs[q] if q < len(ptrs) else None
        d.pitch[q] = pitches[q] if q < len(pitches) else 0
    d.d_taps, d.format, d.width, d.height, d.x_taps, d.y_taps = taps.data_ptr(), fmt_code, W, H, 0, sw


def _contig_desc(eng, d, fmt, f, keep):
    """a descriptor of a contiguous device copy of raw frame f (format name, or "rgb" / "bgr" for packed HWC)"""
    t = torch.from_numpy(f).cuda()
    keep.append(t)
    if fmt in ("rgb", "bgr"):
        H, W = f.shape[:2]
        return _desc(eng, d, int(fmt == "bgr"), W, H, [t.data_ptr()], [3 * W], keep)
    from videollm_online_b200.video_ingest import frame_layout
    W, H, code, _, planes = frame_layout(t, fmt)
    _desc(eng, d, code, W, H, [t.data_ptr() + o for _, o, _ in planes], [p for _, _, p in planes], keep)


def _raw(eng, items, fill=0xAB):
    """vlo_letterbox_planes over [(fmt, raw frame)] in one call, into an output filled with `fill`"""
    from videollm_online_b200._lib import VloFramePlanes, check
    descs, keep = (VloFramePlanes * len(items))(), []
    for d, (fmt, f) in zip(descs, items):
        _contig_desc(eng, d, fmt, f, keep)
    out = torch.full((len(items), 3, R, R), fill, dtype=torch.uint8, device="cuda")
    check(eng.lib.vlo_letterbox_planes(eng._h, descs, len(items), C.c_void_p(out.data_ptr()), _stream()),
          "vlo_letterbox_planes")
    torch.cuda.synchronize()
    return out.cpu()


# ======================================================================================================= A. kernel
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("W,H", SIZES)
def test_kernel_equals_reference(eng, fmt, W, H):
    f = yuv_noise(W, H, fmt, W * 31 + H)
    want = _want(f, fmt)
    assert torch.equal(eng.letterbox([torch.from_numpy(f)], pixel_format=fmt).cpu()[0], want), "CPU frame"
    assert torch.equal(eng.letterbox([torch.from_numpy(f).cuda()], pixel_format=fmt).cpu()[0], want), "device frame"
    assert torch.equal(_raw(eng, [(fmt, f)], fill=0xAB)[0], want) and torch.equal(_raw(eng, [(fmt, f)], fill=0)[0], want)


def test_canvas_size_frame_is_its_conversion(eng):
    for fmt in FORMATS:
        f = yuv_noise(R, R, fmt, 9)
        got = eng.letterbox([torch.from_numpy(f)], pixel_format=fmt).cpu()[0]
        assert torch.equal(got, torch.from_numpy(cv2.cvtColor(f, cv2_code(fmt))).permute(2, 0, 1)), fmt


@pytest.mark.parametrize("fmt", ["nv12", "yuv420p"])
@pytest.mark.parametrize("W,H", [(2, 2), (62, 34), (640, 480), (1920, 1080)])
@pytest.mark.parametrize("pad", [3, 17, 194])
def test_padded_device_planes_are_read_in_place(eng, fmt, W, H, pad):
    """separate plane tensors with padded rows (pitch W + pad: not a multiple of 16, planes 3 bytes off alignment): the
    canvas of the packed frame, whatever the padding holds"""
    f = yuv_noise(W, H, fmt, W + H + pad)
    want = eng.letterbox([torch.from_numpy(f)], pixel_format=fmt).cpu()
    assert torch.equal(want[0], _want(f, fmt))
    for fill in (0xFF, 0x00):
        planes = _planes_420(f, fmt, pad, fill)
        assert all(p.stride(0) != p.shape[1] for p in planes)
        assert torch.equal(eng.letterbox([planes], pixel_format=fmt).cpu(), want), f"padding {fill:#x}"


@pytest.mark.parametrize("W,H", [(2, 2), (640, 480), (1920, 1080)])
def test_pitched_planes_through_the_c_interface(eng, W, H):
    """every format, and packed RGB, with pitches past the row bytes and 0xFF padding, one launch"""
    from videollm_online_b200._lib import VloFramePlanes, check
    items, descs, keep = [], (VloFramePlanes * 4)(), []
    for k, fmt in enumerate(FORMATS + ("rgb",)):
        if fmt == "rgb":
            f = np.random.default_rng(k).integers(0, 256, (H, W, 3), dtype=np.uint8)
            v = _pitched(f.reshape(H, 3 * W), 3 * W + 5)
            _desc(eng, descs[k], 0, W, H, [v.data_ptr()], [v.stride(0)], keep)
            items.append(torch.from_numpy(letterbox_reference(f, R)))
            keep.append(v)
        else:
            f = yuv_noise(W, H, fmt, k)
            ps = _planes_420(f, fmt, 11) if fmt != "yuyv422" else (_pitched(f.reshape(H, 2 * W), 2 * W + 7),)
            _desc(eng, descs[k], CODE[fmt], W, H, [p.data_ptr() for p in ps], [p.stride(0) for p in ps], keep)
            items.append(_want(f, fmt))
            keep.extend(ps)
    out = torch.full((4, 3, R, R), 0xAB, dtype=torch.uint8, device="cuda")
    check(eng.lib.vlo_letterbox_planes(eng._h, descs, 4, C.c_void_p(out.data_ptr()), _stream()), "vlo_letterbox_planes")
    torch.cuda.synchronize()
    for k, want in enumerate(items):
        assert torch.equal(out[k].cpu(), want), k


MIXED = [("nv12", 1920, 1080), ("rgb", 640, 480), ("yuv420p", 1280, 720), ("yuyv422", 640, 480), ("bgr", 97, 61),
         ("nv12", 2, 2), ("yuv420p", 1080, 1920), ("yuyv422", 8192, 2), ("nv12", 384, 384), ("yuv420p", 62, 34)]


def _mixed_frame(fmt, W, H, seed):
    if fmt in ("rgb", "bgr"):
        f = np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8)
        return f, torch.from_numpy(letterbox_reference(f, R, bgr=fmt == "bgr"))
    f = yuv_noise(W, H, fmt, seed)
    return f, _want(f, fmt)


@pytest.mark.parametrize("B", [2, 3, 5, 8, 10])
def test_mixed_batch_equals_solo_launches(eng, B):
    items, wants = [], []
    for k in range(B):
        fmt, W, H = MIXED[(3 * B + k) % len(MIXED)]
        f, want = _mixed_frame(fmt, W, H, 100 * B + k)
        items.append((fmt, f))
        wants.append(want)
    got = _raw(eng, items)
    for k, item in enumerate(items):
        assert torch.equal(got[k], _raw(eng, [item])[0]), f"frame {k} {item[0]} {item[1].shape}"
        assert torch.equal(got[k], wants[k]), f"frame {k} {item[0]} {item[1].shape}"


def test_more_frames_than_one_launch_are_split(eng):
    """MAX_BATCH frames in one vlo_letterbox_planes call: two launches (48 + 8), every frame its reference"""
    items = [("nv12", yuv_noise(64 + 2 * k, 48 + 2 * (k % 5), "nv12", k)) for k in range(MAX_BATCH)]
    n0 = eng.launch_count()
    got = _raw(eng, items)
    assert eng.launch_count() - n0 == 2
    for k, (fmt, f) in enumerate(items):
        assert torch.equal(got[k], _want(f, fmt)), k
    # the public entry: more than max_vit_batch frames go in several calls
    frames = [torch.from_numpy(f) for _, f in items] + [torch.from_numpy(yuv_noise(40, 30, "nv12", 999))]
    got = eng.letterbox(frames, pixel_format="nv12").cpu()
    assert all(torch.equal(got[k], _want(f.numpy(), "nv12")) for k, f in enumerate(frames))


# ==================================================================================================== B. arguments
def test_abi_rejects_bad_arguments_and_leaves_the_canvas(eng):
    from videollm_online_b200._lib import VloFramePlanes
    W, H = 64, 48
    frames = {fmt: yuv_noise(W, H, fmt, 1) for fmt in FORMATS}
    frames["rgb"] = np.zeros((H, W, 3), dtype=np.uint8)
    out = torch.full((2, 3, R, R), 0xAB, dtype=torch.uint8, device="cuda")

    def call(fmt, mutate=None, n=1, h=eng._h, o=out, second=False):
        descs, keep = (VloFramePlanes * 2)(), []
        for d in descs:
            _contig_desc(eng, d, fmt, frames[fmt], keep)
        if mutate:
            mutate(descs[1 if second else 0])
        rc = eng.lib.vlo_letterbox_planes(h, descs, n, None if o is None else C.c_void_p(o.data_ptr()), _stream())
        torch.cuda.synchronize()
        return rc

    def setp(q, v):
        return lambda d: d.d_planes.__setitem__(q, v)

    def pitch(q, v):
        return lambda d: d.pitch.__setitem__(q, v)

    for fmt in list(FORMATS) + ["rgb"]:
        assert call(fmt) == 0 and call(fmt, n=2) == 0
    out.fill_(0xAB)
    torch.cuda.synchronize()
    bad = [
        ("nv12", dict(h=None)), ("nv12", dict(n=0)), ("nv12", dict(n=MAX_BATCH + 1)), ("nv12", dict(o=None)),
        ("nv12", dict(mutate=setp(0, None))), ("nv12", dict(mutate=setp(1, None))),
        ("yuv420p", dict(mutate=setp(1, None))), ("yuv420p", dict(mutate=setp(2, None))),
        ("yuyv422", dict(mutate=setp(0, None))), ("rgb", dict(mutate=setp(0, None))),
        ("nv12", dict(mutate=pitch(0, W - 1))), ("nv12", dict(mutate=pitch(1, W - 1))),
        ("yuv420p", dict(mutate=pitch(0, W - 1))), ("yuv420p", dict(mutate=pitch(1, W // 2 - 1))),
        ("yuv420p", dict(mutate=pitch(2, W // 2 - 1))), ("yuyv422", dict(mutate=pitch(0, 2 * W - 1))),
        ("rgb", dict(mutate=pitch(0, 3 * W - 1))), ("nv12", dict(mutate=pitch(0, -1))),
        ("nv12", dict(mutate=lambda d: setattr(d, "width", W - 1))),
        ("yuv420p", dict(mutate=lambda d: setattr(d, "height", H - 1))),
        ("nv12", dict(mutate=lambda d: setattr(d, "height", H - 1))),
        ("yuyv422", dict(mutate=lambda d: setattr(d, "width", W - 1))),
        ("nv12", dict(mutate=lambda d: setattr(d, "width", 0))), ("yuyv422", dict(mutate=lambda d: setattr(d, "height", 1))),
        ("yuv420p", dict(mutate=lambda d: setattr(d, "width", 8194))), ("nv12", dict(mutate=lambda d: setattr(d, "height", 8194))),
        ("rgb", dict(mutate=lambda d: setattr(d, "width", 8193))),
        ("nv12", dict(mutate=lambda d: setattr(d, "format", 5))), ("nv12", dict(mutate=lambda d: setattr(d, "format", -1))),
        ("nv12", dict(mutate=lambda d: setattr(d, "d_taps", d.d_taps + 4))),
        ("yuyv422", dict(mutate=lambda d: setattr(d, "d_taps", None))),
        ("nv12", dict(mutate=lambda d: setattr(d, "x_taps", -1))), ("yuv420p", dict(mutate=lambda d: setattr(d, "y_taps", -1))),
        # the second frame of a batch is refused before the first is launched
        ("nv12", dict(n=2, second=True, mutate=setp(1, None))), ("yuyv422", dict(n=2, second=True, mutate=pitch(0, 5))),
        ("yuv420p", dict(n=2, second=True, mutate=lambda d: setattr(d, "format", 9))),
    ]
    for k, (fmt, kw) in enumerate(bad):
        rc = call(fmt, **kw)
        msg = eng.lib.vlo_last_error()
        assert rc != 0 and msg, f"case {k} ({fmt}) was accepted"
        assert bool((out == 0xAB).all()), f"case {k} ({fmt}): {msg.decode()} but the canvas changed"


def test_engine_rejects_bad_frames_before_device_work(eng):
    from videollm_online_b200._lib import VloError
    W, H = 64, 48
    f = torch.from_numpy(yuv_noise(W, H, "nv12", 0))
    bad = [([f], dict(pixel_format="nv12", bgr=True)), ([f], dict(pixel_format="nv21")),
           ([f[:-1]], dict(pixel_format="nv12")), ([f[:, :-1]], dict(pixel_format="nv12")),
           ([(f[:H].cuda(), f[H:].cuda()[:, :-2])], dict(pixel_format="nv12")),
           ([(f[:H].cuda(), f[H:])], dict(pixel_format="nv12")),
           ([(f[:H].cuda().t(), f[H:].cuda())], dict(pixel_format="nv12")),
           ([f.cuda(), f.float()], dict(pixel_format="nv12"))]
    for frames, kw in bad:
        with pytest.raises(VloError):
            eng.letterbox(frames, **kw)


# ================================================================================================ C. sessions
FPS = 2
LIVE_FRAMES = 32
AHEAD = 3
SPEAK = {7, 20}
CAM = (320, 240)


def _tiny_live(**kw):
    import ordering_child as OC
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = OC.tiny_state()
    return build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                      max_streams=2, max_step_tokens=128, max_vit_batch=8, **kw)


@pytest.fixture(scope="module")
def tiny_live():
    return _tiny_live(max_kv_tokens=2048)


def _camera(fmt, n, seed=0, size=CAM):
    return [yuv_noise(size[0], size[1], fmt, 1000 * seed + k) for k in range(n)]


def _push_form(frames, fmt, form):
    """(frames to push, push_frames kwargs): cvtColor's RGB, the raw frames on the CPU or device, or device planes"""
    if form == "rgb":
        return [torch.from_numpy(cv2.cvtColor(f, cv2_code(fmt))) for f in frames], {}
    if form == "cpu":
        return [torch.from_numpy(f) for f in frames], dict(pixel_format=fmt)
    if form == "cuda":
        return [torch.from_numpy(f).cuda() for f in frames], dict(pixel_format=fmt)
    return [_planes_420(f, fmt, 5) for f in frames], dict(pixel_format=fmt)


def _script(cfg, speak, resp_len=3):
    I, END, EOS = cfg.frame_token_interval_id, cfg.stream_end_id, cfg.eos_token_id
    raw, state = [], {"k": 0}

    def hook(dec, n, responding):
        raw.append(tuple(getattr(dec, f) for f in type(dec).__slots__))
        if responding:
            t = 300 + state["k"] if state["k"] < resp_len else EOS
            state["k"] = 0 if t == EOS else state["k"] + 1
        else:
            t = END if n in speak else I
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == I else 0.0
        if t != I:
            dec.argmax_excl_id = t
        return dec
    return hook, raw


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).cpu(), eng.kv_read(sid, l, True).cpu()) for l in range(eng.cfg.num_hidden_layers)]


def live_run(model, tok, fmt, form):
    from videollm_online_b200.config import SYSTEM_PROMPT, LiveArguments
    from videollm_online_b200.inference import LiveInfer
    cfg, eng = model.config, model.engine
    li = LiveInfer(LiveArguments(frame_fps=FPS, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    hook, raw = _script(cfg, SPEAK)
    state = {"resp": False}
    respond = li._call_for_response

    def call_for_response(*a):
        state["resp"] = True
        try:
            return respond(*a)
        finally:
            state["resp"] = False
    li._call_for_response = call_for_response
    li.decision_hook = lambda dec, n: hook(dec, n, state["resp"])
    frames, kw = _push_form(_camera(fmt, LIVE_FRAMES), fmt, form)
    pushed = 0

    def feed(upto):   # batches of 1 .. 3 frames
        nonlocal pushed
        while pushed < min(upto, LIVE_FRAMES):
            n = min(1 + pushed % 3, min(upto, LIVE_FRAMES) - pushed)
            li.push_frames(frames[pushed:pushed + n], **kw)
            pushed += n
    li.input_query_stream("Please narrate the video in real time.", video_time=0.0)
    feed(AHEAD + 1)
    conv = []
    for i in range(LIVE_FRAMES):
        li.input_video_stream(i / FPS)
        feed(i + 1 + AHEAD)
        conv.append(li())
    torch.cuda.synchronize()
    out = dict(conv=conv, decisions=raw, kv=_kv_all(eng, li._kv.stream_id))
    assert not li.video_tensor._pushes, "every pushed frame was encoded"
    eng.stream_close(li._kv.stream_id)
    return out


def _same(got, want):
    return {"conv": got["conv"] == want["conv"], "decisions": got["decisions"] == want["decisions"],
            "kv": all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) for a, b in zip(got["kv"], want["kv"]))}


@pytest.mark.parametrize("fmt,form", [("nv12", "cpu"), ("yuv420p", "cpu"), ("yuyv422", "cpu"), ("nv12", "planes"),
                                      ("yuv420p", "cuda")])
def test_live_push_yuv_equals_push_of_cvtcolor_rgb(tiny_live, fmt, form):
    want = live_run(*tiny_live, fmt, "rgb")
    assert len([r for _, r in want["conv"] if r]) >= 2
    got = live_run(*tiny_live, fmt, form)
    same = _same(got, want)
    assert all(same.values()), f"{fmt} {form} differs from cvtColor's RGB: {[k for k, v in same.items() if not v]}"


SCHED_TICKS = 30
SESSIONS = [("nv12", "cpu", (320, 240)), ("yuv420p", "cuda", (200, 300)), ("yuyv422", "cpu", (96, 96)),
            ("nv12", "planes", (320, 240))]


def sched_run(rgb: bool):
    from videollm_online_b200.config import SYSTEM_PROMPT
    from videollm_online_b200.multistream import StreamScheduler
    model, tok = _tiny_live(max_kv_tokens=1024, kv_pool_tokens=1400)
    cfg = model.config
    sched = StreamScheduler(model, tok, len(SESSIONS), frame_fps=FPS, system_prompt=SYSTEM_PROMPT)
    I, E, END = cfg.frame_token_interval_id, cfg.eos_token_id, cfg.stream_end_id
    scripts = [{6 + i: END, 7 + i: 300 + i, 8 + i: 301, 22 + i: END, 23 + i: 302} for i in range(len(SESSIONS))]
    raw = [[] for _ in SESSIONS]

    def hook(i, dec, n):
        raw[i].append(tuple(getattr(dec, f) for f in type(dec).__slots__))
        s = sched.sessions[i]
        t = scripts[i].get(n, E if s.state == s.RESPOND else I)
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == I else 0.0
        if t != I:
            dec.argmax_excl_id = t
        return dec
    sched.decision_hook = hook
    n_frames = SCHED_TICKS * 2
    cams = [_push_form(_camera(fmt, n_frames, seed=7 * i, size=size), fmt, "rgb" if rgb else form)
            for i, (fmt, form, size) in enumerate(SESSIONS)]
    pushed, fed = [0] * len(SESSIONS), [-1] * len(SESSIONS)
    for tick in range(SCHED_TICKS):
        for i, s in enumerate(sched.sessions):
            step = (0, 1, 2, 1)[(tick + i) % 4] if (tick * 7 + i) % 5 else 0
            if step:
                fed[i] = min(fed[i] + step, n_frames - 1)
                if pushed[i] <= fed[i]:
                    upto = min(fed[i] + 4, n_frames)
                    s.push_frames(cams[i][0][pushed[i]:upto], **cams[i][1])
                    pushed[i] = upto
                s.input_video_stream(fed[i] / FPS)
        sched.tick()
    sched.run_until_idle()
    eng = model.engine
    kv = []
    for s in sched.sessions:
        if s.resident:
            kv.append(("resident", _kv_all(eng, s.stream_id)))
        else:
            kv.append(("image", None if s.image is None else s.image.synchronize().data.clone()))
    out = dict(sessions=[(s.events, s.outputs, s.n_calls) for s in sched.sessions], decisions=raw, kv=kv,
               swaps=(sched.swaps_out, sched.swaps_in))
    eng.close()
    return out


def _same_kv_entry(a, b):
    if a[0] != b[0]:
        return False
    if a[0] == "resident":
        return all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a[1], b[1]))
    return (a[1] is None and b[1] is None) or (a[1] is not None and b[1] is not None and torch.equal(a[1], b[1]))


def test_scheduler_push_yuv_equals_push_of_cvtcolor_rgb():
    want = sched_run(rgb=True)
    assert want["swaps"][0] > 0 and want["swaps"][1] > 0
    assert all(any(e[0] == "response" for e in ev) for ev, *_ in want["sessions"])
    got = sched_run(rgb=False)
    same = {"sessions": got["sessions"] == want["sessions"], "decisions": got["decisions"] == want["decisions"],
            "swaps": got["swaps"] == want["swaps"],
            "kv": len(got["kv"]) == len(want["kv"]) and all(_same_kv_entry(a, b) for a, b in zip(got["kv"], want["kv"]))}
    assert all(same.values()), f"YUV pushes differ from cvtColor's RGB: {[k for k, v in same.items() if not v]}"
