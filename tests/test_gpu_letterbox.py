"""Live frames at their native size: vlo_letterbox against the numpy restatement of its integer INTER_CUBIC
(tests/letterbox_reference.py) bit for bit, its argument checks, and sessions fed through push_frames against the same
sessions fed the reference's canvases through load_video.

  A. The kernel: single frames of many sizes (down- and upscaled, odd, prime, 8192 on one side), RGB and BGR, CPU and
     device input; batches of 1 .. max_vit_batch mixed sizes in one launch, each frame equal to its own launch; the
     output buffer filled with 0xAB first, so a byte the kernel does not write shows.
  B. LiveInfer: the conversation, every decision row and the final KV cache of a push_frames session equal those of the
     load_video session at prefetch_depth 1 and 3, with a query mid-stream, on a backlog (segmented steps) and under a
     context window.  Frames are pushed while the session runs, far enough ahead that encode-ahead sees them where it
     sees the loaded clip's.
  C. StreamScheduler: 4 sessions with cameras of 3 sizes on 2 stream slots (swaps) against the same sessions fed the
     reference canvases.
  D. Ordering: the LiveInfer case with a 1 ms spin kernel ahead of every push on the side stream, so a missing wait reads
     unwritten canvases, and in a child process with VLO_NO_PDL=1 (this file run as a script)."""
import ctypes as C
import os
import pathlib
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = pathlib.Path(__file__).resolve().parent
if __name__ == "__main__":   # the PDL-off child: python tests/test_gpu_letterbox.py OUT.pt
    sys.path.insert(0, str(HERE.parent))
    import vlo_bootstrap  # noqa: F401

from letterbox_reference import letterbox_reference

pytestmark = pytest.mark.gpu

R = 384
# torch.cuda._sleep cycles: about 1 ms on an H100 (tests/test_gpu_ordering.py measures it)
SLEEP = 2_000_000
SIZES = [(1920, 1080), (1280, 720), (640, 480), (1080, 1920), (192, 144), (385, 383), (4000, 10), (10, 4000),
         (3840, 2160), (383, 385), (97, 61), (101, 103), (7, 5), (1, 1), (2, 3), (200, 150), (384, 384), (8192, 33),
         (33, 8192)]


def _noise(W, H, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, (H, W, 3), dtype=np.uint8))


def _ref(frame, res, bgr=False):
    return torch.from_numpy(letterbox_reference(frame.cpu().numpy(), res, bgr=bgr))


# ======================================================================================================= A. kernel
@pytest.fixture(scope="module")
def eng():
    from videollm_online_b200 import tiny_config
    from videollm_online_b200.engine import Engine
    e = Engine(tiny_config(frame_resolution=R), "cuda:0", max_vit_batch=8)
    yield e
    e.close()


def _descs(eng, frames, bgr):
    """(descriptor array, tensors to keep alive) of device frames"""
    from videollm_online_b200._lib import VloLetterboxFrame
    d = (VloLetterboxFrame * len(frames))()
    keep = []
    for x, f in zip(d, frames):
        H, W = f.shape[:2]
        taps, sw = eng._letterbox_taps(W, H)
        keep += [f, taps]
        x.d_pixels, x.d_taps, x.width, x.height, x.bgr, x.x_taps, x.y_taps = f.data_ptr(), taps.data_ptr(), W, H, int(bgr), 0, sw
    return d, keep


def _launch(eng, frames, bgr=False, fill=0xAB):
    """raw vlo_letterbox into a buffer filled with `fill`"""
    from videollm_online_b200._lib import check
    dev = [f.cuda().contiguous() for f in frames]
    out = torch.full((len(frames), 3, R, R), fill, dtype=torch.uint8, device="cuda")
    d, keep = _descs(eng, dev, bgr)
    check(eng.lib.vlo_letterbox(eng._h, d, len(frames), C.c_void_p(out.data_ptr()),
                                C.c_void_p(torch.cuda.current_stream().cuda_stream)), "vlo_letterbox")
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("bgr", [False, True])
@pytest.mark.parametrize("W,H", SIZES)
def test_kernel_equals_reference(eng, W, H, bgr):
    f = _noise(W, H, W * 31 + H)
    want = _ref(f, R, bgr)
    assert torch.equal(_launch(eng, [f], bgr)[0], want)
    assert torch.equal(_launch(eng, [f], bgr, fill=0x00)[0], want)
    # the public entry, from host and from device memory
    assert torch.equal(eng.letterbox([f], bgr=bgr).cpu(), want[None])
    assert torch.equal(eng.letterbox([f.cuda()], bgr=bgr).cpu(), want[None])


def test_canvas_size_is_copied(eng):
    f = _noise(R, R, 5)
    assert torch.equal(eng.letterbox([f]).cpu()[0], f.permute(2, 0, 1))


@pytest.mark.parametrize("B", list(range(1, 9)))
def test_mixed_batch_equals_solo_launches(eng, B):
    """B frames of different sizes in one launch: each frame equals its own launch and the reference"""
    sizes = [SIZES[(B * 5 + k * 3) % len(SIZES)] for k in range(B)]
    frames = [_noise(W, H, 100 * B + k) for k, (W, H) in enumerate(sizes)]
    bgr = B % 2 == 0
    got = _launch(eng, frames, bgr)
    for k, f in enumerate(frames):
        assert torch.equal(got[k], _launch(eng, [f], bgr)[0]), f"frame {k} {sizes[k]}"
        assert torch.equal(got[k], _ref(f, R, bgr)), f"frame {k} {sizes[k]}"


def test_more_frames_than_max_vit_batch_are_split(eng):
    frames = [_noise(64 + k, 48 + 2 * k, k) for k in range(11)]
    got = eng.letterbox(frames).cpu()
    assert all(torch.equal(got[k], _ref(f, R)) for k, f in enumerate(frames))


def test_abi_rejects_bad_arguments(eng):
    from videollm_online_b200._lib import VloError, check
    f = _noise(64, 48, 0).cuda()
    out = torch.empty(8, 3, R, R, dtype=torch.uint8, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(mutate=None, n=1, h=eng._h, o=out):
        d, keep = _descs(eng, [f] * max(n, 1), False)
        if mutate:
            mutate(d[0])
        check(eng.lib.vlo_letterbox(h, d, n, None if o is None else C.c_void_p(o.data_ptr()), st), "vlo_letterbox")

    call()
    bad = {
        "null engine": dict(h=None), "no frames": dict(n=0), "above max_vit_batch": dict(n=9), "null output": dict(o=None),
        "null pixels": dict(mutate=lambda d: setattr(d, "d_pixels", None)),
        "null taps": dict(mutate=lambda d: setattr(d, "d_taps", None)),
        "width 0": dict(mutate=lambda d: setattr(d, "width", 0)),
        "height 0": dict(mutate=lambda d: setattr(d, "height", 0)),
        "width 8193": dict(mutate=lambda d: setattr(d, "width", 8193)),
        "height 8193": dict(mutate=lambda d: setattr(d, "height", 8193)),
        "bgr 2": dict(mutate=lambda d: setattr(d, "bgr", 2)),
        "misaligned taps": dict(mutate=lambda d: setattr(d, "d_taps", d.d_taps + 4)),
        "negative offset": dict(mutate=lambda d: setattr(d, "y_taps", -1)),
    }
    for what, kw in bad.items():
        with pytest.raises(VloError):
            call(**kw)
        assert what
    for frame in (torch.zeros(48, 64, 4, dtype=torch.uint8), torch.zeros(48, 64, 3), torch.zeros(48, 64 * 3, dtype=torch.uint8),
                  torch.zeros(48, 8193, 3, dtype=torch.uint8), torch.zeros(0, 64, 3, dtype=torch.uint8)):
        with pytest.raises(VloError):
            eng.letterbox([frame])
    torch.cuda.synchronize()


# ================================================================================================== B. LiveInfer
FPS = 2
LIVE_FRAMES = 48
LIVE_WINDOW = 512
LIVE_SPEAK = {9, 26}
AHEAD = 4   # frames pushed ahead of the one being stepped: encode-ahead then sees every frame it would see in a loaded clip


def _tiny():
    import ordering_child as OC
    return OC.tiny_state()


@pytest.fixture(scope="module")
def tiny_live():
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = _tiny()
    return build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                      max_streams=2, max_kv_tokens=2048, max_step_tokens=128, max_vit_batch=8)


def _camera(n, res_seed=0):
    """native frames of one camera: 320 x 240 (downscaled to 96 x 72 in a tiny canvas)"""
    return [_noise(320, 240, 1000 * res_seed + k) for k in range(n)]


def _script(cfg, speak, resp_len=3):
    """decision hook: frames speak at the calls in `speak`, a response is resp_len ids then EOS; records every row"""
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


def live_run(model, tok, case, push, spin=False, cuda=False):
    """One session over LIVE_FRAMES native frames: pushed (push=True) or loaded as the reference's canvases.  Returns the
    conversation, every decision row, the final cache and the evicted count.  spin: a 1 ms spin kernel on the side stream
    ahead of every push's copy and letterbox.  cuda: every pushed frame is written on the main stream behind a 1 ms spin,
    dropped as soon as it is pushed, and its memory taken by a new allocation filled on the main stream."""
    from videollm_online_b200.config import SYSTEM_PROMPT, LiveArguments
    from videollm_online_b200.inference import LiveInfer
    cfg, eng = model.config, model.engine
    li = LiveInfer(LiveArguments(frame_fps=FPS, system_prompt=SYSTEM_PROMPT,
                                 context_window=LIVE_WINDOW if "window" in case else 0), model=model, tokenizer=tok)
    li.prefetch_depth = 3 if "depth3" in case else 1
    hook, raw = _script(cfg, LIVE_SPEAK)
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
    frames = _camera(LIVE_FRAMES)
    letterbox = eng.letterbox
    if spin:   # every push's copy and letterbox land late on the side stream
        def slow(*a, **kw):
            torch.cuda._sleep(SLEEP)
            return letterbox(*a, **kw)
        eng.letterbox = slow
    pushed = 0

    on_device = [f.cuda() for f in frames] if cuda else None
    torch.cuda.synchronize()
    junk = []

    def feed(upto):   # push frames [pushed, upto) in batches of 1 .. 3
        nonlocal pushed
        while push and pushed < min(upto, LIVE_FRAMES):
            n = min(1 + pushed % 3, min(upto, LIVE_FRAMES) - pushed)
            if cuda:
                torch.cuda._sleep(SLEEP)   # the frames are written late on the main stream
                batch = [f.clone() for f in on_device[pushed:pushed + n]]
                li.push_frames(batch)
                del batch   # dropped at once: a new allocation on the main stream may take their memory
                junk.extend(torch.full_like(f, 0x5A) for f in on_device[pushed:pushed + n])
            else:
                li.push_frames(frames[pushed:pushed + n])
            pushed += n
    if not push:
        li.load_video(torch.stack([_ref(f, cfg.frame_resolution) for f in frames]))
    li.input_query_stream("Please narrate the video in real time.", video_time=0.0)
    conv = []
    try:
        if "backlog" in case:   # bursts of 8 frames queued at once, the next burst pushed before this one drains
            feed(16)
            for end in range(8, LIVE_FRAMES + 1, 8):
                li.input_video_stream((end - 1) / FPS)
                feed(end + 8)
                while li.frame_embeds_queue:
                    conv.append(li())
        else:
            feed(AHEAD + 1)
            for i in range(LIVE_FRAMES):
                if "query" in case and i == 17:
                    li.input_query_stream("What is on the table?", video_time=i / FPS + 0.25)
                li.input_video_stream(i / FPS)
                feed(i + 1 + AHEAD)
                conv.append(li())
    finally:
        eng.letterbox = letterbox
    torch.cuda.synchronize()
    out = dict(conv=conv, decisions=raw, kv=_kv_all(eng, li._kv.stream_id), evicted=li.evicted_tokens)
    if push:
        assert li.video_tensor.size(0) == LIVE_FRAMES and not li.video_tensor._pushes, "every pushed frame was encoded"
    eng.stream_close(li._kv.stream_id)
    return out


def _same(got, want):
    return {"conv": got["conv"] == want["conv"], "decisions": got["decisions"] == want["decisions"],
            "evicted": got["evicted"] == want["evicted"],
            "kv": all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) for a, b in zip(got["kv"], want["kv"]))}


CASES = ["depth1", "depth3", "query", "backlog", "window", "backlog-window"]


@pytest.fixture(scope="module")
def loaded_runs(tiny_live):
    runs = {}

    def get(case):
        if case not in runs:
            runs[case] = live_run(*tiny_live, case, push=False)
        return runs[case]
    return get


@pytest.mark.parametrize("case", CASES)
def test_live_push_equals_load_video(tiny_live, loaded_runs, case):
    want = loaded_runs(case)
    responses = [r for _, r in want["conv"] if r]
    assert len(responses) >= 2 and ("window" not in case or want["evicted"] > 0)
    got = live_run(*tiny_live, case, push=True)
    same = _same(got, want)
    assert all(same.values()), f"push_frames differs from load_video: {[k for k, v in same.items() if not v]}"


def test_live_push_with_the_side_stream_held_back(tiny_live, loaded_runs):
    got = live_run(*tiny_live, "depth1", push=True, spin=True)
    same = _same(got, loaded_runs("depth1"))
    assert all(same.values()), f"a late push changes the bits: {[k for k, v in same.items() if not v]}"


def test_live_push_of_cuda_frames_written_late_on_the_main_stream(tiny_live, loaded_runs):
    """frames produced on the caller's stream: the side stream reads them only once they are written, and their memory
    is not handed to a new allocation before that read"""
    got = live_run(*tiny_live, "depth1", push=True, spin=True, cuda=True)
    same = _same(got, loaded_runs("depth1"))
    assert all(same.values()), f"CUDA frames change the bits: {[k for k, v in same.items() if not v]}"


def test_a_frame_not_pushed_yet_is_refused_and_changes_nothing(tiny_live):
    """input_video_stream past the frames pushed raises before any state changes (LiveInfer and StreamSession), and a
    slice of the ring never returns fewer frames than asked for"""
    from videollm_online_b200.config import SYSTEM_PROMPT, LiveArguments
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.multistream import StreamScheduler
    model, tok = tiny_live
    silent, _ = _script(model.config, set())   # random weights: every frame stays silent
    li = LiveInfer(LiveArguments(frame_fps=FPS, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    li.decision_hook = lambda dec, n: silent(dec, n, False)
    li.push_frames(_camera(2))
    li.input_video_stream(0.0)
    li()
    state = (li.last_frame_idx, li.video_time, len(li.frame_embeds_queue), sorted(li._prefetched))
    with pytest.raises(IndexError):
        li.input_video_stream(2 / FPS)
    assert (li.last_frame_idx, li.video_time, len(li.frame_embeds_queue), sorted(li._prefetched)) == state
    with pytest.raises(IndexError):
        li.video_tensor[1:4]
    li.push_frames(_camera(1))
    li.input_video_stream(2 / FPS)   # the same call succeeds once the frame is there
    li()
    assert li.last_frame_idx == 2 and not li.video_tensor._pushes
    torch.cuda.synchronize()
    model.engine.stream_close(li._kv.stream_id)

    sched = StreamScheduler(model, tok, 1, frame_fps=FPS, system_prompt=SYSTEM_PROMPT)
    sched.decision_hook = lambda i, dec, n: silent(dec, n, False)
    s = sched.sessions[0]
    s.push_frames(_camera(1))
    with pytest.raises(IndexError):
        s.input_video_stream(1 / FPS)
    assert s.last_frame_idx == -1 and not s.pending_frames
    s.input_video_stream(0.0)
    sched.run_until_idle()
    assert s.n_calls >= 1
    torch.cuda.synchronize()
    model.engine.stream_close(s.stream_id)


def test_live_push_with_pdl_off(tiny_live, loaded_runs, tmp_path):
    if os.environ.get("VLO_NO_PDL") == "1":
        pytest.skip("PDL is off in this process: there is nothing to compare")
    path = tmp_path / "out.pt"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [str(HERE / "test_gpu_letterbox.py"), str(path)]
    r = subprocess.run(cmd, env=dict(os.environ, VLO_NO_PDL="1"), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, f"the PDL-off child failed:\n{r.stdout[-2000:]}\n{r.stderr[-6000:]}"
    got = torch.load(path, weights_only=False)
    same = _same(got, loaded_runs("depth1"))
    assert all(same.values()), f"PDL off changes the bits: {[k for k, v in same.items() if not v]}"


def test_push_after_load_video_is_refused_and_reset_drops_pushed_frames(tiny_live):
    from videollm_online_b200.config import SYSTEM_PROMPT, LiveArguments
    from videollm_online_b200.inference import LiveInfer
    model, tok = tiny_live
    li = LiveInfer(LiveArguments(frame_fps=FPS, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    li.load_video(torch.zeros(4, 3, 96, 96, dtype=torch.uint8))
    with pytest.raises(ValueError):
        li.push_frames(_camera(1))
    li.reset()
    li.push_frames(_camera(3))
    assert li.num_video_frames == 3
    li.reset()
    assert li.video_tensor is None
    li.push_frames(_camera(2))
    assert li.video_tensor.size(0) == 2
    torch.cuda.synchronize()
    model.engine.stream_close(li._kv.stream_id)


# ============================================================================================= C. StreamScheduler
SCHED_TICKS = 36
CAMERAS = [(320, 240), (200, 300), (96, 96), (320, 240)]   # 3 sizes: landscape, portrait, the canvas itself


def sched_run(push):
    from videollm_online_b200.config import SYSTEM_PROMPT
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200.multistream import StreamScheduler
    cfg, llm, vis = _tiny()
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=2, max_kv_tokens=1024, max_step_tokens=128, max_vit_batch=8,
                            kv_pool_tokens=1400)
    sched = StreamScheduler(model, tok, len(CAMERAS), frame_fps=FPS, system_prompt=SYSTEM_PROMPT)
    I, E, END = cfg.frame_token_interval_id, cfg.eos_token_id, cfg.stream_end_id
    scripts = [{6 + i: END, 7 + i: 300 + i, 8 + i: 301, 25 + i: END, 26 + i: 302} for i in range(len(CAMERAS))]
    raw = [[] for _ in CAMERAS]

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
    cams = [[_noise(W, H, 77 * i + k) for k in range(n_frames)] for i, (W, H) in enumerate(CAMERAS)]
    pushed = [0] * len(CAMERAS)
    if not push:
        for s, frames in zip(sched.sessions, cams):
            s.load_video(torch.stack([_ref(f, cfg.frame_resolution) for f in frames]))
    fed = [-1] * len(CAMERAS)
    for tick in range(SCHED_TICKS):
        for i, s in enumerate(sched.sessions):
            step = (0, 1, 2, 1)[(tick + i) % 4] if (tick * 7 + i) % 5 else 0
            if step:
                fed[i] = min(fed[i] + step, n_frames - 1)
                if push and pushed[i] <= fed[i]:   # the camera delivers up to 3 frames past the one due
                    upto = min(fed[i] + 4, n_frames)
                    s.push_frames(cams[i][pushed[i]:upto])
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


def test_scheduler_push_equals_load_video():
    want = sched_run(push=False)
    assert want["swaps"][0] > 0 and want["swaps"][1] > 0
    assert all(any(e[0] == "response" for e in ev) for ev, *_ in want["sessions"])
    got = sched_run(push=True)
    same = {"sessions": got["sessions"] == want["sessions"], "decisions": got["decisions"] == want["decisions"],
            "swaps": got["swaps"] == want["swaps"],
            "kv": len(got["kv"]) == len(want["kv"]) and all(_same_kv_entry(a, b) for a, b in zip(got["kv"], want["kv"]))}
    assert all(same.values()), f"push_frames differs from load_video: {[k for k, v in same.items() if not v]}"


if __name__ == "__main__":
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = _tiny()
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=2, max_kv_tokens=2048, max_step_tokens=128, max_vit_batch=8)
    torch.save(live_run(model, tok, "depth1", push=True), sys.argv[1])
