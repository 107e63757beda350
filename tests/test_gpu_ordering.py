"""Results must not depend on timing or on what device memory held before.

A. Every kernel path the engine launches with programmatic dependent launch (PDL) gives the bits it gives with PDL off
   (VLO_NO_PDL=1, read once per process, so the PDL-off run is a child process: tests/ordering_child.py).
B. Encode-ahead (the next frame's ViT on a side CUDA stream while the decoder step runs) gives the bits of the same work
   on one stream, in LiveInfer, in StreamScheduler and at the engine level.  Each overlapped run is repeated with a
   spin kernel (torch.cuda._sleep) enqueued first on the side stream, then on the main stream, before the work whose
   order a wait enforces, so that either stream's work lands late: a missing wait then reads unwritten embeddings or
   races on the ViT workspaces.  Each case runs once.
C. The vision tower chained from the kernel-level entries over buffers filled with NaN and then with a finite pattern,
   each input at the start of a larger poisoned allocation: no stage reads memory it did not write."""
import collections
import os
import pathlib
import subprocess
import sys

import pytest
import torch

import ordering_child as OC
import test_gpu_vit_kernels as VK
from test_gpu_vit_kernels import lib, tower  # noqa: F401  module fixtures

pytestmark = pytest.mark.gpu

HERE = pathlib.Path(__file__).resolve().parent
# torch.cuda._sleep spins this many SM clock cycles.  Measured once with CUDA events on an H100 80GB HBM3 at a 700 W power
# limit: 1.01 ms, against 0.15 ms for a tiny-config frame step (T = 11 at a 1500-token cache) and 0.16-0.21 ms for a
# tiny-config ViT pass of 1 to 8 frames.  So the delayed stream's work starts after the other stream's is done.
SLEEP = 2_000_000


def _same_bits(a, b):
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _same_list(a, b):
    return len(a) == len(b) and all(_same_bits(x, y) for x, y in zip(a, b))


def _dec_row(dec):
    """every field of a Decision, as read back from the device"""
    return tuple(getattr(dec, f) for f in type(dec).__slots__)


def _same_kv(a, b):
    return len(a) == len(b) and all(_same_bits(x[0], y[0]) and _same_bits(x[1], y[1]) for x, y in zip(a, b))


# ================================================================================================= A. PDL on vs off
@pytest.fixture(scope="module")
def pdl_runs(tmp_path_factory):
    if os.environ.get("VLO_NO_PDL") == "1":
        pytest.skip("PDL is off in this process: there is nothing to compare")
    path = tmp_path_factory.mktemp("pdl_off") / "out.pt"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [str(HERE / "ordering_child.py"), str(path)]
    r = subprocess.run(cmd, env=dict(os.environ, VLO_NO_PDL="1"), capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, f"the PDL-off child failed:\n{r.stdout[-2000:]}\n{r.stderr[-6000:]}"
    return OC.scenarios(), torch.load(path)


@pytest.mark.parametrize("group", OC.GROUPS)
def test_pdl_on_equals_pdl_off(pdl_runs, group):
    """logits, decision rows, sampled ids and every layer's K/V of the step scenarios; fp32 tokens and bf16 embeds of
    vit_encode at every tiling; the connector"""
    on, off = pdl_runs
    keys = sorted(k for k in on if k.split("/")[0] == group)
    assert keys and keys == sorted(k for k in off if k.split("/")[0] == group)
    bad = [k for k in keys if not _same_bits(on[k], off[k])]
    assert not bad, f"{len(bad)} of {len(keys)} outputs differ with PDL off: {bad[:12]}"


# ============================================================================== B. encode-ahead vs serial execution
class _Delays:
    """Wraps model.visual_embed and engine.step, and marks the ViT passes made inside `ahead_owner.ahead_name` as
    encode-ahead passes.  where == "side": a spin kernel before every encode-ahead pass; "main": before every in-line
    pass and every step.  Enqueues nothing that makes the host wait: it copies every step's input rows and id rows on
    the step's stream, and brackets every ViT pass with timing events on the pass's stream."""

    def __init__(self, model, where, ahead_owner, ahead_name):
        self.model, self.where, self.steps, self.passes = model, where, [], []
        self.ahead = False
        eng = model.engine
        vit, step, launch = model.visual_embed, eng.step, getattr(ahead_owner, ahead_name)

        def visual_embed(frames):
            if self.where == ("side" if self.ahead else "main"):
                torch.cuda._sleep(SLEEP)
            ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev[0].record()
            out = vit(frames)
            ev[1].record()
            self.passes.append((self.ahead, *ev))
            return out

        def step_(sids, q_lens, embeds, *a, **kw):
            if self.where == "main":
                torch.cuda._sleep(SLEEP)
            ids = kw.get("row_ids")
            self.steps.append((embeds.clone(), None if ids is None else ids.clone()))
            return step(sids, q_lens, embeds, *a, **kw)

        def ahead(*a, **kw):
            self.ahead = True
            try:
                return launch(*a, **kw)
            finally:
                self.ahead = False
        model.visual_embed, eng.step = visual_embed, step_
        setattr(ahead_owner, ahead_name, ahead)
        self.owner, self.name = ahead_owner, ahead_name

    def close(self):
        del self.model.visual_embed, self.model.engine.step
        delattr(self.owner, self.name)

    def embeds(self):
        """the embedding rows every step read (rows with an id >= 0 are gathered on the device and not read)"""
        torch.cuda.synchronize()
        return [e if ids is None else e[ids < 0] for e, ids in self.steps]

    def order(self):
        """(pairs, late): every encode-ahead pass must start after each in-line pass enqueued before it has ended (they
        share the engine's ViT workspaces), and every in-line pass after each encode-ahead pass enqueued before it.
        pairs counts the encode-ahead passes enqueued right after an in-line pass: only the side stream's wait orders
        those two.  late lists (earlier pass, later pass, ms) for a pass that started before the other ended."""
        torch.cuda.synchronize()
        late = []
        for j, (a_j, s_j, _) in enumerate(self.passes):
            for i, (a_i, _, e_i) in enumerate(self.passes[:j]):
                if a_i != a_j and e_i.elapsed_time(s_j) < -0.01:   # 10 us: far below a missed wait's spin
                    late.append((i, j, round(e_i.elapsed_time(s_j), 3)))
        pairs = sum(1 for p, q in zip(self.passes, self.passes[1:]) if q[0] and not p[0])
        return pairs, late


class _Recorded(collections.deque):
    """LiveInfer.frame_embeds_queue that keeps a copy of every frame embedding queued"""

    def __init__(self):
        super().__init__()
        self.log = []

    def extend(self, items):
        items = list(items)
        self.log.extend(e.clone() for _, e in items)
        super().extend(items)


def _script(cfg, speak, resp_len=3):
    """a decision hook: frames speak at the calls in `speak`, a response is resp_len ids then EOS; it records every
    decision as the device wrote it"""
    I, END, EOS = cfg.frame_token_interval_id, cfg.stream_end_id, cfg.eos_token_id
    raw = []

    def hook(dec, n, responding):
        raw.append(_dec_row(dec))
        if responding:
            k = hook.k
            t = 300 + k if k < resp_len else EOS
            hook.k = 0 if t == EOS else k + 1
        else:
            t = END if n in speak else I
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == I else 0.0
        if t != I:
            dec.argmax_excl_id = t
        return dec
    hook.k = 0
    return hook, raw


LIVE_FRAMES = 48
LIVE_WINDOW = 512
LIVE_SPEAK = {9, 26, 40}


@pytest.fixture(scope="module")
def live(tiny):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = tiny
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=2, max_kv_tokens=2048, max_step_tokens=128, max_vit_batch=8)
    return model, tok


def _live_run(live, *, prefetch, depth=1, window=None, delay=None, one_stream=False):
    """cli.main over a seeded clip: the conversation, every decision row, the final cache, every queued frame
    embedding, every step's embedding rows and the evicted count.  one_stream: encode-ahead runs on the main stream
    (the same launches in the same order, without overlap)."""
    from videollm_online_b200 import cli
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    model, tok = live
    cfg, eng = model.config, model.engine
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT, context_window=window or 0), model=model,
                   tokenizer=tok)
    li.prefetch_next, li.prefetch_depth = prefetch, depth
    if one_stream:
        li._side = torch.cuda.current_stream(model.device)
    li.frame_embeds_queue = _Recorded()
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
    d = _Delays(model, delay, li, "_enqueue_step")
    try:
        _, history = cli.main(li, video=cli.synthetic_clip(LIVE_FRAMES, cfg.frame_resolution, seed=21),
                              n_iters=LIVE_FRAMES, quiet=True)
    finally:
        d.close()
    conv = [(c["role"], c["content"]) for c in history["conversation"] if "role" in c]
    out = dict(conv=conv, decisions=raw, kv=_kv_all(eng, li._kv.stream_id), queued=li.frame_embeds_queue.log,
               embeds=d.embeds(), evicted=li.evicted_tokens)
    out["passes"] = [a for a, *_ in d.passes]
    out["order"] = d.order()
    eng.stream_close(li._kv.stream_id)
    return out


def _same_live(got, want):
    return {k: (_same_kv(got[k], want[k]) if k == "kv" else _same_list(got[k], want[k]) if k in ("queued", "embeds")
                else got[k] == want[k]) for k in want if k not in ("passes", "order")}


@pytest.fixture(scope="module")
def live_serial(live):
    runs = {}

    def get(depth, window):
        if (depth, window) not in runs:
            runs[(depth, window)] = _live_run(live, prefetch=True, depth=depth, window=window, one_stream=True)
        return runs[(depth, window)]
    return get


@pytest.mark.parametrize("window", [None, LIVE_WINDOW])
def test_live_prefetch_equals_no_prefetch(live, window):
    """prefetch_next True (the next frame encoded on the side stream) and False (every frame encoded in line): the same
    conversation, decision rows, cache, queued frame embeddings and step inputs"""
    want = _live_run(live, prefetch=False, window=window)
    got = _live_run(live, prefetch=True, window=window)
    assert len(want["conv"]) >= 5 and (window is None or want["evicted"] > 0)
    assert True not in want["passes"] and got["passes"].count(True) >= LIVE_FRAMES // 2
    assert not got["order"][1], f"ViT passes started before the pass they must follow ended: {got['order'][1][:8]}"
    same = _same_live(got, want)
    assert all(same.values()), f"differs from the run without encode-ahead: {[k for k, v in same.items() if not v]}"


@pytest.mark.parametrize("delay", [None, "side", "main"])
@pytest.mark.parametrize("window", [None, LIVE_WINDOW])
@pytest.mark.parametrize("depth", [1, 2, 3])
def test_live_encode_ahead_equals_one_stream(live, live_serial, depth, window, delay):
    """prefetch_depth 1, 2 and 3 (3 frames per pass: the trunk tiling), with and without a context window (evictions
    land between a prefetch and its use), with either stream held back: the bits of the same launches on one stream"""
    want = live_serial(depth, window)
    assert len(want["conv"]) >= 5 and (window is None or want["evicted"] > 0)
    got = _live_run(live, prefetch=True, depth=depth, window=window, delay=delay)
    assert got["passes"] == want["passes"] and got["passes"].count(True) >= LIVE_FRAMES // (2 * depth)
    assert got["order"][0] >= 1
    assert not got["order"][1], f"ViT passes started before the pass they must follow ended: {got['order'][1][:8]}"
    same = _same_live(got, want)
    assert all(same.values()), f"differs from one stream: {[k for k, v in same.items() if not v]}"


# ---------------------------------------------------------------------------------------------- StreamScheduler
SCHED_SESSIONS = 4
SCHED_TICKS = 36
SCHED_WINDOW = 512


def _sched_run(tiny, *, ahead=True, delay=None, one_stream=False, vit_batch=8):
    """4 sessions on 2 stream slots and a pool that holds about two of them (swaps), session 0 windowed.  Frames arrive
    in bursts, so a tick has 0 to 4 pending frames: some are encoded ahead, some in line.  vit_batch=1: every ViT pass
    encodes one frame, whichever path batches it."""
    from videollm_online_b200.cli import synthetic_clip
    from videollm_online_b200.config import SYSTEM_PROMPT
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200.multistream import StreamScheduler
    cfg, llm, vis = tiny
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=2, max_kv_tokens=1024, max_step_tokens=128, max_vit_batch=vit_batch,
                            kv_pool_tokens=1400)
    sched = StreamScheduler(model, tok, SCHED_SESSIONS, frame_fps=2, system_prompt=SYSTEM_PROMPT)
    sched.encode_ahead = ahead
    if one_stream:
        sched._side = torch.cuda.current_stream(model.device)
    I, E, END = cfg.frame_token_interval_id, cfg.eos_token_id, cfg.stream_end_id
    scripts = [{6 + i: END, 7 + i: 300 + i, 8 + i: 301, 25 + i: END, 26 + i: 302} for i in range(SCHED_SESSIONS)]
    raw = [[] for _ in range(SCHED_SESSIONS)]

    def hook(i, dec, n):
        raw[i].append(_dec_row(dec))
        s = sched.sessions[i]
        t = scripts[i].get(n, E if s.state == s.RESPOND else I)
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == I else 0.0
        if t != I:
            dec.argmax_excl_id = t
        return dec
    sched.decision_hook = hook
    n_frames = SCHED_TICKS * 2
    for i, s in enumerate(sched.sessions):
        s.load_video(synthetic_clip(n_frames, cfg.frame_resolution, seed=30 + i))
    sched.sessions[0].context_window = SCHED_WINDOW
    d = _Delays(model, delay, sched, "_launch_encode_ahead")
    fed = [-1] * SCHED_SESSIONS
    try:
        for tick in range(SCHED_TICKS):
            for i, s in enumerate(sched.sessions):
                step = (0, 1, 2, 1)[(tick + i) % 4] if (tick * 7 + i) % 5 else 0
                if step:
                    fed[i] = min(fed[i] + step, n_frames - 1)
                    s.input_video_stream(fed[i] / 2)
            sched.tick()
        sched.run_until_idle()
    finally:
        d.close()
    eng = model.engine
    kv = []
    for s in sched.sessions:
        if s.resident:
            kv.append(("resident", _kv_all(eng, s.stream_id)))
        else:
            kv.append(("image", None if s.image is None else s.image.synchronize().data.clone()))
    out = dict(sessions=[(s.events, s.outputs, s.evicted_tokens, s.n_calls) for s in sched.sessions], decisions=raw,
               kv=kv, embeds=d.embeds(), swaps=(sched.swaps_out, sched.swaps_in))
    out["passes"] = [a for a, *_ in d.passes]
    out["order"] = d.order()
    eng.close()
    return out


def _same_sched(got, want):
    def kv_same(a, b):
        return all(x[0] == y[0] and (_same_kv(x[1], y[1]) if x[0] == "resident" else
                                     (x[1] is None and y[1] is None) or (x[1] is not None and y[1] is not None
                                                                         and torch.equal(x[1], y[1])))
                   for x, y in zip(a, b)) and len(a) == len(b)
    return {k: kv_same(got[k], want[k]) if k == "kv" else _same_list(got[k], want[k]) if k == "embeds"
            else got[k] == want[k] for k in want if k not in ("passes", "order")}


@pytest.fixture(scope="module")
def sched_serial(tiny):
    return _sched_run(tiny, one_stream=True)


def _exercised(run):
    """the run encoded frames ahead, and enqueued an encode-ahead pass right after an in-line pass"""
    return run["passes"].count(True) >= 5 and run["passes"].count(False) >= 5 and run["order"][0] >= 2


def test_scheduler_serial_run_exercises_the_paths(sched_serial):
    """the reference run swaps, evicts, responds and encodes frames both ahead and in line"""
    s = sched_serial
    assert _exercised(s), (s["passes"].count(True), s["passes"].count(False), s["order"][0])
    assert s["swaps"][0] > 0 and s["swaps"][1] > 0
    assert s["sessions"][0][2] > 0
    assert all(any(e[0] == "response" for e in ev) for ev, *_ in s["sessions"])


@pytest.mark.parametrize("delay", [None, "side", "main"])
def test_scheduler_encode_ahead_equals_one_stream(tiny, sched_serial, delay):
    got = _sched_run(tiny, delay=delay)
    assert _exercised(got) and got["passes"] == sched_serial["passes"]
    assert not got["order"][1], f"ViT passes started before the pass they must follow ended: {got['order'][1][:8]}"
    same = _same_sched(got, sched_serial)
    assert all(same.values()), f"differs from one stream: {[k for k, v in same.items() if not v]}"


@pytest.mark.parametrize("delay", [None, "side", "main"])
def test_scheduler_encode_ahead_equals_in_line(tiny, delay):
    """encode_ahead True and False, every ViT pass one frame (max_vit_batch 1): the same bits"""
    want = _sched_run(tiny, ahead=False, vit_batch=1)
    got = _sched_run(tiny, delay=delay, vit_batch=1)
    assert True not in want["passes"] and _exercised(got)
    assert not got["order"][1], f"ViT passes started before the pass they must follow ended: {got['order'][1][:8]}"
    same = _same_sched(got, want)
    assert all(same.values()), f"differs from encode_ahead False: {[k for k, v in same.items() if not v]}"


# ---------------------------------------------------------------------------------------------- engine level
@pytest.mark.parametrize("delay", [None, "side", "main"])
@pytest.mark.parametrize("B", [1, 2, 3, 8])
def test_engine_vit_on_a_side_stream_equals_serial(live, B, delay):
    """Engine.vit_encode of the next B frames on a side stream while Engine.step consumes the current ones on the main
    stream: the side stream waits for an event recorded before the step (the previous pass's workspaces are free), the
    main stream waits for the pass's event before it uses the embeddings.  Steps and embeddings equal a serial run."""
    from videollm_online_b200.cli import synthetic_clip
    model, _ = live
    eng, cfg = model.engine, model.config
    rounds = 4
    frames = synthetic_clip((rounds + 1) * B, cfg.frame_resolution, seed=50 + B).cuda()
    main, side = torch.cuda.current_stream(), torch.cuda.Stream()

    def run(overlap):
        sid = eng.stream_open()
        outs, embeds = [], []
        if overlap and delay == "main":   # the main stream's pass and steps land late: the side pass must wait for them
            torch.cuda._sleep(SLEEP)
        e = eng.vit_encode(frames[:B])
        for r in range(rounds):
            embeds.append(e.clone())
            if overlap and delay == "main":
                torch.cuda._sleep(SLEEP)
            pre = torch.cuda.Event()
            pre.record(main)
            logits, dec = eng.step([sid], [e.shape[0]], e)
            outs += [logits.clone(), dec.clone()]
            nxt = frames[(r + 1) * B:(r + 2) * B]
            if overlap:
                side.wait_event(pre)
                with torch.cuda.stream(side):
                    if delay == "side":
                        torch.cuda._sleep(SLEEP)
                    n = eng.vit_encode(nxt)
                    ev = torch.cuda.Event()
                    ev.record(side)
                main.wait_event(ev)
                n.record_stream(main)
                e = n
            else:
                e = eng.vit_encode(nxt)
        embeds.append(e.clone())
        kv = _kv_all(eng, sid)
        eng.stream_close(sid)
        return outs, embeds, kv

    want = run(False)
    got = run(True)
    assert _same_list(got[1], want[1]), "embeddings differ"
    assert _same_list(got[0], want[0]), "step outputs differ"
    assert _same_kv(got[2], want[2]), "cache differs"


# ================================================================ C. the tower replay over poisoned buffers
class _PoisonedTorch:
    """`torch` for the tower replay of test_gpu_vit_kernels: torch.empty returns the head of a larger allocation that
    is filled with a sentinel (NaN, or a finite pattern) past the returned view as well"""

    def __init__(self, nan):
        self.nan, self.bufs = nan, []

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *shape, dtype=torch.float32, device=None):
        n = 1
        for s in shape:
            n *= s
        base = torch.empty(n + max(n // 2, 1 << 20), dtype=dtype, device=device)
        if self.nan:
            base.fill_(float("nan"))
        else:   # finite, varied, and far from what the tower writes
            base.copy_((torch.arange(base.numel(), device=device) % 23 - 11).to(dtype) * 37)
        t = base[:n].view(*shape)
        self.bufs.append(t)
        return t


def _digest(t):
    """a bitwise digest of a tensor (two different tensors of a replay colliding is not a concern)"""
    w = t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).flatten().long()
    k = torch.arange(w.numel(), device=w.device) % 65521 + 1
    return int((w * k).sum()), int(w.sum())


def _poisoned_replay(monkeypatch, lib, eng, cfg, frames, t, nan):  # noqa: F811
    fake = _PoisonedTorch(nan)
    stages = []
    check = VK._check

    def staged(rc, what):
        check(rc, what)
        torch.cuda.synchronize()
        stages.append((what, [(_digest(b), bool(b.isnan().any())) for b in fake.bufs]))
    monkeypatch.setattr(VK, "torch", fake)
    monkeypatch.setattr(VK, "_check", staged)
    try:
        S = frames.shape[-1]
        padded = torch.full((frames.numel() + (1 << 20),), 0xA5 if nan else 0x5A, dtype=torch.uint8, device="cuda")
        f = padded[:frames.numel()].view(frames.shape)
        f.copy_(frames)
        tokens = VK._replay(lib, eng, cfg, f, t)
    finally:
        monkeypatch.undo()
    assert frames.shape[-1] == S
    return tokens, stages


@pytest.mark.parametrize("B", VK.TOWER_BATCHES)
def test_tower_replay_reads_only_what_it_wrote(monkeypatch, lib, tower, B):  # noqa: F811
    """Every buffer of the replay starts as NaN in one run and as a finite pattern in the other, each with a poisoned
    tail.  After every stage, each buffer the NaN run has fully written must hold the same bits in both runs (the first
    one that does not names the stage that read unwritten memory); the tokens equal vit_encode's."""
    cfg, eng = tower
    frames = VK._frames(B, cfg.frame_resolution, B)
    t = VK._tiling(lib, B, cfg)
    tok = eng.vit_encode(frames, return_vit_tokens=True)[1].clone()
    a, sa = _poisoned_replay(monkeypatch, lib, eng, cfg, frames, t, nan=True)
    b, sb = _poisoned_replay(monkeypatch, lib, eng, cfg, frames, t, nan=False)
    assert [w for w, _ in sa] == [w for w, _ in sb]
    for k, ((what, da), (_, db)) in enumerate(zip(sa, sb)):
        for j, ((ha, has_nan), (hb, _)) in enumerate(zip(da, db)):
            assert has_nan or ha == hb, f"B={B}: stage {k} ({what}) leaves buffer {j} different under the two fills"
    assert not a.isnan().any(), "the replay left a token slot unwritten"
    assert VK._same_bits(a, b), f"B={B}: the tokens depend on the sentinel"
    assert VK._same_bits(a, tok), f"B={B}: the replay over poisoned buffers differs from vit_encode"
