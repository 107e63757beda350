"""Context windows over the KV cache (`vlo_kv_evict`, `Engine.kv_make_room`, `LiveInfer.context_window`,
`StreamSession.context_window`): the re-rotation kernel against an fp32 emulation (bit for bit) and fp64 geometry, the
pool accounting and failures that change nothing, exact continuation after an eviction, and sessions that run past
their cache capacity with the same bits on every path (backlog, drafts, sampling, suspend / resume, scheduler)."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

PAGE = 64


def _engine(cfg, llm, max_streams, max_kv_tokens, kv_pool_tokens=None):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=kv_pool_tokens)
    return model.engine


def _emb(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _same_kv(a, b):
    return len(a) == len(b) and all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))


def _free(eng):
    return eng.kv_pool_info()["free_pages"]


def _emulate(k, cos, sin):
    """the kernel's rotation in torch fp32: separate multiplies and adds, each rounded once, then bf16"""
    x1, x2 = k[..., :64].float(), k[..., 64:].float()
    c, s = cos.cuda(), sin.cuda()
    return torch.cat([(x1 * c + x2 * s).bfloat16(), (x2 * c - x1 * s).bfloat16()], -1)


def _rotate64(k, delta, cfg):
    """k rotated by -delta positions, exactly (fp64)"""
    from videollm_online_b200 import weights as W
    ang = W.rope_inv_freq(cfg).double().cuda() * delta
    c, s = ang.cos(), ang.sin()
    x1, x2 = k[..., :64].double(), k[..., 64:].double()
    return torch.cat([x1 * c + x2 * s, x2 * c - x1 * s], -1)


def _write_random(eng, sid, n, seed):
    g = torch.Generator().manual_seed(seed)
    c = eng.cfg
    for l in range(c.num_hidden_layers):
        for is_v in (False, True):
            eng.kv_write(sid, l, is_v, torch.randn(c.num_key_value_heads, n, c.head_dim, generator=g).bfloat16())


# ------------------------------------------------------------------------------------------------ kernel and ABI
CASES = {"sink_page_kept": (64, 320), "no_sink": (0, 128), "one_page": (128, 64), "many_pages": (64, 512),
         "up_to_the_last_full_page": (64, 576), "everything_full": (0, 640)}


@pytest.mark.parametrize("case", list(CASES))
def test_evict_rotates_kept_keys_and_leaves_the_rest(tiny, case):
    from videollm_online_b200 import weights as W
    cfg, llm, _ = tiny
    first, n = CASES[case]
    eng = _engine(cfg, llm, 3, 2048)
    a, sentinel = eng.stream_open(), eng.stream_open()
    L = 700                                  # not a multiple of 64: 10 full pages and a partial one
    _write_random(eng, sentinel, 333, seed=1)
    _write_random(eng, a, L, seed=2)
    before, sent = _kv_all(eng, a), _kv_all(eng, sentinel)
    free0 = _free(eng)
    eng.kv_evict(a, first, n)
    after = _kv_all(eng, a)
    assert eng.kv_len(a) == L - n and _free(eng) == free0 + n // PAGE
    assert _same_kv(_kv_all(eng, sentinel), sent)
    cos, sin = W.rope_rotation(cfg, n)
    u = 2.0 ** -8                            # bf16 unit roundoff
    for (k0, v0), (k1, v1) in zip(before, after):
        assert torch.equal(k1[:, :first], k0[:, :first]) and torch.equal(v1[:, :first], v0[:, :first])   # sink
        assert torch.equal(v1[:, first:], v0[:, first + n:])                                               # V moves only
        kept = k0[:, first + n:]
        assert torch.equal(k1[:, first:], _emulate(kept, cos, sin))                                        # bit for bit
        exact = _rotate64(kept, n, cfg)
        pair = (kept[..., :64].double().abs() + kept[..., 64:].double().abs()).repeat(1, 1, 2)
        # one bf16 rounding of a value within a few fp32 roundings of the exact one
        assert ((k1[:, first:].double() - exact).abs() <= u * exact.abs() + 2.0 ** -20 * pair).all()


def test_invalid_evictions_change_nothing(tiny):
    from videollm_online_b200 import weights as W
    from videollm_online_b200._lib import check, VloError
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 3, 2048)
    a, b, closed = eng.stream_open(), eng.stream_open(), eng.stream_open()
    eng.stream_close(closed)
    _write_random(eng, a, 700, seed=3)
    _write_random(eng, b, 100, seed=4)
    cos, sin = W.rope_rotation(cfg, 64)
    fp = C.POINTER(C.c_float)
    pc, ps = C.cast(cos.data_ptr(), fp), C.cast(sin.data_ptr(), fp)

    def snap():
        return _free(eng), eng.kv_len(a), eng.kv_len(b), _kv_all(eng, a), _kv_all(eng, b)
    s0 = snap()
    bad = [(a, 32, 64, pc, ps, "multiples"), (a, 64, 96, pc, ps, "multiples"), (a, 64, 640, pc, ps, "full"),
           (a, 0, 704, pc, ps, "full"), (a, 64, 0, pc, ps, "multiples"), (a, 64, -64, pc, ps, "multiples"),
           (a, -64, 64, pc, ps, "multiples"), (a, 64, 64, None, ps, "null"), (a, 64, 64, pc, None, "null"),
           (closed, 0, 64, pc, ps, "invalid stream"), (b, 64, 64, pc, ps, "full")]
    for sid, first, n, c_, s_, msg in bad:
        with pytest.raises(VloError, match=msg):
            check(eng.lib.vlo_kv_evict(eng._h, sid, first, n, c_, s_, eng._stream()), "vlo_kv_evict")
        s1 = snap()
        assert s1[:3] == s0[:3] and _same_kv(s1[3], s0[3]) and _same_kv(s1[4], s0[4]), (first, n)


# ------------------------------------------------------------------------------------------------ geometry
def _rope_bound(kb):
    """|k_A - k_B| bound for one key, per element, from the rounding points (u = 2^-8, the bf16 unit roundoff):
    the append kernel at a position rounds cos / sin to bf16 (u each), both products (u) and the sum (u): each output
    is within 3u (|x1| + |x2|) (1 + u)^2 of the exact rotation of the same x, for B at p and for A at p + delta.  The
    re-rotation is a rotation, so A's error pair stays within sqrt(2) times its per-element bound, and adds a few fp32
    roundings (< 2^-20 (|x1| + |x2|)) and one bf16 rounding (u (|x1| + |x2|) (1 + 4u)).  The difference is then within
    (3 (1 + sqrt 2) + 1) u (1 + u)^4 (|x1| + |x2|) + 2^-20 (|x1| + |x2|), with |x1| + |x2| <= sqrt(2) |(x1, x2)| and
    |(x1, x2)| <= |B's pair| / (1 - 7u) (B's pair is within sqrt(2) 3u (1 + u)^2 (|x1| + |x2|) of the rotated x)."""
    u = 2.0 ** -8
    pair = (kb[..., :64].double() ** 2 + kb[..., 64:].double() ** 2).sqrt() / (1 - 7 * u)
    m = math.sqrt(2.0) * pair
    b = ((3 * (1 + math.sqrt(2.0)) + 1) * u * (1 + u) ** 4 + 2.0 ** -20) * m
    return b.repeat(1, 1, 2)


def test_evicted_keys_land_where_a_fresh_stream_puts_them(tiny):
    """Stream A gets X (3 pages) then Y; stream B gets Y alone, in a step of the same shape.  After evicting X from A
    (first = 0), A's layer-0 keys of Y match B's within the bound derived from the rounding points, and the wrong
    sign or delta +- 1 violate it; V is equal bit for bit."""
    from videollm_online_b200 import weights as W
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 3, 2048)
    a, b = eng.stream_open(), eng.stream_open()
    delta, ny = 3 * PAGE, 100
    for i in range(3):
        eng.step([a], [PAGE], _emb(cfg, PAGE, 10 + i))
    y = _emb(cfg, ny, 99)
    eng.step([a], [ny], y)
    eng.step([b], [ny], y)
    ka0 = eng.kv_read(a, 0, False)[:, delta:].clone()
    eng.kv_evict(a, 0, delta)
    ka, kb = eng.kv_read(a, 0, False), eng.kv_read(b, 0, False)
    assert torch.equal(eng.kv_read(a, 0, True), eng.kv_read(b, 0, True))
    bound = _rope_bound(kb)
    assert ((ka.double() - kb.double()).abs() <= bound).all()
    cos, sin = W.rope_rotation(cfg, delta)
    assert torch.equal(ka, _emulate(ka0, cos, sin))
    for name, (c, s) in {"wrong sign": (cos, -sin), "delta - 1": W.rope_rotation(cfg, delta - 1),
                         "delta + 1": W.rope_rotation(cfg, delta + 1)}.items():
        wrong = _emulate(ka0, c, s)
        assert ((wrong.double() - kb.double()).abs() > bound).any(), name


# ------------------------------------------------------------------------------------------------ continuation
def test_continuation_after_an_eviction_is_exact(tiny):
    """A grows interleaved with another stream (its pages are not in order), loses pages from the middle, then steps;
    a fresh stream holding a copy of A's cache steps with the same input: same logits, decisions and cache."""
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 4, 2048)
    a, other, c = eng.stream_open(), eng.stream_open(), eng.stream_open()
    for i in range(8):
        eng.step([a], [90], _emb(cfg, 90, 20 + i))
        eng.step([other], [30], _emb(cfg, 30, 40 + i))
    eng.kv_evict(a, 128, 320)
    n = eng.kv_len(a)
    for l in range(cfg.num_hidden_layers):
        for is_v in (False, True):
            eng.kv_write(c, l, is_v, eng.kv_read(a, l, is_v))
    assert eng.kv_len(c) == n
    out = []
    for sid in (a, c):
        frame = _emb(cfg, 11, 7)
        logits, dec = eng.step([sid], [11], frame)
        out.append((logits.clone(), dec.clone(), eng.last_step_logits(11).clone()))
    assert all(torch.equal(x, y) for x, y in zip(*out))
    assert _same_kv(_kv_all(eng, a), _kv_all(eng, c))


# ------------------------------------------------------------------------------------------------ sessions
N_FRAMES = 200
WINDOW = 1024
SPEAK_CALLS = {30, 95, 150, 240}
QUERIES = [(0.0, "narrate"), (20.25, "between frames"), (50.0, "at frame 100"), (80.0, "at frame 160")]


def _model(tiny, max_kv_tokens=1536, max_streams=3, kv_pool_tokens=None):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, _ = tiny
    return build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                      max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=kv_pool_tokens)


def _session(model, tok, cfg, window=WINDOW, sampling=None, drafts=True, resp_len=2):
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT, context_window=window or 0), model=model,
                   tokenizer=tok)
    li.sampling = sampling
    if not drafts:
        li.drafter = None
    iid, end_id, eos = cfg.frame_token_interval_id, cfg.stream_end_id, cfg.eos_token_id
    state = {"resp": False}
    respond = li._call_for_response

    def call_for_response(*a):
        state["resp"] = True
        try:
            return respond(*a)
        finally:
            state["resp"] = False
    li._call_for_response = call_for_response

    def hook(dec, n):   # greedy: a response is resp_len scripted ids and EOS; frames speak at the scripted calls
        if state["resp"]:
            k = state.setdefault("k", 0)
            t = 300 + k % 5 if k < resp_len else eos
            state["k"] = 0 if t == eos else k + 1
            if dec.sampled_id is not None:
                dec.sampled_id = eos if t == eos else dec.sampled_id
        else:
            t = end_id if n in SPEAK_CALLS else iid
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == iid else 0.0
        if t != iid:
            dec.argmax_excl_id = t
        return dec
    li.decision_hook = hook
    return li


def _frames(cfg, n=N_FRAMES):
    g = torch.Generator().manual_seed(77)
    return [(i / 2, torch.randn(cfg.frame_num_tokens, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda())
            for i in range(n)]


def _run(model, tok, cfg, *, backlog=False, suspend_after=None, tmp_path=None, **kw):
    """Feed the frames one per call (or all at once: the backlog drain), answer the queries; returns the trace
    (query, response, last id, kv_len), the call count, the final cache, the evicted count and the largest kv_len."""
    eng = model.engine
    li = _session(model, tok, cfg, **kw)
    li.query_queue.extend(QUERIES)
    frames = _frames(cfg)
    trace, calls, peak = [], 0, 0
    if backlog:
        li.frame_embeds_queue.extend(frames)
    fed = 0
    while fed < len(frames) or li.frame_embeds_queue:
        if not backlog and not li.frame_embeds_queue:
            li.frame_embeds_queue.append(frames[fed])
            fed += 1
        elif backlog:
            fed = len(frames)
        query, response = li()
        calls += 1
        peak = max(peak, eng.kv_len(li._kv.stream_id))
        if query or response:
            trace.append((query, response, int(li.last_ids.reshape(-1)[-1]), eng.kv_len(li._kv.stream_id)))
        if calls == suspend_after:
            state = li.suspend()
            torch.save(state, tmp_path / "session.pt")
            del state
            sampling = li.sampling
            eng.stream_close(li._kv.stream_id)
            li = _session(model, tok, cfg, **kw)
            li.resume(torch.load(tmp_path / "session.pt"))
            assert li.sampling == sampling
    out = trace, li._n_calls, _kv_all(eng, li._kv.stream_id), li.evicted_tokens, peak
    eng.stream_close(li._kv.stream_id)
    return out


def _same_run(x, y):
    return x[0] == y[0] and x[1] == y[1] and _same_kv(x[2], y[2]) and x[3] == y[3]


@pytest.fixture(scope="module")
def built(tiny):
    return _model(tiny)


def test_a_window_outlives_the_cache_capacity(built, tiny):
    from videollm_online_b200._lib import VloError
    cfg = tiny[0]
    model, tok = built
    with pytest.raises(VloError, match="capacity exceeded"):
        _run(model, tok, cfg, window=None)
    got = _run(model, tok, cfg)
    assert got[3] > 0 and got[4] <= WINDOW
    assert sum(t[0] is not None for t in got[0]) == len(QUERIES)


def _fresh(tiny):
    return _model(tiny)


def test_backlog_drain_equals_one_frame_per_step(tiny):
    cfg = tiny[0]
    model, tok = _fresh(tiny)
    one = _run(model, tok, cfg)
    drain = _run(model, tok, cfg, backlog=True)
    assert one[3] > 0
    assert _same_run(one, drain)


@pytest.mark.parametrize("sampled", [False, True])
def test_drafts_give_the_ids_of_one_token_per_step_across_evictions(tiny, sampled):
    from videollm_online_b200.config import SamplingConfig
    cfg = tiny[0]
    model, tok = _fresh(tiny)
    s = SamplingConfig(do_sample=True, temperature=0.8, top_k=20, top_p=0.9, seed=5) if sampled else None
    with_drafts = _run(model, tok, cfg, sampling=s, resp_len=40)
    without = _run(model, tok, cfg, sampling=s, resp_len=40, drafts=False)
    assert with_drafts[3] > 0 and with_drafts[4] <= WINDOW
    assert _same_run(with_drafts, without)


def test_suspend_resume_continues_exactly(tiny, tmp_path):
    from videollm_online_b200.config import SamplingConfig
    cfg = tiny[0]
    model, tok = _fresh(tiny)
    s = SamplingConfig(do_sample=True, temperature=0.8, seed=9)
    want = _run(model, tok, cfg, sampling=s, resp_len=30)
    assert want[3] > 0
    for k in (40, 90):
        got = _run(model, tok, cfg, sampling=s, resp_len=30, suspend_after=k, tmp_path=tmp_path)
        assert _same_run(got, want), k


def test_sampled_positions_never_repeat(tiny):
    from videollm_online_b200.config import SamplingConfig
    cfg = tiny[0]
    model, tok = _fresh(tiny)
    eng = model.engine
    seen = []
    sample = eng._sample

    def record(logits, rows):
        seen.extend(r.position for r in rows if r is not None)
        return sample(logits, rows)
    eng._sample = record
    got = _run(model, tok, cfg, sampling=SamplingConfig(do_sample=True, seed=3), resp_len=60, drafts=False)
    assert got[3] > 0 and len(seen) > 100
    assert len(set(seen)) == len(seen)
    assert max(seen) >= WINDOW      # positions count the evicted tokens


# ------------------------------------------------------------------------------------------------ StreamScheduler
SCHED_FRAMES = 70
SCHED_WINDOW = 512


def _sched_run(tiny, turns, n_sessions, max_streams, kv_pool_tokens):
    from videollm_online_b200.config import SYSTEM_PROMPT
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200.multistream import StreamScheduler
    from videollm_online_b200.cli import synthetic_clip
    cfg, llm, vis = tiny
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=max_streams, max_kv_tokens=1024, max_step_tokens=128, max_vit_batch=8,
                            kv_pool_tokens=kv_pool_tokens)
    I, E, END = cfg.frame_token_interval_id, cfg.eos_token_id, cfg.stream_end_id
    sched = StreamScheduler(model, tok, n_sessions, frame_fps=2, system_prompt=SYSTEM_PROMPT)
    scripts = [{10 + i: END, 11 + i: 300 + i, 12 + i: 301, 45 + i: END, 46 + i: 302} for i in range(n_sessions)]

    def hook(i, dec, n):
        s = sched.sessions[i]
        t = scripts[i].get(n, E if s.state == s.RESPOND else I)
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == I else 0.0
        if t != I:
            dec.argmax_excl_id = t
        return dec
    sched.decision_hook = hook
    for i, s in enumerate(sched.sessions):
        s.context_window = SCHED_WINDOW
        s.load_video(synthetic_clip(SCHED_FRAMES, cfg.frame_resolution, seed=i))
    fed, peak = [0] * n_sessions, 0
    for tick in range(max(max(w) for w in turns) + 1):
        for i, s in enumerate(sched.sessions):
            if tick in turns[i]:
                s.input_video_stream(fed[i] / 2)
                fed[i] += 1
        while sched.tick():
            peak = max([peak] + [s.kv_tokens() for s in sched.sessions])
    eng = model.engine
    kv = []
    for s in sched.sessions:
        kv.append(_kv_all(eng, s.stream_id) if s.resident else None)
    return [(s.events, s.outputs, s.evicted_tokens) for s in sched.sessions], kv, sched, peak, (model, tok, scripts)


def test_scheduler_windows_with_more_sessions_than_slots(tiny):
    """Four windowed sessions, one per turn, on an engine with 2 slots and a pool for two windows, against an engine
    that holds all four: the same events, outputs and evictions; no session ever exceeds its window.  Each session
    run alone through LiveInfer with the same window and script ends with the same cache as the scheduler's."""
    n = 4
    turns = [range(SCHED_FRAMES * i, SCHED_FRAMES * (i + 1)) for i in range(n)]
    want, want_kv, _, peak, (model, tok, scripts) = _sched_run(tiny, turns, n, n, None)
    assert peak <= SCHED_WINDOW and all(w[2] > 0 for w in want)
    got, _, sched, peak, _ = _sched_run(tiny, turns, n, 2, 2 * (SCHED_WINDOW + PAGE))
    assert sched.swaps_out > 0 and sched.swaps_in > 0 and peak <= SCHED_WINDOW
    assert got == want
    # the same sessions alone through LiveInfer (vision inside, one frame per call, no encode-ahead)
    from videollm_online_b200.cli import synthetic_clip
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    cfg = tiny[0]
    for i in range(n):
        model.engine.stream_close(i)   # the scheduler's slot i (its cache is in want_kv) is free for this run
        li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT, context_window=SCHED_WINDOW),
                       model=model, tokenizer=tok)
        li.prefetch_next = False
        state = {"resp": False}
        respond = li._call_for_response

        def call_for_response(*a, respond=respond, state=state):
            state["resp"] = True
            try:
                return respond(*a)
            finally:
                state["resp"] = False
        li._call_for_response = call_for_response

        def hook(dec, k, i=i, state=state):
            t = scripts[i].get(k, cfg.eos_token_id if state["resp"] else cfg.frame_token_interval_id)
            dec.argmax_id = dec.argmax_prob_id = t
            dec.p_interval = 1.0 if t == cfg.frame_token_interval_id else 0.0
            if t != cfg.frame_token_interval_id:
                dec.argmax_excl_id = t
            return dec
        li.decision_hook = hook
        li.load_video(synthetic_clip(SCHED_FRAMES, cfg.frame_resolution, seed=i))
        for f in range(SCHED_FRAMES):
            li.input_video_stream(f / 2)
            li()
        assert li.evicted_tokens == want[i][2], i
        assert _same_kv(_kv_all(model.engine, li._kv.stream_id), want_kv[i]), i
        model.engine.stream_close(li._kv.stream_id)
