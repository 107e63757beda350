"""A context window that keeps the conversation (`vlo_kv_compact`, `Engine.kv_compact`, `LiveInfer.context_keep_turns`,
`StreamSession.context_keep_turns`): the in-place compaction kernel against an fp32 emulation (bit for bit) and fp64,
independent of its batching, equal to vlo_kv_evict where both apply, on a full pool, failures that change nothing,
exact continuation, and sessions that keep every recent turn with the same bits on every path."""
import ctypes as C
import re

import pytest
import torch

from test_gpu_kv_evict import _emb, _emulate, _engine, _free, _kv_all, _rotate64, _same_kv, _write_random

pytestmark = pytest.mark.gpu

PAGE = 64
L = 700


def _scatter_streams(eng, cfg, a, other, n_a):
    """grow stream a interleaved with `other`, so a's pages are out of order, then give a random K / V"""
    for done in range(90, n_a + 90, 90):
        eng.kv_fill_synthetic(a, min(done, n_a), seed=done)
        eng.kv_fill_synthetic(other, done // 3, seed=done + 1)
    _write_random(eng, a, n_a, seed=2)


def _expected(cfg, before, spans):
    """per layer (K, V) of the compacted stream, emulated: K of span i rotated by its shift (untouched when 0)"""
    from videollm_online_b200 import weights as W
    out, q = [], 0
    parts = []
    for f, n in spans:
        parts.append((f, n, f - q))
        q += n
    for k0, v0 in before:
        ks, vs = [], []
        for f, n, d in parts:
            kept = k0[:, f:f + n]
            ks.append(kept if d == 0 else _emulate(kept, *W.rope_rotation(cfg, d)))
            vs.append(v0[:, f:f + n])
        out.append((torch.cat(ks, 1), torch.cat(vs, 1)))
    return out, parts


SPANS = {
    "unaligned_shifts_across_pages": [(0, 37), (100, 150), (300, 7), (400, 250)],
    "untouched_first_span_then_moves": [(0, 130), (131, 500), (640, 60)],
    "everything_moves": [(5, 600)],
    "dropped_tail_only": [(0, 500)],
    "many_small_spans": [(7 * i, 3) for i in range(100)],
}


@pytest.mark.parametrize("case", list(SPANS))
def test_compact_moves_and_rotates_like_the_emulation(tiny, case):
    cfg, llm, _ = tiny
    spans = SPANS[case]
    results = []
    for step_tokens in (128, 16):        # the step workspace stages 128 or 16 page-planes per batch
        from videollm_online_b200.modeling_live import build_live
        model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=3,
                              max_kv_tokens=2048, max_step_tokens=step_tokens, max_vit_batch=1)
        eng = model.engine
        a, sentinel, other = eng.stream_open(), eng.stream_open(), eng.stream_open()
        _scatter_streams(eng, cfg, a, other, L)
        _write_random(eng, sentinel, 333, seed=1)
        assert eng.kv_pool_info()["free_pages"] >= 0
        before, sent = _kv_all(eng, a), _kv_all(eng, sentinel)
        free0, bytes0 = _free(eng), eng.device_bytes()
        eng.kv_compact(a, spans)
        new_len = sum(n for _, n in spans)
        after = _kv_all(eng, a)
        assert eng.kv_len(a) == new_len
        assert _free(eng) == free0 + (-(-L // PAGE)) - (-(-new_len // PAGE))
        assert eng.device_bytes() == bytes0
        assert _same_kv(_kv_all(eng, sentinel), sent)
        want, parts = _expected(cfg, before, spans)
        u = 2.0 ** -8
        for (k1, v1), (kw, vw), (k0, _) in zip(after, want, before):
            assert torch.equal(v1, vw)                                          # V moves exactly
            assert torch.equal(k1, kw)                                          # K bit for bit, per span
            q = 0
            for f, n, d in parts:
                kept = k0[:, f:f + n]
                exact = _rotate64(kept, d, cfg)
                pair = (kept[..., :64].double().abs() + kept[..., 64:].double().abs()).repeat(1, 1, 2)
                assert ((k1[:, q:q + n].double() - exact).abs() <= u * exact.abs() + 2.0 ** -20 * pair).all()
                q += n
        results.append(after)
        del eng, model
    assert _same_kv(results[0], results[1])      # the bits do not depend on the batching


def test_one_aligned_span_equals_kv_evict(tiny):
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 4, 2048)
    a, b, other = eng.stream_open(), eng.stream_open(), eng.stream_open()
    _scatter_streams(eng, cfg, a, other, L)
    data = _kv_all(eng, a)
    for l, (k, v) in enumerate(data):
        eng.kv_write(b, l, False, k)
        eng.kv_write(b, l, True, v)
    f0 = _free(eng)
    eng.kv_evict(a, 64, 192)
    f1 = _free(eng)
    eng.kv_compact(b, [(0, 64), (256, L - 256)])
    assert f1 - f0 == _free(eng) - f1 == 3
    assert eng.kv_len(a) == eng.kv_len(b) == L - 192
    assert _same_kv(_kv_all(eng, a), _kv_all(eng, b))


def test_compact_on_a_full_pool(tiny):
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 2, 1024, kv_pool_tokens=16 * PAGE)
    a, b = eng.stream_open(), eng.stream_open()
    _scatter_streams(eng, cfg, a, b, L)                  # a: 11 pages, b: 4, then topped up to the last page
    eng.kv_fill_synthetic(b, 16 * PAGE - 11 * PAGE, seed=3)
    assert _free(eng) == 0
    spans = [(0, 40), (90, 300), (500, 150)]
    before, other = _kv_all(eng, a), _kv_all(eng, b)
    eng.kv_compact(a, spans)
    want, _ = _expected(cfg, before, spans)
    assert _same_kv(_kv_all(eng, a), want) and _same_kv(_kv_all(eng, b), other)
    assert _free(eng) == 11 - (-(-490 // PAGE))


def test_invalid_compactions_change_nothing(tiny):
    from videollm_online_b200._lib import VloError, check
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 3, 2048)
    a, b, closed = eng.stream_open(), eng.stream_open(), eng.stream_open()
    eng.stream_close(closed)
    _scatter_streams(eng, cfg, a, b, L)

    def snap():
        return _free(eng), eng.kv_len(a), eng.kv_len(b), _kv_all(eng, a), _kv_all(eng, b)
    s0 = snap()
    bad = [([(100, 50), (0, 50)], a, "sorted"), ([(0, 60), (50, 50)], a, "sorted"), ([(0, 10), (20, 0)], a, "empty"),
           ([(0, 10), (650, 60)], a, "past kv_len"), ([(0, L)], a, "nothing is dropped"),
           ([(0, 100), (100, L - 100)], a, "nothing is dropped"), ([(0, 10)], closed, "invalid stream"),
           ([(2 * i, 1) for i in range(20000)], a, "n_spans")]
    for spans, sid, msg in bad:
        with pytest.raises(VloError, match=msg):
            eng.kv_compact(sid, spans)
        s1 = snap()
        assert s1[:3] == s0[:3] and _same_kv(s1[3], s0[3]) and _same_kv(s1[4], s0[4]), msg
    i32, fp = C.POINTER(C.c_int32), C.POINTER(C.c_float)
    one = torch.tensor([0], dtype=torch.int32)
    rot = torch.zeros(128)
    p1, pr = C.cast(one.data_ptr(), i32), C.cast(rot.data_ptr(), fp)
    for args in [(None, p1, pr), (p1, None, pr), (p1, p1, None)]:
        with pytest.raises(VloError, match="null"):
            check(eng.lib.vlo_kv_compact(eng._h, a, 1, *args, eng._stream()), "vlo_kv_compact")
    with pytest.raises(VloError, match="n_spans"):
        check(eng.lib.vlo_kv_compact(eng._h, a, 0, p1, p1, pr, eng._stream()), "vlo_kv_compact")
    s1 = snap()
    assert s1[:3] == s0[:3] and _same_kv(s1[3], s0[3])


def test_continuation_after_a_compaction_is_exact(tiny):
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 4, 2048)
    a, other, c = eng.stream_open(), eng.stream_open(), eng.stream_open()
    for i in range(8):
        eng.step([a], [90], _emb(cfg, 90, 20 + i))
        eng.step([other], [30], _emb(cfg, 30, 40 + i))
    spans = [(0, 50), (77, 200), (333, 11), (400, 300)]
    want, _ = _expected(cfg, _kv_all(eng, a), spans)
    eng.kv_compact(a, spans)
    for l, (k, v) in enumerate(want):
        eng.kv_write(c, l, False, k)
        eng.kv_write(c, l, True, v)
    out = []
    for sid in (a, c):
        logits, dec = eng.step([sid], [11], _emb(cfg, 11, 7))
        out.append((logits.clone(), dec.clone(), eng.last_step_logits(11).clone()))
    assert all(torch.equal(x, y) for x, y in zip(*out))
    assert _same_kv(_kv_all(eng, a), _kv_all(eng, c))


# ------------------------------------------------------------------------------------------------ sessions
N_FRAMES = 200
WINDOW = 1024
SPEAK_CALLS = set(range(15, 600, 23))
QUERIES = [(0.0, "narrate"), (20.25, "between frames"), (50.0, "at frame 100"), (80.0, "at frame 160")]


def _model(tiny, max_kv_tokens=1536, max_streams=3):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, _ = tiny
    return build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                      max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1)


def _session(model, tok, cfg, sampling=None, drafts=True, resp_len=30):
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT, context_window=WINDOW,
                                 context_keep_turns=True), model=model, tokenizer=tok)
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

    def hook(dec, n):   # a response is resp_len scripted ids and EOS; frames speak at the scripted calls
        if state["resp"]:
            k = state.setdefault("k", 0)
            t = 300 + k % 5 if k < resp_len else eos
            state["k"] = 0 if t == eos else k + 1
            if dec.sampled_id is not None:
                t = eos if t == eos else (dec.sampled_id if dec.sampled_id not in (eos, end_id) else 301)
                dec.sampled_id = t
        else:
            t = end_id if n in SPEAK_CALLS else iid
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == iid else 0.0
        if t != iid:
            dec.argmax_excl_id = t
        return dec
    li.decision_hook = hook
    return li


def _history(li):
    return list(li._fed_ids())


def _run(model, tok, cfg, *, backlog=False, suspend_after=None, tmp_path=None, **kw):
    from test_gpu_kv_evict import _frames
    eng = model.engine
    li = _session(model, tok, cfg, **kw)
    li.query_queue.extend(QUERIES)
    frames = _frames(cfg, N_FRAMES)
    trace, calls, peak, said = [], 0, 0, []
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
            eng.stream_close(li._kv.stream_id)
            li = _session(model, tok, cfg, **kw)
            li.resume(torch.load(tmp_path / "session.pt"))
    hist = _history(li)
    assert len(hist) == eng.kv_len(li._kv.stream_id)
    out = trace, li._n_calls, _kv_all(eng, li._kv.stream_id), li.evicted_tokens, peak, hist
    eng.stream_close(li._kv.stream_id)
    return out


def _same_run(x, y):
    return x[0] == y[0] and x[1] == y[1] and _same_kv(x[2], y[2]) and x[3] == y[3] and x[5] == y[5]


def _check_template(tok, cfg, hist, prompt_len):
    """after the prompt: messages of frames (one interval row between two), separated by whole turns
    "]\\n[User: ...\\n]Assistant:...<eos>\\n["; the history ends in an open message"""
    runs, i = [], prompt_len
    while i < len(hist):
        j = i
        neg = hist[i] < 0
        while j < len(hist) and (hist[j] < 0) == neg:
            j += 1
        runs.append((neg, hist[i:j]))
        i = j
    assert runs[0][0]
    turns = []
    for k, (neg, r) in enumerate(runs):
        if neg:
            assert len(r) % cfg.frame_num_tokens == 0
        elif r != [cfg.frame_token_interval_id]:
            text = tok.decode(r, skip_special_tokens=False)
            end = r"<\|eos\|>\n\[" if k < len(runs) - 1 else ""    # a response that just ended is not closed yet
            assert re.fullmatch(r"\]\n(User: [^\n]*\n)?Assistant:.*" + end, text, re.S), text
            turns.append(text)
    # an interval row always sits between two frames of one message
    for k, (neg, r) in enumerate(runs):
        if not neg and r == [cfg.frame_token_interval_id]:
            assert runs[k - 1][0] and runs[k + 1][0]
    return turns


@pytest.fixture(scope="module")
def built(tiny):
    return _model(tiny)


def test_a_session_keeps_its_recent_turns_within_the_window(built, tiny):
    cfg = tiny[0]
    model, tok = built
    got = _run(model, tok, cfg)
    trace, _, _, evicted, peak, hist = got
    assert evicted > 0 and peak <= WINDOW
    prompt_len = len(tok.apply_chat_template([{"role": "system", "content": __import__(
        "videollm_online_b200.config", fromlist=["SYSTEM_PROMPT"]).SYSTEM_PROMPT}], add_stream_prompt=True))
    turns = _check_template(tok, cfg, hist, prompt_len)
    assert len(trace) > 8                     # more responses than the turn budget holds: old turns went
    # the latest turns are all still there, in order, with their queries
    kept = turns
    assert 0 < len(kept) < len(trace)
    tail = trace[-len(kept):]
    for (q, r, _, _), text in zip(tail, kept):
        if q is not None:
            assert q.split("User: ", 1)[1] in text
        assert r.split("Assistant:", 1)[1] in text


def test_backlog_drain_equals_one_frame_per_step(tiny):
    cfg = tiny[0]
    model, tok = _model(tiny)
    one = _run(model, tok, cfg)
    drain = _run(model, tok, cfg, backlog=True)
    assert one[3] > 0 and _same_run(one, drain)


@pytest.mark.parametrize("sampled", [False, True])
def test_drafts_give_the_same_session(tiny, sampled):
    from videollm_online_b200.config import SamplingConfig
    cfg = tiny[0]
    model, tok = _model(tiny)
    s = SamplingConfig(do_sample=True, temperature=0.8, top_k=20, top_p=0.9, seed=5) if sampled else None
    with_drafts = _run(model, tok, cfg, sampling=s)
    without = _run(model, tok, cfg, sampling=s, drafts=False)
    assert with_drafts[3] > 0 and with_drafts[4] <= WINDOW
    assert _same_run(with_drafts, without)


@pytest.mark.parametrize("drafts", [True, False])
def test_suspend_resume_continues_exactly(tiny, tmp_path, drafts):
    from videollm_online_b200.config import SamplingConfig
    cfg = tiny[0]
    model, tok = _model(tiny)
    s = SamplingConfig(do_sample=True, temperature=0.8, seed=9)
    want = _run(model, tok, cfg, sampling=s, drafts=drafts)
    assert want[3] > 0
    got = _run(model, tok, cfg, sampling=s, drafts=drafts, suspend_after=120, tmp_path=tmp_path)
    assert _same_run(got, want)


SCHED_FRAMES = 90
SCHED_WINDOW = 768


def test_scheduler_equals_liveinfer_with_swaps(tiny):
    """Three sessions keeping their turns under a window on an engine with 2 slots: each session's events, evictions,
    cache and history equal the same session alone through LiveInfer."""
    from videollm_online_b200.cli import synthetic_clip
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200.multistream import StreamScheduler
    cfg, llm, vis = tiny
    n = 3
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=2, max_kv_tokens=1024, max_step_tokens=128, max_vit_batch=8)
    I, E, END = cfg.frame_token_interval_id, cfg.eos_token_id, cfg.stream_end_id
    scripts = []
    for i in range(n):
        sc = {}
        for k in range(8 + i, 400, 40):
            sc[k] = END
            for j in range(1, 25):
                sc[k + j] = 300 + (i + j) % 7
        scripts.append(sc)
    sched = StreamScheduler(model, tok, n, frame_fps=2, system_prompt=SYSTEM_PROMPT)

    def hook(i, dec, k):
        s = sched.sessions[i]
        t = scripts[i].get(k, E if s.state == s.RESPOND else I)
        if s.state != s.RESPOND and t != END:
            t = I
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == I else 0.0
        if t != I:
            dec.argmax_excl_id = t
        return dec
    sched.decision_hook = hook
    for i, s in enumerate(sched.sessions):
        s.context_window, s.context_keep_turns = SCHED_WINDOW, True
        s.load_video(synthetic_clip(SCHED_FRAMES, cfg.frame_resolution, seed=i))
    for f in range(SCHED_FRAMES):
        for s in sched.sessions:
            s.input_video_stream(f / 2)
        while sched.tick():
            assert all(s.kv_tokens() <= SCHED_WINDOW for s in sched.sessions)
    assert sched.swaps_out > 0
    eng = model.engine
    want = {}
    for s in sched.sessions:          # resident sessions first, then the swapped-out ones through a free slot
        if s.resident:
            want[s.index] = (s.evicted_tokens, _kv_all(eng, s.stream_id), list(s.fed_ids))
            eng.stream_close(s.stream_id)
    for s in sched.sessions:
        if s.index not in want:
            sid = eng.stream_open()
            eng.kv_swap_in(sid, s.image)
            want[s.index] = (s.evicted_tokens, _kv_all(eng, sid), list(s.fed_ids))
            eng.stream_close(sid)
    assert all(w[0] > 0 for w in want.values())
    for i in range(n):
        li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT, context_window=SCHED_WINDOW,
                                     context_keep_turns=True), model=model, tokenizer=tok)
        li.prefetch_next = False
        li.drafter = None
        state = {"resp": False}
        respond = li._call_for_response

        def call_for_response(*a, respond=respond, state=state):
            state["resp"] = True
            try:
                return respond(*a)
            finally:
                state["resp"] = False
        li._call_for_response = call_for_response

        def hook1(dec, k, i=i, state=state):
            t = scripts[i].get(k, E if state["resp"] else I)
            if not state["resp"] and t != END:
                t = I
            dec.argmax_id = dec.argmax_prob_id = t
            dec.p_interval = 1.0 if t == I else 0.0
            if t != I:
                dec.argmax_excl_id = t
            return dec
        li.decision_hook = hook1
        li.load_video(synthetic_clip(SCHED_FRAMES, cfg.frame_resolution, seed=i))
        for f in range(SCHED_FRAMES):
            li.input_video_stream(f / 2)
            li()
        assert li.evicted_tokens == want[i][0], i
        assert li._fed_ids() == want[i][2], i
        assert _same_kv(_kv_all(eng, li._kv.stream_id), want[i][1]), i
        eng.stream_close(li._kv.stream_id)
