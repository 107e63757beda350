"""Host images of a stream's KV cache (`vlo_kv_swap_out` / `vlo_kv_swap_in`): round trips through fragmented pools,
the engine's ordering of page reuse behind a swap-out, failures that change nothing, page accounting, and the session
level (`LiveInfer.suspend` / `resume` through torch.save, `StreamScheduler` with more sessions than the engine holds),
each compared bit for bit with a stream or session that was never swapped."""
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


def _step(eng, sids, lens, seed):
    """one step; returns (last-position logits, decisions, all-position logits), all cloned"""
    emb = _emb(eng.cfg, sum(lens), seed)
    logits, dec = eng.step(list(sids), list(lens), emb)
    out = (logits.clone(), dec.clone(), eng.last_step_logits(sum(lens)).clone())
    torch.cuda.synchronize()
    return out


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _same_kv(a, b):
    return len(a) == len(b) and all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))


def _same_step(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def _image_kv(img):
    """the per-layer (K, V) [kv_heads, n, head_dim] an image holds, as kv_read returns them"""
    L, Hk, D, P = img.layout
    n = img.n_tokens
    pages = -(-n // P)
    x = img.synchronize().data.view(torch.bfloat16).view(pages, L, 2, Hk, P, D)
    x = x.permute(1, 2, 3, 0, 4, 5).reshape(L, 2, Hk, pages * P, D)[:, :, :, :n].cuda()
    return [(x[l, 0].contiguous(), x[l, 1].contiguous()) for l in range(L)]


def _free(eng):
    return eng.kv_pool_info()["free_pages"]


def _pieces(n, k=41):
    return [min(k, n - o) for o in range(0, n, k)]


# ------------------------------------------------------------------------------------------------ engine level
def _round_trip(eng, n, seed):
    """a and its twin grow by the same steps, interleaved with a third stream (fragmented pages); a is swapped out, the
    third stream takes the freed pages and steps, a's image goes into a different slot: same cache, same next step"""
    a, twin, other = eng.stream_open(), eng.stream_open(), eng.stream_open()
    for r, q in enumerate(_pieces(n)):
        _step(eng, [a], [q], seed=seed + r)
        _step(eng, [other], [7 + r % 5], seed=seed + 500 + r)
        _step(eng, [twin], [q], seed=seed + r)
    before = _kv_all(eng, a)
    free0 = _free(eng)
    img = eng.kv_swap_out(a)
    assert eng.kv_len(a) == 0 and img.n_tokens == n
    assert _free(eng) == free0 + -(-n // PAGE)
    assert img.data.numel() == eng.kv_image_bytes(n) == -(-n // PAGE) * 2 * eng.cfg.num_hidden_layers * \
        eng.cfg.num_key_value_heads * PAGE * eng.cfg.head_dim * 2
    for r, q in enumerate(_pieces(-(-n // PAGE) * PAGE + 5, 128)):   # other reuses every page a gave back
        _step(eng, [other], [q], seed=seed + 900 + r)
    b = eng.stream_open()
    assert b not in (a, twin, other)
    eng.stream_close(a)
    eng.kv_swap_in(b, img)
    assert eng.kv_len(b) == n
    assert _same_kv(_kv_all(eng, b), before)
    assert _same_kv(_image_kv(img), before)
    for r, q in enumerate((1, 11, 40)):
        assert _same_step(_step(eng, [b], [q], seed=seed + 2000 + r), _step(eng, [twin], [q], seed=seed + 2000 + r)), q
    assert _same_kv(_kv_all(eng, b), _kv_all(eng, twin))
    for s in (b, twin, other):
        eng.stream_close(s)


@pytest.mark.parametrize("n", [1, 63, 64, 65, 300])
def test_round_trip_on_a_fragmented_pool(tiny, n):
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 4, 1024, kv_pool_tokens=3 * 1024)
    _round_trip(eng, n, seed=10 * n)


def test_round_trip_full_width():
    """Llama-3-8B attention shapes (4096 wide, 32 / 8 heads: 128 KB pages) and a 1000-token multi-page stream"""
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config(hidden_size=4096, num_attention_heads=32, num_key_value_heads=8)
    llm = W.synthetic_llm_state(cfg, seed=3)
    eng = _engine(cfg, llm, 4, 2048, kv_pool_tokens=3 * 2048)
    assert eng.kv_image_bytes(1000) == 16 * 2 * cfg.num_hidden_layers * 131072
    _round_trip(eng, 1000, seed=7)


def _reuse_after_swap_out(cfg, llm, writer):
    """a's swap-out runs on a side CUDA stream; right after it, `writer` on the main stream fills stream b, which is
    handed exactly the released pages (the pool holds nothing else), and b then steps"""
    n, m = 8000, 7800
    # kv_copy_prefix needs a source that holds m tokens of its own
    eng = _engine(cfg, llm, 3, 8192, kv_pool_tokens=n + (m if writer == "kv_copy_prefix" else 0))
    a, b, src = eng.stream_open(), eng.stream_open(), eng.stream_open()
    rows = torch.randn(cfg.num_key_value_heads, m, cfg.head_dim, device="cuda").bfloat16()
    if writer == "kv_copy_prefix":
        eng.kv_fill_synthetic(src, m, seed=2)
    if writer == "kv_swap_in":
        eng.kv_fill_synthetic(b, m, seed=2)
        img_b = eng.kv_swap_out(b)
    eng.kv_fill_synthetic(a, n, seed=1)
    before = _kv_all(eng, a)
    assert _free(eng) == 0
    main, side = torch.cuda.current_stream(), torch.cuda.Stream()
    side.wait_stream(main)
    with torch.cuda.stream(side):
        img = eng.kv_swap_out(a)
    assert _free(eng) == -(-n // PAGE)        # gated pages count as free
    # on the main stream, over a's old pages: b ends up with m tokens
    if writer == "kv_fill_synthetic":
        eng.kv_fill_synthetic(b, m, seed=2)
    elif writer == "kv_write":
        for layer in range(cfg.num_hidden_layers):
            for is_v in (False, True):
                eng.kv_write(b, layer, is_v, rows)
    elif writer == "kv_copy_prefix":
        eng.kv_copy_prefix(src, b, m)
    elif writer == "kv_swap_in":
        eng.kv_swap_in(b, img_b)
    else:
        eng.step([b], [m], _emb(cfg, m, 2))     # split into max_step_tokens pieces, none synchronised
    assert eng.kv_len(b) == m
    _step(eng, [b], [128], seed=3)
    _step(eng, [b], [72], seed=4)
    assert _free(eng) == 0
    assert _same_kv(_image_kv(img), before)
    eng.stream_close(b)
    eng.kv_swap_in(a, img)
    assert _same_kv(_kv_all(eng, a), before)


def test_page_reuse_waits_for_the_swap_out(tiny):
    """Whichever call first writes the pages a swap-out released (kv_fill_synthetic, kv_write, kv_copy_prefix,
    kv_swap_in or a step), the engine makes its CUDA stream wait for the swap-out's copies, so the image still equals
    the cache before the swap."""
    cfg, llm, _ = tiny
    for writer in ("kv_fill_synthetic", "kv_write", "kv_copy_prefix", "kv_swap_in", "step"):
        try:
            _reuse_after_swap_out(cfg, llm, writer)
        except AssertionError as err:
            raise AssertionError(f"first writer {writer}") from err


def test_failed_swap_in_changes_nothing(tiny):
    from videollm_online_b200._lib import VloError
    from videollm_online_b200.engine import KvImage
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 3, 1024, kv_pool_tokens=6 * PAGE)
    a, b = eng.stream_open(), eng.stream_open()
    _step(eng, [a], [100], seed=1)
    _step(eng, [b], [70], seed=2)
    want_a = _kv_all(eng, a)
    img = eng.kv_swap_out(a)
    _step(eng, [b], [128], seed=3)
    _step(eng, [b], [50], seed=4)
    _step(eng, [b], [60], seed=5)    # b: 308 tokens on 5 of the 6 pages; a needs 2
    assert _free(eng) == 1

    def snapshot():
        return _free(eng), eng.kv_len(a), eng.kv_len(b), _kv_all(eng, b)

    def same(x, y):
        return x[:3] == y[:3] and _same_kv(x[3], y[3])
    s0 = snapshot()
    with pytest.raises(VloError, match="KV page pool exhausted"):
        eng.kv_swap_in(a, img)
    assert same(snapshot(), s0)
    with pytest.raises(VloError, match="must be empty"):
        eng.kv_swap_in(b, img)
    assert same(snapshot(), s0)
    with pytest.raises(VloError, match="bytes"):
        eng.kv_swap_in(a, KvImage(img.data[:-2], img.n_tokens, img.layout))
    assert same(snapshot(), s0)
    L, Hk, D, P = img.layout
    with pytest.raises(VloError, match="layout"):
        eng.kv_swap_in(a, KvImage(img.data, img.n_tokens, (L + 1, Hk, D, P)))
    assert same(snapshot(), s0)
    eng.kv_truncate(b, 128)          # 2 pages: now it fits
    eng.kv_swap_in(a, img)
    assert _same_kv(_kv_all(eng, a), want_a)


def test_page_accounting(tiny):
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 3, 1024, kv_pool_tokens=3 * 1024)
    total = eng.kv_pool_info()["total_pages"]
    a, b = eng.stream_open(), eng.stream_open()
    for n in (1, 64, 65, 200):
        eng.kv_fill_synthetic(a, n, seed=n)
        f = _free(eng)
        img = eng.kv_swap_out(a)
        assert _free(eng) == f + -(-n // PAGE) and eng.kv_len(a) == 0
        eng.kv_swap_in(b, img)
        assert _free(eng) == f and eng.kv_len(b) == n
        img = eng.kv_swap_out(b)
        eng.kv_swap_in(a, img)
        eng.stream_reset(a)
    empty = eng.kv_swap_out(b)        # an empty stream gives an empty image
    assert empty.n_tokens == 0 and empty.data.numel() == 0
    eng.kv_swap_in(b, empty)
    assert eng.kv_len(b) == 0 and _free(eng) == total


# ------------------------------------------------------------------------------------------------ LiveInfer
N_FRAMES = 30
SPEAK_CALLS = {4, 9, 17}
QUERIES = [(0.0, "narrate"), (3.25, "between frames 6 and 7"), (8.0, "at frame 16"), (12.0, "at frame 24")]
FRAME = 10


def _session(model, tok, cfg):
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
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

    def hook(dec, n):   # a response is 2 scripted ids and EOS; frames speak ("]\n") at the scripted calls
        if state["resp"]:
            t = {0: 300, 1: 301}.get(state.setdefault("k", 0), eos)
            state["k"] = 0 if t == eos else state["k"] + 1
        else:
            t = end_id if n in SPEAK_CALLS else iid
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == iid else 0.0
        if t != iid:
            dec.argmax_excl_id = t
        return dec
    li.decision_hook = hook
    return li


def _frames(cfg):
    g = torch.Generator().manual_seed(77)
    return [(i / 2, torch.randn(FRAME + 1, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()) for i in range(N_FRAMES)]


def test_liveinfer_suspend_resume_through_torch_save(tiny, tmp_path):
    """Suspend with frames and queries queued, let another stream take the pages, torch.save / torch.load the state,
    resume in a new session on another stream slot: the trace (queries, responses, last ids, kv lengths), the call
    count and the final cache equal those of the uninterrupted session."""
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, _ = tiny
    model, tok = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=3,
                            max_kv_tokens=2048, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=2048)
    eng = model.engine

    def run(suspend_after):
        li = _session(model, tok, cfg)
        li.frame_embeds_queue.extend(_frames(cfg))
        li.query_queue.extend(QUERIES)
        trace = []
        calls = 0
        while li.frame_embeds_queue:
            query, response = li()
            calls += 1
            if query or response:
                trace.append((query, response, int(li.last_ids.reshape(-1)[-1]), eng.kv_len(li._kv.stream_id)))
            if calls == suspend_after:
                assert li.frame_embeds_queue and li.query_queue
                state = li.suspend()
                assert eng.kv_len(li._kv.stream_id) == 0 and not li.frame_embeds_queue
                intruder = eng.stream_open()     # takes the pages the session gave back, and more
                eng.kv_fill_synthetic(intruder, 1500, seed=5)
                eng.stream_close(intruder)
                torch.save(state, tmp_path / "session.pt")
                del state
                eng.stream_close(li._kv.stream_id)
                li = _session(model, tok, cfg)   # its hook is the same script; no response is under way
                li.resume(torch.load(tmp_path / "session.pt"))
        out = trace, li._n_calls, _kv_all(eng, li._kv.stream_id)
        eng.stream_close(li._kv.stream_id)
        return out

    want = run(None)
    assert any(t[0] is None for t in want[0]) and sum(t[0] is not None for t in want[0]) == len(QUERIES)
    for k in (1, 3):
        got = run(k)
        assert got[0] == want[0] and got[1] == want[1], k
        assert _same_kv(got[2], want[2]), k


# ------------------------------------------------------------------------------------------------ StreamScheduler
def _sched_run(tiny, windows, n_sessions, max_streams, kv_pool_tokens):
    """sessions take turns: session i is fed its clip at ticks windows[i] (one frame per feed); every decision is
    scripted, so each session's events and outputs depend on its own calls only"""
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
    scripts = [{2 + i % 3: END, 3 + i % 3: 300 + i, 4 + i % 3: 301} for i in range(n_sessions)]

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
        s.load_video(synthetic_clip(len(windows[i]), cfg.frame_resolution, seed=i))
    fed = [0] * n_sessions
    for tick in range(max(max(w) for w in windows) + 1):
        for i, s in enumerate(sched.sessions):
            if tick in windows[i]:
                s.input_video_stream(fed[i] / 2)
                fed[i] += 1
        sched.run_until_idle()
    eng = model.engine
    kv = []
    for s in sched.sessions:
        kv.append(_kv_all(eng, s.stream_id) if s.resident else (_image_kv(s.image) if s.image is not None else []))
    return [(s.events, s.outputs) for s in sched.sessions], kv, sched


def test_scheduler_with_more_sessions_than_slots_and_pages(tiny):
    """Six sessions on an engine with 2 stream slots and a pool that holds two of them, against an engine that holds
    all six.  Turns without overlap (one session steps per tick): events, outputs and every final cache are equal.
    Overlapping turns (up to three sessions want to step at once): events and outputs are equal."""
    n = 6
    alone = [range(6 * i, 6 * i + 5) for i in range(n)]
    want, want_kv, ref = _sched_run(tiny, alone, n, n, None)
    longest = max(kv[0][0].shape[1] for kv in want_kv)   # tokens of the longest session's cache
    pool = 2 * -(-(longest + 64) // PAGE) * PAGE
    got, got_kv, sched = _sched_run(tiny, alone, n, 2, pool)
    assert sched.swaps_out > 0 and sched.swaps_in > 0
    assert got == want
    for a, b in zip(got_kv, want_kv):
        assert _same_kv(a, b)
    overlap = [range(2 * i, 2 * i + 5) for i in range(n)]
    want, _, _ = _sched_run(tiny, overlap, n, n, None)
    got, _, sched = _sched_run(tiny, overlap, n, 2, pool)
    assert sched.swaps_out > 0
    assert got == want
