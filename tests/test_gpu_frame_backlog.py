"""Segmented decoder steps: a backlog of queued frames goes through one step [prefix | F1 | , | F2 | , ...] with one
decision per frame.  Every check is bit for bit against the same frames stepped one at a time: the attention op per
segment, the engine's logits, decisions and KV cache, cutting a step back after one of its frames, and LiveInfer's
trace with the whole clip queued at once."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

PAGE = 64
FRAME = 10   # frame rows of a segment; with the interval id row a segment is 11 tokens, as in the frame step


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


# ------------------------------------------------------------------------------------------------ op level
SEGMENTS = [[11] * k for k in range(1, 12)] + [[1, 11, 11], [14, 11, 11, 11], [45, 11, 11], [11, 1, 14, 45, 11],
                                               [6, 11], [1, 1, 1]]


@pytest.mark.parametrize("Hq,Hk", [(32, 8), (4, 2)])
@pytest.mark.parametrize("kv_end", [17, 1000, 12288 + 40, 66011])
def test_segments_op_matches_each_segment_alone(lib, kv_end, Hq, Hk):
    """Every segment of a segmented plan gets the bits the paged op gives its rows alone (kv length = the segment's
    end): at 12 328 keys an 11-frame batch has segments on both sides of the 12 288 split-grid change.  Pages are
    scattered in a pool whose unused pages hold NaN.  Items of one split grid run in clusters with a multicast cache
    pass (groups of 2 .. 8 items: one cluster; 9 .. 11: two), lone items on the per-item kernel."""
    from videollm_online_b200._lib import check
    torch.manual_seed(kv_end + Hq)
    D = 128
    nblk = (kv_end + PAGE - 1) // PAGE
    n_pages = nblk + 7
    perm = torch.randperm(n_pages, device="cuda")[:nblk]
    kp = torch.full((n_pages, Hk, PAGE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    vp = torch.full_like(kp, float("nan"))
    kp[perm] = torch.randn(nblk, Hk, PAGE, D, device="cuda").bfloat16()
    vp[perm] = torch.randn(nblk, Hk, PAGE, D, device="cuda").bfloat16()
    pt = perm.to(torch.int32).contiguous()
    ran = 0
    for segs in SEGMENTS:
        n_tok = sum(segs)
        if n_tok > kv_end:
            continue
        ran += 1
        q = torch.randn(n_tok, Hq, D, device="cuda").bfloat16()
        out = torch.full((n_tok, Hq * D), float("nan"), device="cuda", dtype=torch.bfloat16)
        lens = (C.c_int32 * len(segs))(*segs)
        check(lib.vlo_op_attn_kvappend_segments(_p(q), _p(kp), _p(vp), _p(pt), n_pages, _p(out), len(segs), lens, Hq, Hk,
                                                D, kv_end, _st()), "attn_segments")
        o = 0
        for j, n in enumerate(segs):
            end = kv_end - n_tok + o + n
            alone = torch.empty(n, Hq * D, device="cuda", dtype=torch.bfloat16)
            ws = torch.empty(lib.vlo_op_attn_ws_bytes(n, Hq, D, end), device="cuda", dtype=torch.uint8)
            qj = q[o:o + n].contiguous()
            check(lib.vlo_op_attn_kvappend_paged(_p(qj), _p(kp), _p(vp), _p(pt), n_pages, _p(alone), _p(ws), n, Hq, Hk, D,
                                                 end, _st()), "attn_paged")
            torch.cuda.synchronize()
            assert torch.equal(out[o:o + n], alone), f"segments {segs}, segment {j}"
            o += n
        assert torch.isfinite(out.float()).all()
    assert ran > 0


# ------------------------------------------------------------------------------------------------ engine level
def _engine(cfg, llm, max_streams, max_kv_tokens, kv_pool_tokens=None):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=kv_pool_tokens)
    return model.engine


@pytest.fixture(scope="module")
def wide():
    """two full-width Llama-3-8B decoder layers (hidden 4096, 32 / 8 heads, intermediate 14336)"""
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config(hidden_size=4096, num_attention_heads=32, num_key_value_heads=8, intermediate_size=14336)
    return cfg, W.synthetic_llm_state(cfg, seed=5)


def _frames(cfg, k, seed):
    """k frames of FRAME embedding rows + the row ids of a frame run: segment 1 = [prefix id | F1], then [, | Fj]"""
    g = torch.Generator().manual_seed(seed)
    emb = torch.randn(k * (FRAME + 1), cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
    ids = torch.full((k, FRAME + 1), -1, dtype=torch.int64)
    ids[:, 0] = cfg.frame_token_interval_id
    ids[0, 0] = 7   # the prefix of the first frame (a token other than the interval id)
    return emb, ids.view(-1).cuda()


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _same_kv(a, b):
    return len(a) == len(b) and all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))


def _one_by_one(eng, sid, emb, ids, k):
    """the k frames as k single steps; per frame (logits row, decision row)"""
    out = []
    for j in range(k):
        r = slice(j * (FRAME + 1), (j + 1) * (FRAME + 1))
        lg, dc = eng.step([sid], [FRAME + 1], emb[r].contiguous(), row_ids=ids[r])
        out.append((lg[0].clone(), dc[0].clone()))
    return out


def _segmented(eng, sid, emb, ids, k):
    lg, dc = eng.step([sid], [k * (FRAME + 1)], emb, row_ids=ids, segments=[[FRAME + 1] * k])
    assert lg.shape[0] == k and dc.shape[0] == k
    return [(lg[j].clone(), dc[j].clone()) for j in range(k)]


def _prefixed_pair(eng, fill):
    """two streams with identical contents: a synthetic fill copied across, then the same real steps on both"""
    a, b = eng.stream_open(), eng.stream_open()
    eng.kv_fill_synthetic(a, fill, seed=3)
    eng.kv_copy_prefix(a, b, fill)
    for r, n in enumerate((40, 11, 1)):
        g = torch.Generator().manual_seed(90 + r)
        emb = torch.randn(n, eng.cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
        eng.step([a], [n], emb)
        eng.step([b], [n], emb)
    return a, b


@pytest.mark.parametrize("model,fill", [("tiny", 300), ("wide", 12288 - 140)])
def test_segmented_step_equals_one_frame_per_step(tiny, wide, model, fill):
    """K = 1 .. 11 frames as one segmented step on stream a and as K single steps on stream b (same contents): every
    segment's logits row and decision, every layer's K and V and the kv length agree bit for bit.  The step's token
    tile runs through the widths 16 / 32 / 64 / 96 / 128; at the wide model's 12k fill the later batches cross the
    12 288-key change of the single-frame split grid."""
    cfg, llm = (tiny[0], tiny[1]) if model == "tiny" else wide
    eng = _engine(cfg, llm, 2, fill + 1024)
    a, b = _prefixed_pair(eng, fill)
    for k in range(1, 12):
        emb, ids = _frames(cfg, k, seed=k)
        got, want = _segmented(eng, a, emb, ids, k), _one_by_one(eng, b, emb, ids, k)
        torch.cuda.synchronize()
        for j in range(k):
            assert torch.equal(got[j][0], want[j][0]), f"K={k}: logits of frame {j}"
            assert torch.equal(got[j][1], want[j][1]), f"K={k}: decision of frame {j}"
        assert eng.kv_len(a) == eng.kv_len(b)
        assert _same_kv(_kv_all(eng, a), _kv_all(eng, b)), f"K={k}: KV cache"
    assert torch.isfinite(got[-1][0].float()).all()


def test_cut_back_after_a_segment_then_continue(tiny):
    """A 6-frame step cut back to the end of frame 2 (a frame that speaks), then the next steps: the same as stepping
    frames 1-3 alone and continuing.  The cut gives the pages of the dropped frames back."""
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 2, 2048)
    a, b = _prefixed_pair(eng, 290)   # 290 + 52 = 342: the 6-frame step spans a page boundary after frame 3
    emb, ids = _frames(cfg, 6, seed=21)
    kv0 = eng.kv_len(a)
    _segmented(eng, a, emb, ids, 6)
    eng.kv_truncate(a, kv0 + 3 * (FRAME + 1))
    _one_by_one(eng, b, emb, ids, 3)
    info = eng.kv_pool_info()
    assert info["total_pages"] - info["free_pages"] == sum((eng.kv_len(s) + PAGE - 1) // PAGE for s in (a, b))
    for r, (n, k) in enumerate(((3, 4), (1, 1))):   # an AR token, then 4 more frames / 1 frame
        g = torch.Generator().manual_seed(40 + r)
        tok = torch.randn(n, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
        la, da = eng.step([a], [n], tok)
        la, da = la.clone(), da.clone()
        lb, db = eng.step([b], [n], tok)
        assert torch.equal(la, lb) and torch.equal(da, db)
        emb, ids = _frames(cfg, k, seed=50 + r)
        got, want = _segmented(eng, a, emb, ids, k), _one_by_one(eng, b, emb, ids, k)
        assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(got, want))
    assert eng.kv_len(a) == eng.kv_len(b)
    assert _same_kv(_kv_all(eng, a), _kv_all(eng, b))


def test_segmented_step_on_an_exhausted_pool_changes_nothing(tiny):
    from videollm_online_b200._lib import VloError
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 2, 1024, kv_pool_tokens=256)
    a = eng.stream_open()
    eng.kv_fill_synthetic(a, 200, seed=1)
    before = _kv_all(eng, a)
    emb, ids = _frames(cfg, 6, seed=3)   # 200 + 66 > 256
    with pytest.raises(VloError, match="KV page pool exhausted"):
        _segmented(eng, a, emb, ids, 6)
    torch.cuda.synchronize()
    assert eng.kv_len(a) == 200 and eng.kv_pool_info()["free_pages"] == 0
    assert _same_kv(_kv_all(eng, a), before)
    emb, ids = _frames(cfg, 5, seed=3)   # 200 + 55 fits
    _segmented(eng, a, emb, ids, 5)
    assert eng.kv_len(a) == 255


def test_segmented_step_arguments(tiny):
    from videollm_online_b200._lib import VloError
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 1, 1024)
    a = eng.stream_open()
    emb = torch.zeros(130, cfg.hidden_size, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(VloError, match="not chunked"):
        eng.step([a], [130], emb, segments=[[65, 65]])
    with pytest.raises(VloError, match="add up"):
        eng.step([a], [22], emb[:22], segments=[[11, 10]])
    assert eng.kv_len(a) == 0


# ------------------------------------------------------------------------------------------------ LiveInfer
@pytest.fixture(scope="module")
def built(tiny):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, _ = tiny
    return build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=2,
                      max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=1)


N_FRAMES = 40
SPEAK_CALLS = {4, 9, 10, 23, 30}        # decisions (by call index) scripted to speak
QUERIES = [(0.0, "narrate"), (3.25, "between frames 6 and 7"), (8.0, "at frame 16"), (12.0, "at frame 24")]


def _run(built, tiny, mode):
    """mode 'queued': every frame queued before the first call; 'one_per_call': one frame queued per call;
    'single_steps': everything queued, but the session steps one frame at a time"""
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    cfg = tiny[0]
    model, tok = built
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

    def hook(dec, n):   # the response is a single EOS; frames speak ("]\n") at the scripted calls, else stay silent
        t = eos if state["resp"] else (end_id if n in SPEAK_CALLS else iid)
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == iid else 0.0
        if t != iid:
            dec.argmax_excl_id = t
        return dec
    li.decision_hook = hook
    if mode == "single_steps":
        li._backlog_run = lambda: 1
    runs = []
    backlog = li._stream_backlog

    def stream_backlog(n):
        runs.append(n)
        return backlog(n)
    li._stream_backlog = stream_backlog
    g = torch.Generator().manual_seed(77)
    frames = [(i / 2, torch.randn(FRAME, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()) for i in range(N_FRAMES)]
    for t, q in QUERIES:
        li.query_queue.append((t, q))
    trace = []

    def call():
        query, response = li()
        if query or response:
            trace.append((query, response, int(li.last_ids.reshape(-1)[-1]), li._kv.engine.kv_len(li._kv.stream_id)))
    if mode == "one_per_call":
        for f in frames:
            li.frame_embeds_queue.append(f)
            call()
    else:
        li.frame_embeds_queue.extend(frames)
    while li.frame_embeds_queue:
        call()
    out = trace, li._n_calls, li._kv.engine.kv_len(li._kv.stream_id)
    model.engine.stream_close(li._kv.stream_id)
    return out, runs


def test_liveinfer_backlog_equals_one_frame_per_step(built, tiny):
    """The clip queued at once (segmented steps), one frame queued per call, and one frame per step: the same
    (query, response, last id, kv length) trace and the same number of consumed decisions.  The script speaks inside
    batches, and queries fall due between two queued frames and exactly at a frame's time."""
    want, runs = _run(built, tiny, "single_steps")
    assert not runs
    assert [t[0] for t in want[0] if t[0]] == [f"(Video Time = {t}s) User: {q}" for t, q in QUERIES]
    assert any(t[0] is None for t in want[0])   # frames that spoke
    got, runs = _run(built, tiny, "queued")
    assert got == want
    assert runs and max(runs) > 2
    got, _ = _run(built, tiny, "one_per_call")
    assert got == want


def test_cli_whole_video_drains_the_clip(tiny):
    """`cli --whole_video`: the clip is queued at t = 0 and drained through segmented steps.  The conversation and the
    number of consumed decisions are those of the per-frame cli loop on the same clip (the ViT encodes the clip in
    batches there and frame by frame here, so the trace is compared, not the cache bits)."""
    from videollm_online_b200 import cli
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = tiny
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=1, max_kv_tokens=2048, max_step_tokens=128, max_vit_batch=4)
    clip = cli.synthetic_clip(30, cfg.frame_resolution, seed=4)
    I, E, END = cfg.frame_token_interval_id, cfg.eos_token_id, cfg.stream_end_id
    script = {0: I, 1: E, 13: END, 14: E}   # narration query answered at once; a frame speaks in the middle

    def run(whole):
        li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
        li.prefetch_next = False

        def hook(dec, n):
            t = script.get(n, I)
            dec.argmax_id = dec.argmax_prob_id = t
            dec.p_interval = 1.0 if t == I else 0.0
            if t != I:
                dec.argmax_excl_id = t
            return dec
        li.decision_hook = hook
        fps, history = cli.main(li, video=clip, n_iters=30, quiet=True, whole_video=whole)
        out = [(c["role"], c["content"]) for c in history["conversation"] if "role" in c], li._n_calls, \
            li.past_key_values.get_seq_length(), len(li.frame_embeds_queue)
        model.engine.stream_close(li._kv.stream_id)
        return fps, out
    fps, got = run(True)
    _, want = run(False)
    assert fps > 0 and got == want and got[3] == 0
    assert [r for r, _ in got[0]] == ["user", "assistant", "assistant"]


def test_many_short_segments_equal_single_steps(tiny):
    """40 segments of 3 tokens: the lm_head and the decision run on 40 rows (a 64-wide token tile), the attention on 40
    items of one stream in clusters; every segment still equals its own step."""
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm, 2, 2048)
    a, b = _prefixed_pair(eng, 500)
    g = torch.Generator().manual_seed(8)
    emb = torch.randn(120, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
    lg, dc = eng.step([a], [120], emb, segments=[[3] * 40])
    got = [(lg[j].clone(), dc[j].clone()) for j in range(40)]
    for j in range(40):
        lb, db = eng.step([b], [3], emb[3 * j:3 * j + 3].contiguous())
        assert torch.equal(got[j][0], lb[0]) and torch.equal(got[j][1], db[0]), f"segment {j}"
    assert _same_kv(_kv_all(eng, a), _kv_all(eng, b))
