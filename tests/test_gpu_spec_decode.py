"""Greedy responses several tokens per step from drafts: a verify step [last | d1 | ... | dk] runs k + 1 one-token
segments, whose attention goes through one packed CTA per (split, kv head).  Every check is bit for bit against one
token per step: the attention op per segment, the engine's logits, decisions and KV cache, the generated ids for
scripted drafts of every kind, and LiveInfer's trace."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

PAGE = 64


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _plan_counts(lib, segs, Hq, Hk, kv_end):
    from videollm_online_b200._lib import check
    out = (C.c_int32 * 4)()
    check(lib.vlo_op_attn_plan_counts(len(segs), (C.c_int32 * len(segs))(*segs), Hq, Hk, 128, kv_end, out),
          "attn_plan_counts")
    return {"items": out[0], "clusters": out[1], "packs": out[2], "packed_items": out[3]}


# ------------------------------------------------------------------------------------------------ op level
def _runs(G):
    per = 64 // G
    lens = sorted({1, 2, 3, 5, 8, min(11, per), per})
    return [[1] * n for n in lens] + [[11] + [1] * n for n in (1, 4, per)] + [[3] + [1] * per + [2, 1, 1]]


@pytest.mark.parametrize("Hq,Hk", [(32, 8), (4, 2), (8, 8), (8, 1)])
@pytest.mark.parametrize("kv_end", [17, 1000, 1030, 12288 + 7, 66011])
def test_packed_runs_match_each_segment_alone(lib, kv_end, Hq, Hk):
    """Runs of 1 .. 64/G one-token segments, alone and behind longer segments: every segment gets the bits the paged op
    gives its rows alone.  kv_end 1030 and 12 295 put 64-key block boundaries inside the runs (rows of a run then
    cover one block fewer than its last row), 12 295 also the 12 288-key change of the single-token split grid, where
    the planner cuts a run.  Unused pool pages hold NaN."""
    from videollm_online_b200._lib import check
    torch.manual_seed(kv_end + 7 * Hq + Hk)
    D, G = 128, Hq // Hk
    nblk = (kv_end + PAGE - 1) // PAGE
    n_pages = nblk + 5
    perm = torch.randperm(n_pages, device="cuda")[:nblk]
    kp = torch.full((n_pages, Hk, PAGE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    vp = torch.full_like(kp, float("nan"))
    kp[perm] = torch.randn(nblk, Hk, PAGE, D, device="cuda").bfloat16()
    vp[perm] = torch.randn(nblk, Hk, PAGE, D, device="cuda").bfloat16()
    pt = perm.to(torch.int32).contiguous()
    ran = packed = 0
    for segs in _runs(G):
        n_tok = sum(segs)
        if n_tok > kv_end:
            continue
        ran += 1
        counts = _plan_counts(lib, segs, Hq, Hk, kv_end)
        ones = sum(1 for s in segs if s == 1)
        if ones >= 3 and kv_end != 12288 + 7:
            assert counts["packs"] >= 1, (segs, counts)
        packed += counts["packs"]
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
    assert ran > 0 and packed > 0


def test_plans_without_one_token_runs_are_unchanged(lib):
    """Frame batches, prompts and single tokens get no pack; a run cut by the split-grid change packs on each side."""
    for segs in ([1], [11] * 5, [40], [3] * 10, [11, 1], [1, 11]):
        assert _plan_counts(lib, segs, 32, 8, 12000)["packs"] == 0, segs
    c = _plan_counts(lib, [1] * 16, 32, 8, 12288 + 8)     # segments end at 12 281 .. 12 296
    assert c["packed_items"] == 16 and c["packs"] in (1, 2)   # 2 on 132 SMs: the grid changes past 12 288 keys
    c = _plan_counts(lib, [1] * 16, 8, 8, 12000)          # G = 1: one pack of up to 64 segments
    assert c["packs"] == 1 and c["packed_items"] == 16


# ------------------------------------------------------------------------------------------------ engine level
def _engine(cfg, llm, max_streams, max_kv_tokens, kv_pool_tokens=None):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=kv_pool_tokens)
    return model


@pytest.fixture(scope="module")
def wide():
    """two full-width Llama-3-8B decoder layers (hidden 4096, 32 / 8 heads, intermediate 14336)"""
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config(hidden_size=4096, num_attention_heads=32, num_key_value_heads=8, intermediate_size=14336)
    return cfg, W.synthetic_llm_state(cfg, seed=5)


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _same_kv(a, b):
    return len(a) == len(b) and all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))


def _pair(eng, fill):
    """two streams with identical contents: a synthetic fill copied across, then the same prompt step on both"""
    a, b = eng.stream_open(), eng.stream_open()
    eng.kv_fill_synthetic(a, fill, seed=3)
    eng.kv_copy_prefix(a, b, fill)
    g = torch.Generator().manual_seed(90)
    emb = torch.randn(21, eng.cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
    eng.step([a], [21], emb)
    eng.step([b], [21], emb)
    return a, b


def _tok_step(eng, sid, ids, segs=None):
    zeros = torch.zeros(len(ids), eng.cfg.hidden_size, dtype=torch.bfloat16, device="cuda")
    lg, dc = eng.step([sid], [len(ids)], zeros, row_ids=torch.tensor(ids, dtype=torch.int64), segments=segs)
    return lg.clone(), dc.clone()


@pytest.mark.parametrize("model,fill", [("tiny", 300), ("wide", 12288 - 150)])
def test_verify_step_equals_one_token_steps(tiny, wide, model, fill):
    """k = 0 .. 15 drafts: the verify step's logits rows and decisions equal those of k + 1 one-token steps; cut back
    after every acceptance point j, every layer's KV equals one token per step over the accepted tokens.  The wide
    model's cache grows across the 12 288-key change of the single-token split grid."""
    cfg, llm = (tiny[0], tiny[1]) if model == "tiny" else wide
    eng = _engine(cfg, llm, 2, fill + 2048).engine
    a, b = _pair(eng, fill)
    g = torch.Generator().manual_seed(11)
    for k in range(16):
        for j in range(k + 1):
            ids = torch.randint(0, cfg.vocab_size, (k + 1,), generator=g).tolist()
            kv0 = eng.kv_len(a)
            lg, dc = _tok_step(eng, a, ids, [[1] * (k + 1)] if k else None)
            for i, t in enumerate(ids):
                lb, db = _tok_step(eng, b, [t])
                assert torch.equal(lg[i], lb[0]) and torch.equal(dc[i], db[0]), f"k={k} j={j}: segment {i}"
            eng.kv_truncate(a, kv0 + j + 1)
            eng.kv_truncate(b, kv0 + j + 1)
            assert _same_kv(_kv_all(eng, a), _kv_all(eng, b)), f"k={k} j={j}: KV"
    assert eng.kv_len(a) > 12288 or model == "tiny"


# ------------------------------------------------------------------------------------------------ generation
def _one_token_loop(eng, sid, first, max_new, eos):
    """the parent's fast_greedy_generate over token ids: one step per token"""
    out, ids = [], list(first)
    while len(out) < max_new:
        _, dc = _tok_step(eng, sid, ids)
        new_id = eng.read_decisions(1)[0].argmax_id
        out.append(new_id)
        if new_id == eos:
            break
        ids = [new_id]
    return out


class Scripted:
    """a drafter that proposes fn(ids generated so far) (history calls are ignored)"""

    def __init__(self, fn):
        self.fn, self.n = fn, 0

    def sync(self, n):
        pass

    def extend(self, ids):
        pass

    def propose(self, k):
        return self.fn(self.n)[:k]


def _generate(eng, sid, first, max_new, eos, drafter):
    from videollm_online_b200.speculative import greedy_generate
    steps = []

    def step(ids, drafts):
        steps.append(len(drafts))
        _tok_step(eng, sid, ids + drafts, [[len(ids)] + [1] * len(drafts)] if drafts else None)

    def consume(d):
        drafter.n += 1
        return d
    return greedy_generate(eng, sid, step, len(first), max_new, eos, first_ids=first, drafter=drafter,
                           consume=consume), steps


@pytest.mark.parametrize("model", ["tiny", "wide"])
def test_generation_with_drafts_equals_one_token_per_step(tiny, wide, model):
    cfg, llm = (tiny[0], tiny[1]) if model == "tiny" else wide
    eng = _engine(cfg, llm, 2, 4096).engine
    first = [5, 17, 9]

    def case(max_new, eos, drafts_of, fill=700):
        a, b = _pair(eng, fill)
        want = _one_token_loop(eng, b, first, max_new, eos)
        got, steps = _generate(eng, a, first, max_new, eos, Scripted(lambda n: drafts_of(want, n)))
        assert got == want
        assert eng.kv_len(a) == eng.kv_len(b) and _same_kv(_kv_all(eng, a), _kv_all(eng, b))
        eng.stream_close(a)
        eng.stream_close(b)
        return want, steps

    ref, steps = case(40, -1, lambda w, n: w[n:n + 15])                 # perfect drafts
    assert len(ref) == 40 and steps == [13, 15, 9]                        # a 3-token prompt keeps its 16-row tile
    for bad in range(8):                                                  # a wrong draft at each position
        case(40, -1, lambda w, n, bad=bad: [x + 1 if i == bad else x for i, x in enumerate(w[n:n + 8])])
    _, steps = case(20, -1, lambda w, n: [])                              # no drafts
    assert steps == [0] * 20
    eos = ref[9]                                                          # EOS inside an accepted run
    want, _ = case(40, eos, lambda w, n: w[n:n + 15])
    assert want[-1] == eos and len(want) == ref.index(eos) + 1
    _, steps = case(20, -1, lambda w, n: w[n:n + 15])                     # the buffer ends inside a run
    assert steps == [13, 5]


def test_generation_caps_per_stream_and_pool(tiny):
    """Near max_kv_tokens, and on a pool without a free page, fewer drafts are verified than the drafter offers; ids and
    KV are those of one token per step, which ends at an EOS before either limit."""
    cfg, llm, _ = tiny
    first = [5, 17, 9]

    def case(model, fill, cap):
        eng = model.engine
        a, b = _pair(eng, fill)
        kv0 = eng.kv_len(b)
        eos = _one_token_loop(eng, b, first, 9, -1)[5]
        eng.kv_truncate(b, kv0)
        want = _one_token_loop(eng, b, first, 100, eos)
        assert want[-1] == eos and len(want) <= 6
        got, steps = _generate(eng, a, first, 100, eos, Scripted(lambda n: (want + [1] * 20)[n:n + 15]))
        assert got == want and eng.kv_len(a) == eng.kv_len(b)
        assert _same_kv(_kv_all(eng, a), _kv_all(eng, b))
        assert steps[0] == cap, steps
        return eng

    case(_engine(cfg, llm, 2, 1024), 1024 - 21 - 14, 11)        # kv 1010 + 3 prompt rows: room for 11 more
    eng = case(_engine(cfg, llm, 2, 1024, kv_pool_tokens=2 * 320), 320 - 21 - 12, 9)   # 308 rows in 5 of 10 pages
    assert eng.kv_pool_info()["free_pages"] == 0                 # each: no page free, room for 9 more rows


def test_fast_greedy_generate_matches_one_token_per_step(tiny):
    """fast_greedy_generate drafts from its own response: the ids and the cache are the one-token loop's."""
    from videollm_online_b200.modeling_live import StreamKV, fast_greedy_generate
    cfg, llm, _ = tiny
    model = _engine(cfg, llm, 2, 4096)
    eng = model.engine
    a, b = _pair(eng, 500)
    g = torch.Generator().manual_seed(4)
    emb = torch.randn(1, 6, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
    buf = torch.zeros(1, 100, dtype=torch.long)
    ids, kv = fast_greedy_generate(model=model, inputs_embeds=emb, past_key_values=StreamKV(eng, a), eos_token_id=-1,
                                   inplace_output_ids=buf)
    want = []
    x = emb[0]
    for _ in range(100):
        eng.step([b], [x.shape[0]], x.contiguous())
        want.append(eng.read_decisions(1)[0].argmax_id)
        x = eng.embed_tokens(torch.tensor([want[-1]]))
    assert ids[0].tolist() == want and kv.stream_id == a
    assert _same_kv(_kv_all(eng, a), _kv_all(eng, b))


# ------------------------------------------------------------------------------------------------ LiveInfer
@pytest.fixture(scope="module")
def built(tiny):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, _ = tiny
    return build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=2,
                      max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=1)


SPEAK_CALLS = {4, 9, 23}
QUERIES = [(0.0, "narrate"), (3.25, "between frames 6 and 7"), (8.0, "at frame 16")]


def _live_run(built, tiny, drafter):
    """scripted speaks and queries; every response is the same scripted id sequence ending in EOS"""
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    cfg = tiny[0]
    model, tok = built
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    iid, end_id, eos = cfg.frame_token_interval_id, cfg.stream_end_id, cfg.eos_token_id
    resp = [40, 41, 42, 40, 41, 42, 43, 44, 40, 41, 42, 43, 45, eos]
    state = {"resp": None}
    respond = li._call_for_response

    def call_for_response(*a):
        state["resp"] = 0
        try:
            return respond(*a)
        finally:
            state["resp"] = None
    li._call_for_response = call_for_response

    def hook(dec, n):
        if state["resp"] is not None:
            t = resp[state["resp"]]
            state["resp"] += 1
        else:
            t = end_id if n in SPEAK_CALLS else iid
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == iid else 0.0
        if t != iid:
            dec.argmax_excl_id = t
        return dec
    li.decision_hook = hook
    if drafter == "scripted":
        li.drafter = Scripted(lambda n: resp[state["resp"]:] if state["resp"] is not None else [])
    elif drafter is None:
        li.drafter = None
    g = torch.Generator().manual_seed(77)
    frames = [(i / 2, torch.randn(10, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()) for i in range(30)]
    for t, q in QUERIES:
        li.query_queue.append((t, q))
    trace = []
    li.frame_embeds_queue.extend(frames)
    while li.frame_embeds_queue:
        query, response = li()
        if query or response:
            trace.append((query, response, li.last_ids.reshape(-1).tolist(), li._kv.engine.kv_len(li._kv.stream_id)))
    kv = _kv_all(model.engine, li._kv.stream_id)
    out = trace, li._n_calls
    model.engine.stream_close(li._kv.stream_id)
    return out, kv


def test_liveinfer_with_drafts_equals_one_token_per_step(built, tiny):
    """A drafter that proposes the scripted response, the default n-gram drafter and none: the same trace (queries,
    responses, last ids, kv lengths), the same number of consumed decisions and the same final KV cache."""
    want, kv_want = _live_run(built, tiny, None)
    assert sum(1 for t in want[0] if t[1]) >= 3
    for d in ("scripted", "default"):
        got, kv_got = _live_run(built, tiny, d)
        assert got == want, d
        assert _same_kv(kv_got, kv_want), d
