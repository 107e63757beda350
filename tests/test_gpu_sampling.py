"""Response sampling on the device (sample_kernel, vlo_sample): the filters against transformers' own logits processors,
the draw against a NumPy restatement of the noise, the distribution, determinism, and the exactness of sampled
responses under draft verification, batching and suspend / resume."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

from sampling_reference import gumbel, penalised

pytestmark = pytest.mark.gpu


def _p(t):
    return C.c_void_p(t.data_ptr())


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _op_sample(lib, logits, params, penalty_ids=()):
    """vlo_op_sample over logits [n, V]; params: one dict of vlo_sample_row fields per row.  Returns (ids, kept,
    top-k threshold, top-p threshold) as host lists."""
    from videollm_online_b200._lib import VloSampleRow, check
    n = logits.shape[0]
    rows = (VloSampleRow * n)()
    for r, p in zip(rows, params):
        for k, v in p.items():
            setattr(r, k, v)
    pen = (C.c_int32 * max(1, len(penalty_ids)))(*penalty_ids)
    out = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    info = torch.zeros(n, 4, dtype=torch.int32, device="cuda")
    check(lib.vlo_op_sample(_p(logits), n, logits.shape[1], rows, C.cast(pen, C.c_void_p), len(penalty_ids), _p(out),
                            _p(info), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "vlo_op_sample")
    info = info.cpu()
    f = info.view(torch.float32)
    return out.cpu().tolist(), info[:, 0].tolist(), f[:, 1].tolist(), f[:, 2].tolist()


def _row(seed=1, position=0, temperature=1.0, top_k=0, top_p=1.0, repetition_penalty=1.0, off=0, count=0):
    return dict(seed=seed, position=position, temperature=temperature, top_k=top_k, top_p=top_p,
                repetition_penalty=repetition_penalty, penalty_offset=off, penalty_count=count)


def _hf_mask(l, top_k, top_p):
    """kept ids of transformers' TopK / TopP warpers (fp32, CPU) on the already penalised and tempered scores l"""
    from transformers.generation.logits_process import TopKLogitsWarper, TopPLogitsWarper
    s = l[None].clone()
    ids = torch.zeros(1, 1, dtype=torch.long)
    if top_k:
        s = TopKLogitsWarper(top_k)(ids, s)
    if top_p < 1:
        s = TopPLogitsWarper(top_p)(ids, s)
    return s[0] != -float("inf")


def _hf_penalised(row, temperature, penalty, penalty_ids):
    """transformers' RepetitionPenalty + Temperature processors (fp32, CPU)"""
    from transformers.generation.logits_process import RepetitionPenaltyLogitsProcessor, TemperatureLogitsWarper
    s = row.float()[None].clone()
    if penalty != 1.0 and len(penalty_ids):
        s = RepetitionPenaltyLogitsProcessor(penalty)(torch.tensor([list(penalty_ids)]), s)
    if temperature != 1.0:
        s = TemperatureLogitsWarper(temperature)(torch.zeros(1, 1, dtype=torch.long), s)
    return s[0]


def _top_p_ambiguous(l, top_k, top_p, tol=1e-6):
    """The row's top-p boundary lies within rounding reach (1e-6 plus HF's own fp32 cumulative-sum error against fp64)
    or in a tie group HF may split by its sort order."""
    if top_p >= 1:
        return False
    keep_k = l >= torch.topk(l, top_k).values[-1] if 0 < top_k < l.numel() else torch.ones_like(l, dtype=torch.bool)
    lk = l.masked_fill(~keep_k, -float("inf"))
    asc = torch.sort(lk).values
    err = float((torch.softmax(asc, 0).cumsum(0).double() - torch.softmax(asc.double(), 0).cumsum(0)).abs().max())
    vals, counts = torch.unique(torch.softmax(lk.double(), 0), return_counts=True)
    vals, counts = vals.flip(0), counts.flip(0)            # distinct probabilities, descending
    mass = vals * counts
    above = torch.cumsum(mass, 0) - mass                   # mass strictly above each value
    b = int((above < top_p).sum()) - 1                     # the boundary group: the last one kept
    eps = tol + err
    near = abs(float(above[b]) - top_p) < eps or (b + 1 < vals.numel() and abs(float(above[b + 1]) - top_p) < eps)
    split = int(counts[b]) > 1 and float(above[b] + (counts[b] - 1) * vals[b]) >= top_p - eps
    return near or split


CONFIGS = [  # temperature, top_k, top_p, penalty
    (1.0, 0, 0.9, 1.0), (0.6, 0, 0.9, 1.0), (0.7, 50, 1.0, 1.0), (1.3, 40, 0.8, 1.0), (0.8, 0, 0.95, 1.3),
    (1.0, 1000, 0.7, 0.7), (0.5, 7, 1.0, 2.0), (1.0, 0, 1.0, 1.2),
]


def _rows_for(V, g, n):
    """peaky bf16 rows: a noise floor and a few hot ids, so that top-p boundaries mostly fall between distinct values"""
    rows = torch.randn(n, V, generator=g) * 1.5
    for r in rows:
        hot = torch.randperm(V, generator=g)[:24]
        r[hot] = 4 + 10 * torch.rand(24, generator=g)
    return rows.to(torch.bfloat16)


@pytest.mark.parametrize("V", [128256, 1024])
def test_filtering_equals_transformers(lib, V):
    g = torch.Generator().manual_seed(V)
    checked = skipped = 0
    for ci, (T, K, P, pen) in enumerate(CONFIGS):
        rows = _rows_for(V, g, 6)
        pids = []
        params = []
        for r in range(rows.shape[0]):
            hot = torch.topk(rows[r].float(), 30).indices.tolist()
            neg = torch.topk(-rows[r].float(), 10).indices.tolist()
            ids = hot[::2] + neg + hot[:3] + [V + 5, -1]             # positive and negative logits, repeats, out of range
            params.append(_row(seed=ci, position=r, temperature=T, top_k=K, top_p=P, repetition_penalty=pen,
                               off=len(pids), count=len(ids)))
            pids += ids
        ids_out, kept, thr_k, thr_p = _op_sample(lib, rows.cuda(), params, pids)
        for r in range(rows.shape[0]):
            ids = pids[params[r]["penalty_offset"]:params[r]["penalty_offset"] + params[r]["penalty_count"]]
            l = penalised(rows[r], T, pen, ids)
            assert torch.equal(l, _hf_penalised(rows[r], T, pen, [i for i in ids if 0 <= i < V])), (ci, r)
            if _top_p_ambiguous(l, K, P):
                skipped += 1
                continue
            checked += 1
            want = _hf_mask(l, K, P)
            got = l >= max(thr_k[r], thr_p[r])
            assert torch.equal(got, want), (ci, r, int(got.sum()), int(want.sum()))
            assert kept[r] == int(want.sum())
            assert bool(want[ids_out[r]])
    assert checked >= 30 and skipped <= checked // 3, (checked, skipped)


def test_draw_equals_numpy_restatement(lib):
    g = torch.Generator().manual_seed(3)
    checked = excused = 0
    for V, n in ((128256, 24), (1024, 64)):
        rows = _rows_for(V, g, n)
        params = [_row(seed=(i * 2654435761) % 2 ** 64 + 2 ** 40, position=1000 * i + 3, temperature=(0.6, 1.0, 1.7)[i % 3],
                       top_k=(0, 50)[i % 2], top_p=(1.0, 0.9)[(i // 2) % 2]) for i in range(n)]
        ids, kept, thr_k, thr_p = _op_sample(lib, rows.cuda(), params)
        for i in range(n):
            p = params[i]
            l = penalised(rows[i], p["temperature"], 1.0, [])
            mask = (l >= max(thr_k[i], thr_p[i])).numpy()
            sc = np.where(mask, l.double().numpy() + gumbel(p["seed"], p["position"], V), -np.inf)
            top2 = np.sort(sc)[-2:]
            if top2[1] - top2[0] < 1e-4:
                excused += 1
                continue
            checked += 1
            assert ids[i] == int(np.argmax(sc)), i
    assert checked >= 80 and excused <= 2, (checked, excused)


def test_distribution_chi_square(lib):
    from scipy.stats import chisquare
    V, N, per = 1024, 120_000, 30_000
    g = torch.Generator().manual_seed(9)
    row = (torch.randn(V, generator=g) * 2).to(torch.bfloat16)
    T, K, P = 0.8, 60, 0.9
    counts = np.zeros(V, dtype=np.int64)
    for b in range(N // per):
        logits = row[None].repeat(per, 1).cuda()
        ids, kept, thr_k, thr_p = _op_sample(lib, logits, [_row(seed=424242, position=b * per + i, temperature=T,
                                                                  top_k=K, top_p=P) for i in range(per)])
        counts += np.bincount(np.array(ids), minlength=V)
        assert len(set(kept)) == 1 and len(set(thr_k)) == 1 and len(set(thr_p)) == 1
    l = penalised(row, T, 1.0, []).double()
    mask = l >= max(thr_k[0], thr_p[0])
    p = torch.softmax(l.masked_fill(~mask, -float("inf")), 0).numpy()
    assert counts[~mask.numpy()].sum() == 0
    exp = p * N
    big = exp >= 5
    obs = np.append(counts[big], counts[~big & mask.numpy()].sum())
    e = np.append(exp[big], exp[~big & mask.numpy()].sum())
    if e[-1] == 0:
        obs, e = obs[:-1], e[:-1]
    assert chisquare(obs, e).pvalue > 1e-4


def test_determinism_and_batch_invariance(lib):
    g = torch.Generator().manual_seed(5)
    rows = _rows_for(128256, g, 64).cuda()
    params = [_row(seed=17 + i, position=i * 7, temperature=0.9, top_k=(0, 100)[i % 2], top_p=(0.9, 1.0)[(i // 2) % 2],
                   repetition_penalty=1.2, off=0, count=40) for i in range(64)]
    pids = list(range(0, 4000, 100))
    a = _op_sample(lib, rows, params, pids)[0]
    assert a == _op_sample(lib, rows, params, pids)[0]
    for i in (0, 13, 63):
        assert _op_sample(lib, rows[i:i + 1], [params[i]], pids)[0] == [a[i]]
    rev = _op_sample(lib, rows.flip(0).contiguous(), params[::-1], pids)[0]
    assert rev[::-1] == a


def test_top_k_one_is_the_argmax(lib):
    from videollm_online_b200._lib import VloDecision, check
    g = torch.Generator().manual_seed(6)
    rows = (torch.randn(32, 128256, generator=g) * 3).to(torch.bfloat16).cuda()
    ids = _op_sample(lib, rows, [_row(seed=i, position=i, temperature=(0.3, 1.0, 2.0)[i % 3], top_k=1) for i in range(32)])[0]
    dec = torch.zeros(32, 8, dtype=torch.int32, device="cuda")
    check(lib.vlo_op_decision(_p(rows), 32, 128256, -1, _p(dec), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
          "decision")
    dec = dec.cpu()
    margin = dec.view(torch.float32)[:, 4]
    n = 0
    for i in range(32):
        if float(margin[i]) > 0:   # no tied maximum
            n += 1
            assert ids[i] == int(dec[i, 0])
    assert n >= 16


def test_skipped_rows_and_bad_parameters(lib):
    from videollm_online_b200._lib import VloError
    rows = torch.randn(3, 1024).to(torch.bfloat16).cuda()
    ids = _op_sample(lib, rows, [_row(temperature=0.0), _row(top_k=1), _row(temperature=0.0)])[0]
    assert ids[0] == -1 and ids[2] == -1 and float(rows[1, ids[1]]) == float(rows[1].float().max())
    for bad in (dict(temperature=-1.0), dict(top_p=0.0), dict(top_k=-2), dict(repetition_penalty=0.0),
                dict(repetition_penalty=1.5, count=5)):
        with pytest.raises(VloError):
            _op_sample(lib, rows[:1], [_row(**bad)], [1, 2])


# ------------------------------------------------------------------------------------------------ engine and generation
def _engine(cfg, llm, max_streams=2, max_kv_tokens=4096):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1)
    return model


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _same_kv(a, b):
    return len(a) == len(b) and all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))


def _pair(eng, fill):
    a, b = eng.stream_open(), eng.stream_open()
    eng.kv_fill_synthetic(a, fill, seed=3)
    eng.kv_copy_prefix(a, b, fill)
    g = torch.Generator().manual_seed(90)
    emb = torch.randn(21, eng.cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
    eng.step([a], [21], emb)
    eng.step([b], [21], emb)
    return a, b


def _tok_step(eng, sid, ids, segs=None, sample=None):
    zeros = torch.zeros(len(ids), eng.cfg.hidden_size, dtype=torch.bfloat16, device="cuda")
    eng.step([sid], [len(ids)], zeros, row_ids=torch.tensor(ids, dtype=torch.int64), segments=segs, sample=sample)


def _one_token_sampled(eng, sid, first, max_new, eos, s):
    """one step per token; the SampleRow restated from the documented rule: the position of the logits' token and the
    prompt plus the ids so far"""
    from videollm_online_b200.engine import SampleRow
    out, ids = [], list(first)
    while len(out) < max_new:
        pos = eng.kv_len(sid) + len(ids) - 1
        row = SampleRow(s.seed, pos, s.temperature, s.top_k, s.top_p, s.repetition_penalty, list(first) + out)
        _tok_step(eng, sid, ids, sample=[row])
        d = eng.read_decisions(1)[0]
        assert d.sampled_id is not None
        out.append(d.sampled_id)
        if out[-1] == eos:
            break
        ids = [out[-1]]
    return out


class Scripted:
    def __init__(self, fn):
        self.fn, self.n = fn, 0

    def sync(self, n):
        pass

    def extend(self, ids):
        pass

    def propose(self, k):
        return self.fn(self.n)[:k]


SAMPLING = [dict(temperature=0.7, top_k=0, top_p=1.0, repetition_penalty=1.0, seed=1),
            dict(temperature=1.3, top_k=20, top_p=0.9, repetition_penalty=1.0, seed=2),
            dict(temperature=1.0, top_k=0, top_p=0.8, repetition_penalty=1.3, seed=2 ** 63 + 5),
            dict(temperature=0.5, top_k=50, top_p=1.0, repetition_penalty=0.8, seed=77)]


@pytest.mark.parametrize("si", range(len(SAMPLING)))
def test_sampled_generation_with_drafts_equals_one_token_per_step(tiny, si):
    from videollm_online_b200.config import SamplingConfig
    from videollm_online_b200.speculative import generate_ids
    cfg, llm, _ = tiny
    s = SamplingConfig(do_sample=True, **SAMPLING[si])
    eng = _engine(cfg, llm).engine
    first = [5, 17, 9]

    def case(max_new, eos, drafts_of, fill=700):
        a, b = _pair(eng, fill)
        want = _one_token_sampled(eng, b, first, max_new, eos, s)
        dr = Scripted(lambda n: drafts_of(want, n))
        steps = []

        def step(ids, drafts, rows):
            steps.append(len(drafts))
            _tok_step(eng, a, ids + drafts, [[len(ids)] + [1] * len(drafts)] if drafts else None, sample=rows)

        def consume(d):
            dr.n += 1
            return d
        got = generate_ids(eng, a, step, len(first), max_new, eos, first_ids=first, drafter=dr, consume=consume,
                           sampling=s)
        assert got == want
        assert eng.kv_len(a) == eng.kv_len(b) and _same_kv(_kv_all(eng, a), _kv_all(eng, b))
        eng.stream_close(a)
        eng.stream_close(b)
        return want, steps

    ref, steps = case(40, -1, lambda w, n: w[n:n + 15])                 # perfect drafts
    assert len(ref) == 40 and max(steps) >= 5
    for bad in (0, 3, 7):                                                 # a wrong draft
        case(40, -1, lambda w, n, bad=bad: [(x + 1) % cfg.vocab_size if i == bad else x for i, x in enumerate(w[n:n + 8])])
    case(20, -1, lambda w, n: [])                                         # no drafts
    eos = ref[9]                                                          # EOS inside an accepted run
    want, _ = case(40, eos, lambda w, n: w[n:n + 15])
    assert want[-1] == eos and len(want) == ref.index(eos) + 1
    assert len(set(ref)) > 5


def test_sampled_ids_depend_on_seed_and_config(tiny):
    from videollm_online_b200.config import SamplingConfig
    cfg, llm, _ = tiny
    eng = _engine(cfg, llm).engine
    outs = []
    for kw in (SAMPLING[0], dict(SAMPLING[0], seed=2), dict(SAMPLING[0], temperature=2.0)):
        a, b = _pair(eng, 300)
        outs.append(_one_token_sampled(eng, a, [5, 17, 9], 30, -1, SamplingConfig(do_sample=True, **kw)))
        eng.stream_close(a)
        eng.stream_close(b)
    assert outs[0] != outs[1] and outs[0] != outs[2]


# ------------------------------------------------------------------------------------------------ sessions
@pytest.fixture(scope="module")
def built(tiny):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = tiny
    return build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                      max_streams=4, max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=4)


SPEAK = {2, 6}   # frame decisions (counted per session) that speak; responses are left to the model


def _force(cfg, dec, speak):
    t = cfg.stream_end_id if speak else cfg.frame_token_interval_id
    dec.argmax_id = dec.argmax_prob_id = t
    dec.p_interval = 0.0 if speak else 1.0
    if speak:
        dec.argmax_excl_id = t
    return dec


def _live(built, sampling):
    """a LiveInfer whose frame decisions are scripted (SPEAK); st["ids"] collects each response's ids"""
    from videollm_online_b200.config import LiveArguments, SamplingConfig, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    model, tok = built
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    li.sampling = SamplingConfig(do_sample=True, **sampling) if sampling else None
    st = {"resp": False, "frames": 0, "ids": []}
    respond = li._call_for_response

    def call_for_response(*a):
        st["resp"] = True
        st["ids"].append([])
        try:
            return respond(*a)
        finally:
            st["resp"] = False
    li._call_for_response = call_for_response

    def hook(dec, n):
        if st["resp"]:
            st["ids"][-1].append(dec.argmax_id if dec.sampled_id is None else dec.sampled_id)
            return dec
        st["frames"] += 1
        return _force(model.config, dec, st["frames"] - 1 in SPEAK)
    li.decision_hook = hook
    return li, st


def _frames(cfg, n=12, seed=77):
    g = torch.Generator().manual_seed(seed)
    return [(i / 2, torch.randn(10, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()) for i in range(n)]


def _drain(li, stop_after=None):
    trace = []
    while li.frame_embeds_queue:
        q, r = li()
        if q or r:
            trace.append((q, r, li.last_ids.reshape(-1).tolist(), li._kv.engine.kv_len(li._kv.stream_id)))
            if stop_after is not None and len(trace) == stop_after:
                break
    return trace


@pytest.mark.parametrize("si", [1, 2])
def test_liveinfer_sampled_with_drafts_equals_one_token_per_step(built, tiny, si):
    """LiveInfer's trace, response ids, consumed decisions and cache: the same with the default n-gram drafter and with
    drafts of the right response as with one token per step (no drafter)"""
    cfg = tiny[0]
    model = built[0]
    runs = []
    for drafter in (None, "default", "perfect"):
        li, st = _live(built, SAMPLING[si])
        if drafter is None:
            li.drafter = None
        elif drafter == "perfect":
            want = runs[0][3]
            li.drafter = Scripted(lambda n: want[len(st["ids"]) - 1][len(st["ids"][-1]):] if st["resp"] else [])
        li.query_queue.append((0.0, "narrate"))
        li.frame_embeds_queue.extend(_frames(cfg))
        tr = _drain(li)
        runs.append((tr, li._n_calls, _kv_all(model.engine, li._kv.stream_id), st["ids"]))
        model.engine.stream_close(li._kv.stream_id)
    assert len(runs[0][3]) >= 3 and len({t for r in runs[0][3] for t in r}) > 5
    for r in runs[1:]:
        assert r[0] == runs[0][0] and r[1] == runs[0][1] and r[3] == runs[0][3]
        assert _same_kv(r[2], runs[0][2])


def test_liveinfer_suspend_resume_continues_sampled_ids(built, tiny):
    """suspended through torch.save after its second output, a sampled session resumed in a fresh LiveInfer (whose own
    sampling is greedy: the state brings the config) continues with the ids of the uninterrupted run"""
    cfg = tiny[0]
    model = built[0]
    li, st = _live(built, SAMPLING[2])
    li.query_queue.append((0.0, "narrate"))
    li.frame_embeds_queue.extend(_frames(cfg))
    want = _drain(li)
    kv_want = _kv_all(model.engine, li._kv.stream_id)
    model.engine.stream_close(li._kv.stream_id)
    assert len(want) >= 3

    li, st = _live(built, SAMPLING[2])
    li.query_queue.append((0.0, "narrate"))
    li.frame_embeds_queue.extend(_frames(cfg))
    got = _drain(li, stop_after=2)
    assert li.frame_embeds_queue
    buf = io.BytesIO()
    torch.save(li.suspend(), buf)
    model.engine.stream_close(li._kv.stream_id)
    buf.seek(0)
    li2, st2 = _live(built, None)
    st2["frames"] = st["frames"]
    li2.resume(torch.load(buf))
    assert li2.sampling == li.sampling
    got += _drain(li2)
    assert got == want
    assert _same_kv(_kv_all(model.engine, li2._kv.stream_id), kv_want)
    model.engine.stream_close(li2._kv.stream_id)


def test_scheduler_mixed_sampling_equals_independent_liveinfer(built, tiny, golden):
    """a greedy and two sampled sessions (own configs), stepped together with one sampling launch per tick, give the
    responses and KV lengths of separate LiveInfer sessions"""
    from videollm_online_b200.config import SamplingConfig, SYSTEM_PROMPT
    from videollm_online_b200.multistream import StreamScheduler
    cfg = tiny[0]
    model, tok = built
    confs = [None, SAMPLING[1], SAMPLING[3]]
    videos = [torch.cat([golden["sm_video"]] * 2)[i:i + 8] for i in range(3)]
    refs = []
    for s in range(3):
        li, st = _live(built, confs[s])
        li.load_video(videos[s])
        outs = []
        for i in range(8):
            li.input_video_stream(i / 2)
            q, r = li()
            if r:
                outs.append(r)
        refs.append((outs, li._kv.engine.kv_len(li._kv.stream_id)))
        model.engine.stream_close(li._kv.stream_id)

    sched = StreamScheduler(model, tok, 3, frame_fps=2, system_prompt=SYSTEM_PROMPT)
    frames_seen = [0, 0, 0]

    def hook(s, dec, n):
        sess = sched.sessions[s]
        if sess.state == sess.RESPOND:
            return dec
        frames_seen[s] += 1
        return _force(cfg, dec, frames_seen[s] - 1 in SPEAK)
    sched.decision_hook = hook
    for s, sess in enumerate(sched.sessions):
        sess.load_video(videos[s])
        sess.sampling = SamplingConfig(do_sample=True, **confs[s]) if confs[s] else None
    for i in range(8):
        for sess in sched.sessions:
            sess.input_video_stream(i / 2)
        sched.run_until_idle()
    for s, sess in enumerate(sched.sessions):
        assert [o[2] for o in sess.outputs] == refs[s][0], s
        assert model.engine.kv_len(sess.stream_id) == refs[s][1]
        model.engine.stream_close(sess.stream_id)
    assert all(len(r[0]) == 2 for r in refs)
    assert refs[1][0] != refs[0][0] and refs[2][0] != refs[1][0]
