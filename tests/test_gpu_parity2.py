"""GPU parity, part 2 (round 2): what the tiny goldens and the 2-layer full-width test did not cover.

  * the query path end to end (demo/cli.py:23 -> demo/inference.py:42, 57-59, 72-74, 93-100) through LiveInfer,
    StreamScheduler and cli.main, against the trace of the reference's own methods (tests/golden: smq_*);
  * joint_embed / forward(input_ids, frames) (models/modeling_live.py:29-42);
  * the FULL 32-layer Llama-3-8B-width stack at a 12k-token cache against the oracle (bf16 error compounding over 64
    residual adds), logits + greedy id;
  * a full-width RAGGED batch (8 streams, mixed q = 11 / 1 / 17, mixed cache lengths up to 12k: the BN = 128 stream-K
    plan, multi-item split-KV) and a q = 1 step at 12k against the oracle;
  * merged-LoRA engine logits against the UNMERGED LoRA forward of the reference (models/modeling_live.py:203-216);
  * the KV-append attention at 66k keys (BASELINE.json configs[3]: 10 FPS x 10 min) against an fp32 SDPA restatement.

Observed errors are printed (visible with -s) and, when VLO_PARITY_LOG names a file, appended to it as JSON lines, so drift
stays visible.
Tolerances: see test_gpu_parity.py (LOGIT_ATOL + LOGIT_RTOL*|x|); where a test loosens them it says why."""
import dataclasses
import json
import math
import os
import pathlib
import sys

import pytest
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "oracle"))
sys.path.insert(0, str(ROOT / "tests" / "golden"))

pytestmark = pytest.mark.gpu

LOGIT_ATOL, LOGIT_RTOL = 0.25, 0.02
EMBED_ATOL = 6e-2


def _report(name, **vals):
    rec = {"test": name, **{k: (float(v) if isinstance(v, (int, float)) else v) for k, v in vals.items()}}
    log = os.environ.get("VLO_PARITY_LOG")
    if log:
        with open(log, "a") as f:
            f.write(json.dumps(rec) + "\n")
    print("PARITY", json.dumps(rec))


def _close(a, b, atol, rtol):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs()
    bad = err > atol + rtol * b.abs()
    return float(err.max()), float(bad.float().mean())


def _rms_rel(a, b):
    """rms error over the standard deviation of the reference (scale-free; 1 bf16 ulp of rounding alone is ~0.2 %)"""
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).pow(2).mean().sqrt() / b.std().clamp_min(1e-12))


@pytest.fixture(scope="module")
def built(tiny):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = tiny
    model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                            max_streams=4, max_kv_tokens=1024, max_step_tokens=128, max_vit_batch=4)
    return model, tok


def _force(cfg, dec, t):
    if t is not None:
        dec.argmax_id = dec.argmax_prob_id = t
        dec.p_interval = 1.0 if t == cfg.frame_token_interval_id else 0.0
        if t != cfg.frame_token_interval_id:
            dec.argmax_excl_id = t
    return dec


# ------------------------------------------------------------------------------------------- query path
def test_query_path_liveinfer_vs_reference(built, golden, tiny):
    """LiveInfer over the engine, narration request at t=0 (rule 2) + a mid-stream query (rule 1): same (iteration,
    query string, last id, KV length) trace and the same number of forwards as the reference's LiveInfer methods."""
    import make_golden as MG
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    cfg, _, _ = tiny
    model, tok = built
    sched = MG.query_schedule(cfg)
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    li.decision_hook = lambda dec, call: _force(cfg, dec, sched.get(call))
    li.load_video(golden["sm_video"])
    trace, notes = [], []
    for i in range(8):
        if i == 0:
            notes.append(li.input_query_stream(MG.QUERY_0, video_time=0.0))
        if i == MG.QUERY_MID_BEFORE_ITER:
            notes.append(li.input_query_stream(MG.QUERY_MID, video_time=MG.QUERY_MID_AT))
        li.input_video_stream(i / 2)
        query, response = li()
        trace.append((i, query, response, int(li.last_ids.reshape(-1)[-1]), li.past_key_values.get_seq_length()))
    ref = golden["smq_trace"]
    assert [(t[0], t[1], t[3], t[4]) for t in trace] == [(t[0], t[1], t[3], t[4]) for t in ref]
    # responses: scripted parts exact (the natural tokens come from near-tied random logits)
    for t, r in zip(trace, ref):
        assert (t[2] is None) == (r[2] is None)
        if r[2] is not None:
            assert t[2].startswith(r[2].split("Assistant:")[0] + "Assistant:")
    assert li._n_calls == golden["smq_calls"]
    assert notes == golden["smq_notes"]
    model.engine.stream_close(li._kv.stream_id)


def test_query_path_scheduler_vs_reference(built, golden, tiny):
    """The multi-stream scheduler runs the same query protocol per stream: stream 0 replays the query golden, stream 1
    runs without queries alongside it (mixed phases in one ragged step) and must match its own LiveInfer trace."""
    import make_golden as MG
    from videollm_online_b200.config import SYSTEM_PROMPT
    from videollm_online_b200.multistream import StreamScheduler
    cfg, _, _ = tiny
    model, tok = built
    scheds = [MG.query_schedule(cfg), MG.golden_schedule(cfg)]
    sch = StreamScheduler(model, tok, 2, frame_fps=2, system_prompt=SYSTEM_PROMPT)
    sch.decision_hook = lambda s, d, n: _force(cfg, d, scheds[s].get(n))
    for sess in sch.sessions:
        sess.load_video(golden["sm_video"])
    for i in range(8):
        if i == 0:
            sch.sessions[0].input_query_stream(MG.QUERY_0, video_time=0.0)
        if i == MG.QUERY_MID_BEFORE_ITER:
            sch.sessions[0].input_query_stream(MG.QUERY_MID, video_time=MG.QUERY_MID_AT)
        for sess in sch.sessions:
            sess.input_video_stream(i / 2)
        sch.run_until_idle()
    # The scheduler is event-driven: after answering a query that pre-empted a frame (rule 1) it goes on with that frame in
    # the same run_until_idle, where the reference's __call__ returns and consumes it on the next call.  Same operations in
    # the same order per stream, so the forwards, the query strings, the frame decisions and the final cache length agree.
    for s, key in enumerate(("smq_trace", "sm_trace")):
        ref = golden[key]
        sess = sch.sessions[s]
        assert model.engine.kv_len(sess.stream_id) == ref[-1][4], (s, model.engine.kv_len(sess.stream_id))
        got_q = [o[1] for o in sess.outputs]
        want_q = [t[1] for t in ref if t[2] is not None]
        assert got_q == want_q, (s, got_q, want_q)
        assert [o[2].split("Assistant:")[0] for o in sess.outputs] == [t[2].split("Assistant:")[0] for t in ref if t[2] is not None]
        assert sess.n_calls == golden["smq_calls" if s == 0 else "sm_calls"]
        n_frames = sum(1 for e in sess.events if e[0] == "frame")
        assert n_frames + (1 if s == 0 else 0) == 8          # stream 0: the t=0 frame's decision is pre-empted by the query (rule 2)
        model.engine.stream_close(sess.stream_id)


def test_cli_main_vs_oracle_liveinfer(built, golden, tiny):
    """cli.main (demo/cli.py:12-50: load clip, narration query at t=0, N x (input_video_stream, __call__)) on the GPU
    against the CPU oracle's LiveInfer driven the same way with the same scripted decisions."""
    import vlo_oracle as O
    import make_golden as MG
    from videollm_online_b200 import cli
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.tokenization_live import ByteTokenizer
    cfg, llm, vis = tiny
    model, tok = built
    I, E, END = cfg.frame_token_interval_id, cfg.eos_token_id, cfg.stream_end_id
    sched = {0: I, 3: E, 4: I, 5: I, 6: END, 8: E, 9: I, 10: I, 11: END, 12: E, 13: I}
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    li.decision_hook = lambda dec, call: _force(cfg, dec, sched.get(call))
    fps, history = cli.main(li, video=golden["sm_video"], n_iters=8, quiet=True)
    assert fps > 0
    calls = [0]

    def hook(logits, kind):
        t = sched.get(calls[0])
        calls[0] += 1
        if t is not None:
            logits = logits.clone()
            logits[t] += 1000.0
        return logits

    ol = O.OracleLiveInfer(llm, vis, cfg, ByteTokenizer(cfg), frame_fps=2, system_prompt=SYSTEM_PROMPT, logit_hook=hook)
    ol.load_video(golden["sm_video"])
    ol.input_query_stream(MG.QUERY_0, video_time=0.0)
    want = []
    for i in range(8):
        ol.input_video_stream(i / 2)
        q, r = ol()
        if q:
            want.append(("user", q, i / 2))
        if r:
            want.append(("assistant", r.split("Assistant:")[0] + "Assistant:", i / 2))
        if not q and not r:
            want.append((None, None, i / 2))
    got = []
    for e in history["conversation"]:
        role = e.get("role")
        content = e.get("content")
        if role == "assistant":
            content = content.split("Assistant:")[0] + "Assistant:"
        got.append((role, content, e["time"]))
    assert got == want
    assert li._n_calls == calls[0] and li.past_key_values.get_seq_length() == ol.cache.get_seq_length()
    model.engine.stream_close(li._kv.stream_id)


# ------------------------------------------------------------------------------------------- joint_embed
def test_joint_embed_and_forward_with_ids_and_frames(built, golden, tiny):
    cfg, _, _ = tiny
    model, _ = built
    ids = golden["joint_ids"]
    emb = model.joint_embed(ids.cuda(), golden["frames"][:2].cuda())
    ref = golden["joint_embed"]
    assert tuple(emb.shape) == tuple(ref.shape) and emb.dtype == torch.bfloat16
    is_v = (ids[0] == cfg.v_placeholder_id)
    assert torch.equal(emb[0].cpu()[~is_v], ref[0][~is_v])                      # token rows: exact gather
    mx, frac = _close(emb[0].cpu()[is_v], ref[0][is_v], EMBED_ATOL, 3e-2)
    assert frac == 0.0, mx
    # ids only / frames only
    assert torch.equal(model.joint_embed(input_ids=ids[:, :2].cuda()).cpu(), ref[:, :2])
    only_f = model.joint_embed(frames=golden["frames"][:2].cuda())
    assert _close(only_f, golden["visual_embed"][:2 * cfg.frame_num_tokens], EMBED_ATOL, 3e-2)[1] == 0.0
    # forward(input_ids, frames): all-position logits of the step against the reference's
    out = model(input_ids=ids.cuda(), frames=golden["frames"][:2].cuda(), use_cache=True)
    allpos = model.engine.last_step_logits(ids.shape[1])
    mx, frac = _close(allpos, golden["joint_logits"], LOGIT_ATOL, LOGIT_RTOL)
    _report("joint_forward", max_err=mx, outliers=frac)
    assert frac == 0.0, mx
    assert _close(out.logits[0, 0], golden["joint_logits"][-1], LOGIT_ATOL, LOGIT_RTOL)[1] == 0.0


# ------------------------------------------------------------------------------------------- full width
def _cycled_llm_state(cfg, n_distinct, seed):
    """Full-depth state dict whose layers cycle through `n_distinct` independently drawn layers (host memory stays
    at n_distinct x 436 MB; the arithmetic and the error compounding over depth are those of distinct layers)."""
    from videollm_online_b200 import weights as W
    small = dataclasses.replace(cfg, num_hidden_layers=n_distinct)
    sd = W.synthetic_llm_state(small, seed=seed)
    for i in range(n_distinct, cfg.num_hidden_layers):
        src = f"model.layers.{i % n_distinct}."
        for k in [k for k in sd if k.startswith(src)]:
            sd[f"model.layers.{i}." + k[len(src):]] = sd[k]
    sd["lm_head.weight"] = (sd["lm_head.weight"].float() * 8).to(torch.bfloat16)
    return sd


def _oracle_cache_from_engine(eng, sid, n_layers):
    import vlo_oracle as O
    cache = O.KVCache(n_layers)
    for layer in range(n_layers):
        cache.update(layer, eng.kv_read(sid, layer, False).cpu()[None], eng.kv_read(sid, layer, True).cpu()[None])
    return cache


def test_full_depth_32_layers_at_12k_context():
    """One frame step (q = 11) of the FULL Llama-3-8B stack (32 layers, full width, 128 256-row lm_head) on a
    12 000-token cache against the oracle.  bf16 rounding differences (fp32 accumulation order only) compound over 64
    residual adds, so the tolerance is the 2-layer one with a wider outlier allowance; the observed numbers are
    reported.  Greedy id must agree whenever the oracle's top-1 margin exceeds twice the observed max error."""
    import vlo_oracle as O
    from videollm_online_b200 import llama3_8b_siglip_l
    from videollm_online_b200.modeling_live import build_live
    cfg = llama3_8b_siglip_l()
    llm = _cycled_llm_state(cfg, 4, seed=13)
    N, q = 12000, 11
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=1,
                          max_kv_tokens=N + 256, max_step_tokens=128, max_vit_batch=1)
    eng = model.engine
    kv = model.new_stream()
    eng.kv_fill_synthetic(kv.stream_id, N, seed=21)
    cache = _oracle_cache_from_engine(eng, kv.stream_id, cfg.num_hidden_layers)
    g = torch.Generator().manual_seed(17)
    emb = (torch.randn(q, cfg.hidden_size, generator=g) * 0.5).to(torch.bfloat16)
    out = model(inputs_embeds=emb[None].cuda(), past_key_values=kv, use_cache=True)
    allpos = eng.last_step_logits(q)
    dec = eng.read_decisions(1)[0]
    ref = O.llama_forward(llm, cfg, emb, cache)
    assert kv.get_seq_length() == N + q == cache.get_seq_length()
    mx, frac = _close(allpos, ref, LOGIT_ATOL, LOGIT_RTOL)
    mx_last, frac_last = _close(out.logits[0, 0], ref[-1], LOGIT_ATOL, LOGIT_RTOL)
    top2 = ref[-1].float().topk(2).values
    margin = float(top2[0] - top2[1])
    diff = allpos.float().cpu() - ref.float()
    ref_std = float(ref.float().std())
    rms_rel = float(diff.pow(2).mean().sqrt()) / ref_std
    corr = float(torch.corrcoef(torch.stack([allpos.float().cpu().flatten(), ref.float().flatten()]))[0, 1])
    agree = float((allpos.float().cpu().argmax(-1) == ref.float().argmax(-1)).float().mean())
    _report("full_depth_32_layers_12k", max_err=mx, outliers_2layer_tol=frac, max_err_last=mx_last, rms_err_over_std=rms_rel,
            correlation=corr, ref_abs_max=float(ref.float().abs().max()), ref_std=ref_std, top1_margin=margin,
            argmax_rows_agreeing=agree)
    # Tolerance at FULL DEPTH.  Engine and oracle round to bf16 at the same points; what differs is the fp32 summation
    # order inside each GEMM / attention, i.e. an occasional 1-ulp (2^-8 relative) difference per Linear output.  Through
    # 32 layers x 7 Linears of random weights (which do not damp perturbations) these walk to a few percent of the hidden
    # state: observed rms error 3 % of the logit std (max 1.5 at std 10.3), versus 0.3 % for the 2-layer stack of
    # test_full_width_layers_at_12k_context, which keeps the per-layer tolerance.  Bounds: rms <= 6 % of the logit std,
    # max <= 25 % of it, correlation >= 0.995, and the greedy id must agree whenever the oracle's margin exceeds twice the
    # observed max error.
    assert rms_rel < 0.06 and mx < 0.25 * ref_std and corr > 0.995, f"rms/std {rms_rel}, max {mx}, corr {corr}"
    if margin > 2 * mx_last:
        assert dec.argmax_id == int(ref[-1].float().argmax())
    # the rows appended by the LAST layer (input = 31 layers of compounded hidden state)
    # (same compounding as the logits: bounded the same way, rms <= 6 % of the std of the reference rows)
    L = cfg.num_hidden_layers - 1
    k_new, v_new = eng.kv_read(kv.stream_id, L, False)[:, N:], eng.kv_read(kv.stream_id, L, True)[:, N:]
    k_rms, v_rms = _rms_rel(k_new, cache.k[L][0, :, N:]), _rms_rel(v_new, cache.v[L][0, :, N:])
    k_out = _close(k_new, cache.k[L][0, :, N:], 8e-2, 4e-2)[1]
    v_out = _close(v_new, cache.v[L][0, :, N:], 8e-2, 4e-2)[1]
    # layer 0 rows see no compounding: the per-layer tolerance holds there
    k0_out = _close(eng.kv_read(kv.stream_id, 0, False)[:, N:], cache.k[0][0, :, N:], 4e-2, 2e-2)[1]
    _report("full_depth_32_layers_12k_kv_rows", k_rms_over_std=k_rms, v_rms_over_std=v_rms, k_outliers=k_out,
            v_outliers=v_out, k_layer0_outliers=k0_out)
    assert k0_out == 0.0
    assert k_rms < 0.06 and v_rms < 0.06 and k_out < 2e-2 and v_out < 2e-2, (k_rms, v_rms, k_out, v_out)
    eng.stream_close(kv.stream_id)


def test_full_width_ragged_batch_and_ar_step_vs_oracle():
    """Full-width layers (2-layer stack), 8 concurrent streams in ONE ragged step: q = 11 x5, 1 (AR token at 12k), 17
    (response prompt), 11, cache lengths 12 000 / 6 000 / 300 / ... -> T = 84 (BN = 128 stream-K plan, 8 attention work
    items with uneven split budgets); then a q = 1 step of the 12k stream alone.  Each stream against the oracle."""
    import vlo_oracle as O
    from videollm_online_b200 import llama3_8b_siglip_l, weights as W
    from videollm_online_b200.modeling_live import build_live
    cfg = llama3_8b_siglip_l()
    cfg.num_hidden_layers = 2
    llm = W.synthetic_llm_state(cfg, seed=5)
    llm["lm_head.weight"] = (llm["lm_head.weight"].float() * 8).to(torch.bfloat16)
    kv_lens = [12000, 6000, 300, 12000, 2049, 64, 9000, 1]
    q_lens = [11, 11, 11, 1, 17, 11, 11, 11]
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=8,
                          max_kv_tokens=12000 + 256, max_step_tokens=128, max_vit_batch=1)
    eng = model.engine
    sids = [eng.stream_open() for _ in kv_lens]
    g = torch.Generator().manual_seed(23)
    caches = []
    for s, n in zip(sids, kv_lens):
        eng.kv_fill_synthetic(s, n, seed=100 + s)
        caches.append(_oracle_cache_from_engine(eng, s, cfg.num_hidden_layers))
    embs = [(torch.randn(q, cfg.hidden_size, generator=g) * 0.5).to(torch.bfloat16) for q in q_lens]
    logits, _ = eng.step(sids, q_lens, torch.cat(embs, 0).cuda())
    decs = eng.read_decisions(len(sids))
    # Per-stream statistics first (all reported), then the bounds.  The short-context streams carry the largest error:
    # with few keys the attention output is not averaged down (|o| ~ 1/sqrt(n_keys)), so it is a larger share of the
    # residual stream and its bf16 roundings weigh more in the logits.  Bounds per stream: rms error <= 1.5 % of the
    # logit std, at most 2e-3 of the 128 256 logits outside LOGIT_ATOL + LOGIT_RTOL |x|, none beyond twice that.
    stats, fails = [], []
    for i, (e, c) in enumerate(zip(embs, caches)):
        ref = O.llama_forward(llm, cfg, e, c)[-1]
        mx, frac = _close(logits[i], ref, LOGIT_ATOL, LOGIT_RTOL)
        frac2 = _close(logits[i], ref, 2 * LOGIT_ATOL, 2 * LOGIT_RTOL)[1]
        rr = _rms_rel(logits[i], ref)
        top2 = ref.float().topk(2).values
        id_ok = decs[i].argmax_id == int(ref.float().argmax()) or float(top2[0] - top2[1]) <= 2 * LOGIT_ATOL
        stats.append({"kv": kv_lens[i], "q": q_lens[i], "max_err": round(mx, 4), "outliers": frac, "rms_over_std": round(rr, 5)})
        if not (rr < 0.015 and frac < 2e-3 and frac2 == 0.0 and id_ok):
            fails.append(i)
        assert eng.kv_len(sids[i]) == kv_lens[i] + q_lens[i] == c.get_seq_length()
    _report("full_width_ragged_8_streams", streams=stats)
    assert not fails, [stats[i] for i in fails]
    # appended rows of the 17-token stream (crosses a 128-key block boundary at 2049..2065)
    for layer in range(cfg.num_hidden_layers):
        k = eng.kv_read(sids[4], layer, False)[:, 2049:]
        assert _close(k, caches[4].k[layer][0, :, 2049:], 4e-2, 2e-2)[1] == 0.0
    # q = 1 AR step of the 12k stream alone (N = 16-token tile with one live column, 18-way split-KV)
    one = (torch.randn(1, cfg.hidden_size, generator=g) * 0.5).to(torch.bfloat16)
    lg, _ = eng.step([sids[0]], [1], one.cuda())
    ref = O.llama_forward(llm, cfg, one, caches[0])[-1]
    mx, frac = _close(lg[0], ref, LOGIT_ATOL, LOGIT_RTOL)
    rr = _rms_rel(lg[0], ref)
    _report("full_width_q1_at_12k", max_err=mx, outliers=frac, rms_over_std=rr)
    assert rr < 0.015 and frac < 2e-3 and _close(lg[0], ref, 2 * LOGIT_ATOL, 2 * LOGIT_RTOL)[1] == 0.0, (mx, frac, rr)
    for s in sids:
        eng.stream_close(s)


# ------------------------------------------------------------------------------------------- LoRA
def test_merged_lora_vs_unmerged_reference_forward(tiny):
    """The reference keeps the PEFT adapter UNMERGED at inference (models/modeling_live.py:203-216: every wrapped Linear
    computes W x + (alpha/r) * B(A(x)), bf16 ops, scaling 256/128 = 2.0); the engine merges W' = W + 2 B A at load
    (weights.merge_lora, fp32 product, one bf16 rounding).  Same logits within the bf16 tolerance, same greedy id."""
    import vlo_oracle as O
    from videollm_online_b200 import weights as W
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, _ = tiny
    g = torch.Generator().manual_seed(31)
    r, alpha = 16, 32
    adapter = {}
    names = ["self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj",
             "mlp.down_proj"]
    targets = [f"model.layers.{i}.{n}" for i in range(cfg.num_hidden_layers) for n in names] + ["lm_head"]
    for t in targets:
        out_f, in_f = llm[t + ".weight"].shape
        adapter[f"base_model.model.{t}.lora_A.default.weight"] = (torch.randn(r, in_f, generator=g) * 0.05).to(torch.bfloat16)
        adapter[f"base_model.model.{t}.lora_B.default.weight"] = (torch.randn(out_f, r, generator=g) * 0.05).to(torch.bfloat16)
    merged = W.merge_lora(llm, adapter, lora_alpha=alpha, lora_r=r)
    model, _ = build_live(config=cfg, llm_state=merged, set_vision_inside=False, device="cuda:0", max_streams=1,
                          max_kv_tokens=256, max_step_tokens=64, max_vit_batch=1)
    emb = (torch.randn(29, cfg.hidden_size, generator=g)).to(torch.bfloat16)
    out = model(inputs_embeds=emb[None].cuda(), past_key_values=None, use_cache=True)
    allpos = model.engine.last_step_logits(29)
    ref = O.llama_forward(llm, cfg, emb, O.KVCache(cfg.num_hidden_layers), lora=O.LoraAdapter(adapter, alpha / r))
    base = O.llama_forward(llm, cfg, emb, O.KVCache(cfg.num_hidden_layers))
    mx, frac = _close(allpos, ref, LOGIT_ATOL, LOGIT_RTOL)
    moved = float((ref.float() - base.float()).abs().max())
    _report("merged_lora_vs_unmerged", max_err=mx, outliers=frac, adapter_effect_max=moved)
    assert moved > 4 * LOGIT_ATOL, "the synthetic adapter must move the logits well beyond the tolerance"
    assert frac < 1e-3 and mx < 3 * LOGIT_ATOL, f"merged-LoRA logits differ from the unmerged forward by {mx}, outliers {frac}"
    top2 = ref[-1].float().topk(2).values
    if float(top2[0] - top2[1]) > 2 * LOGIT_ATOL:
        assert int(out.logits[0, 0].float().argmax()) == int(ref[-1].float().argmax())


# ------------------------------------------------------------------------------------------- 66k keys
def test_attention_at_66k_keys_vs_sdpa():
    """BASELINE.json configs[3] (10 FPS x 10 min ~ 66k-token cache): the KV-append attention kernel at 66 011 keys
    (516 key blocks, row indices past 2^19 per head) against the fp64 reference within the bound of attn_reference.py,
    q = 11 and q = 1."""
    from attn_reference import DECODER, decoder_chain, reference
    from videollm_online_b200 import _lib
    lib = _lib.load()
    dev = "cuda"
    torch.manual_seed(3)
    H, Hk, D = 32, 8, 128
    kv_len = 66011
    stride = 66048 + 128
    k = torch.randn(Hk, stride, D, device=dev).bfloat16()
    v = torch.randn(Hk, stride, D, device=dev).bfloat16()
    for n_tok in (11, 1):
        q = torch.randn(n_tok, H, D, device=dev).bfloat16()
        out = torch.empty(n_tok, H * D, device=dev, dtype=torch.bfloat16)
        ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, H, D, kv_len), device=dev, dtype=torch.uint8)
        rc = lib.vlo_op_attn_kvappend(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), ws.data_ptr(), n_tok, H, Hk, D,
                                      kv_len, stride, torch.cuda.current_stream().cuda_stream)
        assert rc == 0, lib.vlo_last_error()
        torch.cuda.synchronize()
        res = reference(q, k[:, :kv_len], v[:, :kv_len], torch.arange(kv_len - n_tok, kv_len), DECODER,
                        decoder_chain(kv_len, torch.cuda.get_device_properties(0).multi_processor_count))
        err = float((out.view(n_tok, H, D).double() - res.ref).abs().max())
        ex = res.excess(out.view(n_tok, H, D))
        _report("attn_66k_keys", n_tok=n_tok, max_err=err, bound_excess=ex)
        assert ex <= 0 and bool(torch.isfinite(out.float()).all()), (err, ex)


# ------------------------------------------------------------------------------------------- stream_evaluate
def test_stream_evaluate_vs_reference(golden, tiny):
    """SURVEY 8(f) row 4: stream_evaluate on the engine's cache (teacher-forced chunks through vlo_step_ids +
    vlo_last_step_logits, look-ahead on a vlo_kv_copy_prefix scratch stream) against the reference's own method.
    Integer-valued metrics (frame_diff, fluency, lm_correctness) must agree exactly; perplexity is exp(mean CE) of
    random weights (~e^50), compared in log space within the logit tolerance."""
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = tiny
    sd = dict(llm)
    w = sd["lm_head.weight"].clone()
    w[cfg.frame_token_interval_id] = golden["se_lm_head_row"]
    sd["lm_head.weight"] = w
    model, _ = build_live(config=cfg, llm_state=sd, vision_state=vis, set_vision_inside=True, device="cuda:0",
                          max_streams=2, max_kv_tokens=256, max_step_tokens=32, max_vit_batch=4)   # 91 tokens -> 3 chunks
    for thr in (0.0, 0.9):
        got = model.stream_evaluate(golden["se_ids"].cuda(), golden["se_labels"].cuda(), golden["se_frames"].cuda(),
                                    frame_token_interval_threshold=thr).cpu()
        ref = golden[f"se_metrics_thr{thr}"].float()
        _report("stream_evaluate", thr=thr, log_ppl=float(got[0].log()), log_ppl_ref=float(ref[0].log()),
                frame_diff=float(got[1]), fluency=float(got[2]), lm_correctness=float(got[3]))
        assert torch.equal(got[1:], ref[1:]), (got, ref)
        assert abs(float(got[0].log()) - float(ref[0].log())) < LOGIT_ATOL, (got, ref)
    # pre-extracted features instead of raw frames (the evaluation path of the reference: data/stream.py:90-91)
    feats = golden["vit_tokens"]          # [4, 10, C] of golden["frames"]; just exercise the connector-only route
    assert model.visual_embed(feats.cuda()).shape[0] == 4 * cfg.frame_num_tokens


# ------------------------------------------------------------------------------------------- f2 / f3 on the GPU
def _write_clip(cv2, np, path, n, size, fps, seed):
    w = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"MJPG"), fps, size)
    if not w.isOpened():
        pytest.skip("no MJPG encoder in this OpenCV build")
    rng = np.random.default_rng(seed)
    for i in range(n):
        f = rng.integers(0, 256, (size[1], size[0], 3), dtype=np.uint8)
        f[:, : size[0] // 2] = (i * 9) % 256          # large flat areas survive the JPEG round trip
        w.write(f)
    w.release()


def test_cli_on_a_video_file(built, tiny, tmp_path):
    """SURVEY 8(f).2: demo/cli.py's flow on a clip ON DISK (decode -> 2 FPS resample -> letterbox, data/utils.py:51-66 +
    demo/inference.py:111-115) feeding the engine: `cli.main(LiveInfer, video=<path>)`.  The frame embeddings the
    state machine consumed must equal the oracle's on the frames the ingest produced."""
    cv2 = pytest.importorskip("cv2")
    import numpy as np
    import vlo_oracle as O
    from videollm_online_b200 import cli
    from videollm_online_b200.config import LiveArguments, SYSTEM_PROMPT
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.video_ingest import read_video_resampled
    cfg, llm, vis = tiny
    model, tok = built
    path = tmp_path / "clip.avi"
    _write_clip(cv2, np, path, 90, (160, 90), 30.0, seed=3)          # 3 s of 16:9 video at 30 fps -> 6 frames at 2 FPS
    li = LiveInfer(LiveArguments(frame_fps=2, system_prompt=SYSTEM_PROMPT), model=model, tokenizer=tok)
    I, E = cfg.frame_token_interval_id, cfg.eos_token_id
    sched = {0: I, 1: E}                                             # narration query answered with an immediate EOS
    li.decision_hook = lambda dec, call: _force(cfg, dec, sched.get(call, I))
    fps, history = cli.main(li, video=str(path), n_iters=6, quiet=True)
    assert li.num_video_frames == 6 and tuple(li.video_tensor.shape) == (6, 3, cfg.frame_resolution, cfg.frame_resolution)
    assert fps > 0 and len(history["conversation"]) == 7             # query + response at t=0, then 5 silent frames
    assert history["conversation"][0]["role"] == "user" and history["conversation"][1]["role"] == "assistant"
    frames = read_video_resampled(str(path), fps=2, resolution=cfg.frame_resolution)
    assert torch.equal(frames, li.video_tensor.cpu())
    assert int(frames[:, :, :20].max()) == 0                         # letterbox bars of the 16:9 source
    ref = O.visual_embed(llm, vis, cfg, frames)
    got = model.visual_embed(li.video_tensor)
    assert _close(got, ref, EMBED_ATOL, 3e-2)[1] == 0.0
    # KV accounting: start prompt + 11 + query prompt + 1 (EOS) + 5 x (stream prompt / interval + 10)
    assert li.past_key_values.get_seq_length() > 6 * 11
    model.engine.stream_close(li._kv.stream_id)


def test_offline_encode_directory_on_the_engine(built, tiny, tmp_path):
    """SURVEY 8(f).3: distributed_encode's host loop (data/utils.py:86-104) with `build_live_vision(config, engine)` as
    the encoder: batches larger than the engine's max_vit_batch are chunked, the saved bf16 features equal the oracle's
    SigLIP tokens (models/vision_live.py:10-30) of the decoded frames."""
    cv2 = pytest.importorskip("cv2")
    import numpy as np
    import vlo_oracle as O
    from videollm_online_b200.offline_encode import encode_directory, encoded_root
    from videollm_online_b200.vision_live import build_live_vision
    from videollm_online_b200.video_ingest import read_video_resampled
    cfg, _, vis = tiny
    model, _ = built
    R = cfg.frame_resolution
    src = tmp_path / "clips_2fps_384"
    src.mkdir()
    for k, (name, n) in enumerate({"a.avi": 11, "b.avi": 3}.items()):
        _write_clip(cv2, np, src / name, n, (R, R), 2.0, seed=10 + k)
    enc, fn = build_live_vision(cfg, model.engine)
    written = encode_directory(src_root=str(src) + "/", vision_pretrained="google/siglip-large-patch16-384", vision_encode=fn,
                               encoder=enc, batch_size=256, embed_mark="2fps_384_1+3x3", save_bf16=True, device="cuda:0")
    assert [pathlib.Path(p).name for p in written] == ["a.pt", "b.pt"]
    dst = encoded_root(str(src), "2fps_384_1+3x3", "google/siglip-large-patch16-384")
    for name, n in (("a", 11), ("b", 3)):
        feats = torch.load(pathlib.Path(dst) / f"{name}.pt")
        assert feats.dtype == torch.bfloat16 and tuple(feats.shape) == (n, cfg.frame_num_tokens, cfg.vision_hidden_size)
        ref = O.siglip_vision_encode(vis, cfg, read_video_resampled(str(src / f"{name}.avi")))
        mx, frac = _close(feats, ref, 3e-2 + 8e-3, 2e-2)             # VIT_ATOL + one bf16 ulp of O(1) tokens
        assert frac == 0.0, (name, mx)

