"""Seeded scenarios whose outputs must not depend on programmatic dependent launch (PDL).

`scenarios()` runs every kernel path the engine launches with PDL on fresh engines and returns the outputs by name.
tests/test_gpu_ordering.py runs it in its own process with PDL on and, through this script, in a child process with
VLO_NO_PDL=1 (read once per process), then compares the two bit for bit:

    VLO_NO_PDL=1 python tests/ordering_child.py OUT.pt
"""
import pathlib
import sys

import torch

HERE = pathlib.Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))
import vlo_bootstrap  # noqa: E402,F401  registers `videollm_online_b200`

IID = 11
FORMS = ["bf16", "fp8", "w8a8"]
VIT_BATCHES = [1, 2, 3, 8, 11]


def tiny_state():
    """the suite's `tiny` fixture"""
    from videollm_online_b200 import tiny_config
    from videollm_online_b200 import weights as W
    cfg = tiny_config()
    llm = W.synthetic_llm_state(cfg, seed=0)
    llm["lm_head.weight"] = (llm["lm_head.weight"].float() * 8).to(torch.bfloat16)
    return cfg, llm, W.synthetic_vision_state(cfg, seed=1)


def _emb(H, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, H, generator=g).to(torch.bfloat16).cuda()


def _kv(out, name, eng, sid):
    for l in range(eng.cfg.num_hidden_layers):
        out[f"{name}.L{l}.k"] = eng.kv_read(sid, l, False).clone()
        out[f"{name}.L{l}.v"] = eng.kv_read(sid, l, True).clone()


def _step(out, name, eng, sids, q_lens, emb, **kw):
    logits, dec = eng.step(sids, q_lens, emb, interval_id=IID, **kw)
    out[f"{name}.logits"] = logits.clone()
    out[f"{name}.dec"] = dec.clone()


def _tiny_model(tiny, form, **kw):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, vis = tiny
    model, _ = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                          max_streams=4, max_kv_tokens=512, max_step_tokens=128, max_vit_batch=2,
                          fp8_weights=form != "bf16", fp8_activations=form == "w8a8", **kw)
    return model.engine


def step_forms(tiny, form):
    """one sequence on a fragmented page pool: T = 1, 11, 128, then segments [1, 10, 1, 10]; every layer's K/V"""
    out = {}
    eng = _tiny_model(tiny, form)
    H = eng.cfg.hidden_size
    a, b = eng.stream_open(), eng.stream_open()
    for n in (64, 128):        # grown in turns, then one closed: the next stream's pages are not contiguous
        for s in (a, b):
            eng.kv_fill_synthetic(s, n, seed=n + s)
    eng.stream_close(a)
    sid = eng.stream_open()
    eng.kv_fill_synthetic(sid, 60, seed=3)
    for T in (1, 11, 128):
        _step(out, f"{form}.T{T}", eng, [sid], [T], _emb(H, T, T))
    _step(out, f"{form}.segs", eng, [sid], [22], _emb(H, 22, 22), segments=[[1, 10, 1, 10]])
    _kv(out, f"{form}.kv", eng, sid)
    eng.close()
    return out


def step_full_width(form):
    """a 2-layer stack at Llama-3-8B width: T = 1, 11, 128"""
    from test_gpu_decoder_step import _Engines
    engines = _Engines()
    out = {}
    try:
        cfg, eng = engines.get("full", form)
        sid = eng.stream_open()
        eng.kv_fill_synthetic(sid, 70, seed=4)
        for T in (1, 11, 128):
            _step(out, f"full.{form}.T{T}", eng, [sid], [T], _emb(cfg.hidden_size, T, 100 + T))
        _kv(out, f"full.{form}.kv", eng, sid)
    finally:
        engines.close()
    return out


def ragged_sampled_kv_ops(tiny):
    """a ragged 3-stream step, a sampled step, then kv_evict, kv_compact and a swap round trip, each followed by a step"""
    from videollm_online_b200.engine import SampleRow
    out = {}
    eng = _tiny_model(tiny, "bf16")
    H = eng.cfg.hidden_size
    s = [eng.stream_open() for _ in range(3)]
    for i, n in enumerate((5, 130, 300)):
        eng.kv_fill_synthetic(s[i], n, seed=10 + i)
    ids = torch.tensor([IID] + [-1] * 11 + [300] + [-1] * 10 + [301, 302] + [-1] * 27, dtype=torch.int64, device="cuda")
    _step(out, "ragged", eng, s, [12, 11, 29], _emb(H, 52, 5), row_ids=ids)
    row = SampleRow(seed=7, position=eng.kv_len(s[0]), temperature=0.8, top_k=20, top_p=0.9, repetition_penalty=1.2,
                    penalty_ids=[3, 300, 301, 500])
    _step(out, "sampled", eng, [s[0]], [3], _emb(H, 3, 6), sample=[row])
    out["sampled.id"] = torch.tensor([eng.read_decisions(1)[0].sampled_id])
    eng.kv_evict(s[2], 64, 128)
    _step(out, "evict", eng, [s[2]], [11], _emb(H, 11, 7))
    eng.kv_compact(s[1], [(0, 40), (64, 30), (100, eng.kv_len(s[1]) - 100)])
    _step(out, "compact", eng, [s[1]], [11], _emb(H, 11, 8))
    img = eng.kv_swap_out(s[2])
    eng.stream_close(s[2])
    t = eng.stream_open()
    eng.kv_swap_in(t, img)
    _step(out, "swap", eng, [t], [11], _emb(H, 11, 9))
    for name, sid in (("s0", s[0]), ("s1", s[1]), ("swapped", t)):
        _kv(out, f"ops.{name}", eng, sid)
    eng.close()
    return out


def vit_and_connector():
    """vit_encode at B = 1, 2 (CTAs beside the decoder), 3, 8, 11 (trunk tilings) on a full-width 2-layer SigLIP-L tower,
    and the connector alone"""
    from test_gpu_vit_kernels import _frames, _tower_config, _tower_engine
    out = {}
    cfg = _tower_config()
    eng = _tower_engine(cfg)
    for B in VIT_BATCHES:
        emb, tok = eng.vit_encode(_frames(B, cfg.frame_resolution, 40 + B), return_vit_tokens=True)
        out[f"vit.B{B}.tokens"], out[f"vit.B{B}.embeds"] = tok.clone(), emb.clone()
    g = torch.Generator().manual_seed(12)
    tokens = torch.randn(3 * cfg.frame_num_tokens, cfg.vision_hidden_size, generator=g).bfloat16()
    out["connector"] = eng.connector(tokens).clone()
    eng.close()
    return out


GROUPS = ["step.bf16", "step.fp8", "step.w8a8", "full.bf16", "full.fp8", "full.w8a8", "ragged_sampled_kv_ops", "vit"]


def scenarios() -> dict:
    tiny = tiny_state()
    out = {}
    for f in FORMS:
        out.update({f"step.{f}/{k}": v for k, v in step_forms(tiny, f).items()})
        out.update({f"full.{f}/{k}": v for k, v in step_full_width(f).items()})
    out.update({f"ragged_sampled_kv_ops/{k}": v for k, v in ragged_sampled_kv_ops(tiny).items()})
    out.update({f"vit/{k}": v for k, v in vit_and_connector().items()})
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


if __name__ == "__main__":
    torch.save(scenarios(), sys.argv[1])
