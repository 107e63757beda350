"""FP8 (e4m3) decoder weights: the FP8 GEMM kernels bit for bit against the bf16 kernels on the exactly upcast weights,
the FP8 engine against the CPU oracle on the dequantized weights, and the engine's exactness promises in the FP8 form.

Every finite e4m3 value is a bf16 value, so `codes.view(float8_e4m3fn).bfloat16()` is the exact upcast; the bf16
kernels on it produce the partials P_p the FP8 kernels must reproduce before their one scale multiplication.
"""
import ctypes as C
import os
import pathlib
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import test_gpu_decoder_kernels as DK  # noqa: E402  (its exact SwiGLU emulation and stream-K plane counts)
import test_gpu_frame_backlog as FB     # noqa: E402  (frame runs, one-by-one vs segmented steps)


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    from videollm_online_b200._lib import check
    check(rc, what)


def _upcast(codes):
    return codes.view(torch.float8_e4m3fn).bfloat16()


def _quantized(N, K, seed):
    from videollm_online_b200 import weights as W
    g = torch.Generator(device="cuda").manual_seed(seed)
    return W.quantize_fp8_rows((torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16())


def _planes_bf16(lib, wb, N, x, T, K, n_ctas):
    planes = C.c_int(0)
    _check(lib.vlo_op_gemm_ws(1, 0, _p(wb), N, _p(x), T, K, None, N, T * N, None, 0, n_ctas, 0, C.byref(planes), _st()),
           "plan bf16")
    out = torch.zeros(planes.value, T, N, device="cuda")
    _check(lib.vlo_op_gemm_ws(1, 0, _p(wb), N, _p(x), T, K, _p(out), N, T * N, None, 0, n_ctas, 0, C.byref(planes), _st()),
           "gemm_ws bf16")
    return out


def _planes_f8(lib, codes, scale, N, x, T, K, n_ctas):
    planes = C.c_int(0)
    _check(lib.vlo_op_gemm_ws_f8(_p(codes), _p(scale), N, _p(x), T, K, None, T * N, n_ctas, C.byref(planes), _st()),
           "plan f8")
    out = torch.zeros(planes.value, T, N, device="cuda")
    _check(lib.vlo_op_gemm_ws_f8(_p(codes), _p(scale), N, _p(x), T, K, _p(out), T * N, n_ctas, C.byref(planes), _st()),
           "gemm_ws_f8")
    return out


# ============================================================================================ kernels
@pytest.mark.parametrize("T", [16, 64, 128])
def test_conversion_is_exact(lib, T):
    """Weight rows hold every finite e4m3 code at the positions one-hot activation rows select, s = 1: the plane sum of
    token t, feature n is the decoded code W[n, k_t] exactly."""
    N, K = 256, 4096
    g = torch.Generator(device="cuda").manual_seed(T)
    codes = torch.randint(0, 256, (N, K), dtype=torch.uint8, device="cuda", generator=g)
    k_t = (torch.arange(T, device="cuda") * 61 + 5) % K
    hit = (torch.arange(N, device="cuda")[:, None] * T + torch.arange(T, device="cuda")[None, :]) % 256
    codes[:, k_t] = hit.to(torch.uint8)
    codes[(codes & 0x7F) == 0x7F] = 0   # the two NaN codes
    assert len(torch.unique(codes[:, k_t])) == 254
    x = torch.zeros(T, K, dtype=torch.bfloat16, device="cuda")
    x[torch.arange(T), k_t] = 1.0
    ones = torch.ones(N, device="cuda")
    out = _planes_f8(lib, codes, ones, N, x, T, K, 0).sum(0)
    torch.cuda.synchronize()
    want = codes[:, k_t].view(torch.float8_e4m3fn).float().t()
    assert torch.equal(out, want)


F8_SHAPES = [(6144, 4096), (4096, 4096), (4096, 14336)]      # q|k|v, o_proj, down_proj of Llama-3-8B
F8_ROWS = [1, 11, 16, 17, 33, 65, 97, 128]                   # every decoder token tile: 16 / 32 / 64 / 96 / 128


@pytest.fixture(scope="module")
def f8_operands():
    ops = {}
    for N, K in F8_SHAPES:
        codes, scale = _quantized(N, K, N + K)
        g = torch.Generator(device="cuda").manual_seed(K)
        ops[(N, K)] = (codes, scale, torch.randn(128, K, device="cuda", generator=g).bfloat16())
    return ops


@pytest.mark.parametrize("n_ctas", [0, 37])
@pytest.mark.parametrize("T", F8_ROWS)
@pytest.mark.parametrize("N,K", F8_SHAPES)
def test_planes_are_the_bf16_kernels_scaled(lib, f8_operands, N, K, T, n_ctas):
    """vlo_op_gemm_ws_f8 plane p = fl(P_p[t][n] * s[n]) bit for bit, P_p = plane p of the bf16 kernel (mode 0, same
    n_ctas) on the upcast weights; the same plan (plane count) either way."""
    codes, scale, x_all = f8_operands[(N, K)]
    x = x_all[:T].contiguous()
    ref = _planes_bf16(lib, _upcast(codes), N, x, T, K, n_ctas)
    out = _planes_f8(lib, codes, scale, N, x, T, K, n_ctas)
    torch.cuda.synchronize()
    assert out.shape == ref.shape
    if n_ctas:
        assert max(DK._sk_planes(N, K, n_ctas)) == ref.shape[0]
    assert torch.equal(out.view(torch.int32), (ref * scale).view(torch.int32))


def test_explicit_ctas_change_the_plane_count():
    for N, K in F8_SHAPES:
        assert max(DK._sk_planes(N, K, 37)) != max(DK._sk_planes(N, K, 0))


@pytest.fixture(scope="module")
def gate_up_f8():
    """28672 x 4096 interleaved gate|up, a quarter of the gate rows scaled so that gates reach +-100"""
    from videollm_online_b200 import weights as W
    I, K = 14336, 4096
    gs = torch.where(torch.arange(I, device="cuda") % 4 == 0, 40.0, 1.0)
    g = torch.Generator(device="cuda").manual_seed(7)
    gate = (torch.randn(I, K, device="cuda", generator=g) * gs[:, None] / K ** 0.5).bfloat16()
    up = (torch.randn(I, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    codes, scale = W.quantize_fp8_rows(W.interleave_gate_up(gate, up))
    x = torch.randn(128, K, device="cuda", generator=g).bfloat16()
    return codes, scale, x


@pytest.mark.parametrize("T", F8_ROWS)
def test_fused_gate_up(lib, gate_up_f8, T):
    """vlo_op_gemm_swiglu_f8 = the exact SwiGLU of g | u = bf16(sum_p fl(P_p * s)) in plane order, P_p the bf16 kernel's
    partials on the upcast weights; counters back at zero, rows past rows_x untouched."""
    codes, scale, x_all = gate_up_f8
    N, K = codes.shape
    I = N // 2
    x = x_all[:T].contiguous()
    ns = DK._sk_planes(N, K, 0)
    planes_buf = torch.full((max(1, max(ns) - 1) * T * N,), float("nan"), device="cuda")
    flags = torch.zeros(N // 128, dtype=torch.int32, device="cuda")
    act = DK._sentinel(T + 3, I)
    _check(lib.vlo_op_gemm_swiglu_f8(_p(codes), _p(scale), N, _p(x), T, K, _p(act), _p(planes_buf), planes_buf.numel(),
                                     _p(flags), flags.numel(), _st()), "gemm_swiglu_f8")
    torch.cuda.synchronize()
    assert int(flags.abs().sum()) == 0
    assert DK._same_bits(act[T:], DK._sentinel(3, I))
    act = act[:T]
    ref = _planes_bf16(lib, _upcast(codes), N, x, T, K, 0) * scale
    torch.cuda.synchronize()
    y = DK._fixup_sum(ref, torch.tensor(ns, device="cuda").repeat_interleave(128)).bfloat16().double()
    y = y.view(T, I // 64, 2, 64)
    g, u = y[:, :, 0].reshape(T, I), y[:, :, 1].reshape(T, I)
    e = torch.exp(-g)
    silu = torch.where(e > DK.FLT_MAX, -0.0 * g.abs(), g / (1 + e))
    lo, hi = DK._either(silu, DK._silu_delta())
    DK._assert_in(act, [DK._bf(lo * u), DK._bf(hi * u)], f"SwiGLU f8 T={T}")


# ============================================================================================ engine
def _engine(cfg, llm, fp8, max_streams=2, max_kv_tokens=2048):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, fp8_weights=fp8)
    return model.engine


@pytest.fixture(scope="module")
def tiny():
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config()
    llm = W.synthetic_llm_state(cfg, seed=0)
    llm["lm_head.weight"] = (llm["lm_head.weight"].float() * 8).to(torch.bfloat16)
    return cfg, llm


def _dequantized_state(cfg, llm):
    """the HF-style state with every quantized matrix replaced by bf16(fp32(q) * s): per-row scales commute with the
    q|k|v concatenation and the gate|up interleave"""
    from videollm_online_b200 import weights as W
    out = dict(llm)
    for i in range(cfg.num_hidden_layers):
        for m in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj",
                  "mlp.up_proj", "mlp.down_proj"):
            k = f"model.layers.{i}.{m}.weight"
            out[k] = W.dequantize_fp8_rows(*W.quantize_fp8_rows(llm[k].cuda())).bfloat16().cpu()
    return out


def test_engine_vs_oracle_on_dequantized_weights(tiny):
    """all-position logits of the FP8 engine vs the CPU oracle on bf16(q * s) weights within 0.25 + 0.02 |x|; greedy ids
    exact where the oracle's top-2 margin exceeds 0.5"""
    sys.path.insert(0, str(ROOT / "oracle"))
    import vlo_oracle as O
    cfg, llm = tiny
    eng = _engine(cfg, llm, True)
    assert eng.fp8_weights
    sid = eng.stream_open()
    g = torch.Generator().manual_seed(4)
    emb = torch.randn(40, cfg.hidden_size, generator=g).bfloat16()
    eng.step([sid], [40], emb.cuda())
    got = eng.last_step_logits(40).float().cpu()
    ref = O.llama_forward(_dequantized_state(cfg, llm), cfg, emb, O.KVCache(cfg.num_hidden_layers)).float()
    err = (got - ref).abs()
    assert bool((err <= 0.25 + 0.02 * ref.abs()).all()), f"worst {err.max().item()}"
    top2 = ref.topk(2, dim=-1).values
    sure = (top2[:, 0] - top2[:, 1]) > 0.5
    assert int(sure.sum()) > 0
    assert torch.equal(got.argmax(-1)[sure], ref.argmax(-1)[sure])


def test_segmented_backlog_equals_one_frame_per_step(tiny):
    cfg, llm = tiny
    eng = _engine(cfg, llm, True)
    a, b = FB._prefixed_pair(eng, 300)
    for k in range(1, 12):
        emb, ids = FB._frames(cfg, k, 50 + k)
        seg = FB._segmented(eng, a, emb, ids, k)
        one = FB._one_by_one(eng, b, emb, ids, k)
        for j in range(k):
            assert torch.equal(seg[j][0], one[j][0]) and torch.equal(seg[j][1], one[j][1]), f"k={k} frame {j}"
        assert eng.kv_len(a) == eng.kv_len(b)
    assert FB._same_kv(FB._kv_all(eng, a), FB._kv_all(eng, b))


def test_verify_step_with_drafts_equals_one_token_per_step(tiny):
    """rows [id | d1 .. dn] as segments [1] * (n + 1) give each token's logits and cache rows of one token per step"""
    cfg, llm = tiny
    eng = _engine(cfg, llm, True)
    a, b = FB._prefixed_pair(eng, 200)
    ids = torch.tensor([17, 40, 99, 3, 250, 8], dtype=torch.int64)
    n = ids.numel()
    zeros = torch.zeros(n, cfg.hidden_size, dtype=torch.bfloat16, device="cuda")
    lg, _ = eng.step([a], [n], zeros, row_ids=ids, segments=[[1] * n])
    verify = lg[:n].clone()
    for j in range(n):
        lg1, _ = eng.step([b], [1], zeros[:1], row_ids=ids[j:j + 1])
        assert torch.equal(lg1[0], verify[j]), f"token {j}"
    assert FB._same_kv(FB._kv_all(eng, a), FB._kv_all(eng, b))


def test_ragged_multistream_equals_single_streams(tiny):
    cfg, llm = tiny
    eng = _engine(cfg, llm, True, max_streams=3)
    q = [11, 1, 29]
    s = [eng.stream_open() for _ in q]
    for i, sid in enumerate(s):
        eng.kv_fill_synthetic(sid, 100 + 37 * i, seed=i)
    g = torch.Generator().manual_seed(9)
    emb = torch.randn(sum(q), cfg.hidden_size, generator=g).bfloat16().cuda()
    lg, dc = eng.step(s, q, emb)
    batched = (lg.clone(), dc.clone())
    for i, sid in enumerate(s):
        eng.kv_truncate(sid, 100 + 37 * i)
    o = 0
    for i, sid in enumerate(s):
        lg1, dc1 = eng.step([sid], [q[i]], emb[o:o + q[i]].contiguous())
        assert torch.equal(lg1[0], batched[0][i]) and torch.equal(dc1[0], batched[1][i]), f"stream {i}"
        o += q[i]


def test_sampled_ids_reproducible_from_seed(tiny):
    from videollm_online_b200.engine import SampleRow
    cfg, llm = tiny
    eng = _engine(cfg, llm, True)
    draws = []
    for _ in range(2):
        sid = eng.stream_open()
        eng.kv_fill_synthetic(sid, 64, seed=2)
        g = torch.Generator().manual_seed(3)
        emb = torch.randn(5, cfg.hidden_size, generator=g).bfloat16().cuda()
        row = SampleRow(seed=1234, position=64, temperature=0.9, top_k=50, top_p=0.95)
        eng.step([sid], [5], emb, sample=[row])
        draws.append(eng.read_decisions(1)[0].sampled_id)
        eng.stream_close(sid)
    assert draws[0] is not None and draws[0] == draws[1]


# ============================================================================================ errors / accounting
def test_finalize_rejects_mixed_missing_and_wrong_sizes(tiny):
    from videollm_online_b200 import weights as W
    from videollm_online_b200._lib import VloError
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    bf = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512)
    f8 = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512, fp8_weights=True)

    def attempt(packed, match):
        eng = Engine(cfg, "cuda:0", max_streams=1, max_kv_tokens=256, max_step_tokens=32, max_vit_batch=1)
        try:
            with pytest.raises(VloError, match=match):
                eng.load_weights(packed)
        finally:
            eng.close()

    mixed = {k: v for k, v in bf.items() if not k.startswith("L1.o")}
    mixed["L1.o.f8"], mixed["L1.o.scale"] = f8["L1.o.f8"], f8["L1.o.scale"]
    attempt(mixed, "L1.o.f8")
    no_scale = {k: v for k, v in f8.items() if k != "L0.down.scale"}
    attempt(no_scale, "L0.down.scale")
    short = dict(f8)
    short["L0.gate_up.f8"] = f8["L0.gate_up.f8"][:-1].contiguous()
    attempt(short, "L0.gate_up.f8")
    short_s = dict(f8)
    short_s["L1.qkv.scale"] = f8["L1.qkv.scale"][:-4].contiguous()
    attempt(short_s, "L1.qkv.scale")
    both = dict(f8)
    both["L0.o"] = bf["L0.o"]
    attempt(both, "L0.o")


def test_resume_rejects_a_state_of_the_other_form(tiny):
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200._lib import VloError
    from videollm_online_b200 import weights as W
    cfg, llm = tiny
    vis = W.synthetic_vision_state(cfg, seed=1)
    sessions = {}
    for fp8 in (False, True):
        model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                                max_streams=1, max_kv_tokens=512, max_step_tokens=64, max_vit_batch=2, fp8_weights=fp8)
        sessions[fp8] = LiveInfer(LiveArguments(), model=model, tokenizer=tok)
    state = sessions[False].suspend()
    assert state.fp8_weights is False
    with pytest.raises(VloError, match="bf16 layer weights"):
        sessions[True].resume(state)
    sessions[False].resume(state)
    state8 = sessions[True].suspend()
    assert state8.fp8_weights is True
    with pytest.raises(VloError, match="FP8 layer weights"):
        sessions[False].resume(state8)


def test_no_bf16_copy_and_weight_bytes(tiny):
    cfg, llm = tiny
    eng = _engine(cfg, llm, True)
    H, I = cfg.hidden_size, cfg.intermediate_size
    A, QKV = cfg.num_attention_heads * cfg.head_dim, (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * cfg.head_dim
    w = eng.weights
    for i in range(cfg.num_hidden_layers):
        for m in ("qkv", "o", "gate_up", "down"):
            assert f"L{i}.{m}" not in w
            assert w[f"L{i}.{m}.f8"].dtype == torch.uint8 and w[f"L{i}.{m}.scale"].dtype == torch.float32
    from videollm_online_b200 import weights as W
    L, mats = cfg.num_hidden_layers, [(QKV, H), (H, A), (2 * I, H), (H, I)]
    f8_bytes = L * sum(n * k + 4 * n for n, k in mats)      # 1 B per weight + one fp32 scale per row
    assert sum(t.numel() * t.element_size() for k, t in w.items() if k.endswith((".f8", ".scale"))) == f8_bytes
    # everything else is the bf16 engine's: its layer matrices take 2 B per weight
    eng16 = _engine(cfg, llm, False)
    assert not eng16.fp8_weights
    assert W.engine_weight_bytes(w) == W.engine_weight_bytes(eng16.weights) - L * sum(2 * n * k for n, k in mats) + f8_bytes


# ============================================================================================ full size, reported
def test_full_size_fp8_vs_bf16_report():
    """32-layer Llama-3-8B-width synthetic stack at 12k keys, 11-token frame steps, 64 steps on a bf16 and an FP8 engine
    of the same seed: logit rms / max difference, correlation, argmax and speak / silent agreement are printed and
    appended to VLO_PARITY_LOG; only finiteness is asserted (synthetic weights say little about answer quality)."""
    import json
    from videollm_online_b200 import llama3_8b_siglip_l
    from videollm_online_b200.modeling_live import build_live
    cfg = llama3_8b_siglip_l()
    fill, steps, q = 12288, 64, 11
    res = {}
    for fp8 in (False, True):
        model, _ = build_live(config=cfg, synthetic_weights=True, seed=0, set_vision_inside=False, device="cuda:0",
                              max_streams=1, max_kv_tokens=fill + steps * q + 64, max_step_tokens=128, max_vit_batch=1,
                              fp8_weights=fp8)
        eng = model.engine
        sid = eng.stream_open()
        eng.kv_fill_synthetic(sid, fill, seed=5)
        g = torch.Generator().manual_seed(6)
        logits, speak = [], []
        for s in range(steps):
            emb = (torch.randn(q, cfg.hidden_size, generator=g) * 0.02).bfloat16().cuda()
            ids = torch.full((q,), -1, dtype=torch.int64)
            ids[0] = cfg.frame_token_interval_id
            lg, _ = eng.step([sid], [q], emb, row_ids=ids)
            logits.append(lg[0].float().cpu())
            d = eng.read_decisions(1)[0]
            speak.append(d.next_id(cfg.frame_token_interval_id, 0.725) != cfg.frame_token_interval_id)
        res[fp8] = (torch.stack(logits), speak)
        del model, eng
        torch.cuda.empty_cache()
    a, b = res[False][0], res[True][0]
    assert bool(torch.isfinite(b).all()) and bool(torch.isfinite(a).all())
    d = (b - a)
    rep = {"test": "fp8_weights_full_size", "steps": steps, "keys": fill, "q": q,
           "logit_rms_diff": d.pow(2).mean().sqrt().item(), "logit_max_diff": d.abs().max().item(),
           "logit_rms": a.pow(2).mean().sqrt().item(),
           "corr": torch.corrcoef(torch.stack([a.flatten(), b.flatten()]))[0, 1].item(),
           "argmax_agree": (a.argmax(-1) == b.argmax(-1)).float().mean().item(),
           "speak_agree": sum(x == y for x, y in zip(res[False][1], res[True][1])) / steps,
           "gpu": torch.cuda.get_device_name(0)}
    print(json.dumps(rep))
    log = os.environ.get("VLO_PARITY_LOG")
    if log:
        with open(log, "a") as fh:
            fh.write(json.dumps(rep) + "\n")
