"""Int4 (W4A16) decoder weights: the int4 GEMM kernels bit for bit against the bf16 kernels on the dequantized weights
W4 = bf16_rn(q * s), and an int4 engine bit for bit against a bf16 engine loaded with W4.

weights.dequantize_int4_groups is the definition of W4; the int4 kernels dequantize the codes into the wgmma A fragment
in registers and run the bf16 wgmma chain over the bf16 kernels' stream-K units, so every partial plane, and everything
computed from the planes, must be the bf16 engine's.
"""
import ctypes as C
import os
import pathlib
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import test_gpu_decoder_kernels as DK  # noqa: E402  (stream-K plane counts, sentinels)
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


def _quantized(N, K, seed, spread=False):
    """(packed codes, bf16 scales, W4) of a random [N, K] weight; spread: row magnitudes over 2^-20 .. 2^4"""
    from videollm_online_b200 import weights as W
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    if spread:
        w = w * torch.pow(2.0, torch.randint(-20, 5, (N, 1), device="cuda", generator=g).float())
    q, s = W.quantize_int4_groups(w.bfloat16())
    return W.pack_int4_codes(q), s, W.dequantize_int4_groups(q, s)


def _planes_bf16(lib, wb, N, x, T, K, n_ctas):
    planes = C.c_int(0)
    _check(lib.vlo_op_gemm_ws(1, 0, _p(wb), N, _p(x), T, K, None, N, T * N, None, 0, n_ctas, 0, C.byref(planes), _st()),
           "plan bf16")
    out = torch.full((planes.value + 1, T, N), float("nan"), device="cuda")
    _check(lib.vlo_op_gemm_ws(1, 0, _p(wb), N, _p(x), T, K, _p(out), N, T * N, None, 0, n_ctas, 0, C.byref(planes), _st()),
           "gemm_ws bf16")
    return out


def _planes_i4(lib, codes, gs, N, x, T, K, n_ctas):
    planes = C.c_int(0)
    _check(lib.vlo_op_gemm_ws_i4(_p(codes), _p(gs), N, _p(x), T, K, None, T * N, n_ctas, C.byref(planes), _st()),
           "plan i4")
    out = torch.full((planes.value + 1, T, N), float("nan"), device="cuda")   # one spare plane: must stay NaN
    _check(lib.vlo_op_gemm_ws_i4(_p(codes), _p(gs), N, _p(x), T, K, _p(out), T * N, n_ctas, C.byref(planes), _st()),
           "gemm_ws_i4")
    return out


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


# ============================================================================================ kernels
SHAPES = [(6144, 4096), (4096, 4096), (4096, 14336), (256, 128), (200, 384), (1000, 640)]   # Llama-3-8B, tiny and odd
ROWS = [1, 11, 16, 17, 31, 33, 64, 65, 97, 128]                 # every decoder token tile: 16 / 32 / 64 / 96 / 128


@pytest.fixture(scope="module")
def operands():
    cache = {}

    def get(N, K):
        if (N, K) not in cache:
            codes, gs, w4 = _quantized(N, K, N + K, spread=(N, K) == (200, 384))
            g = torch.Generator(device="cuda").manual_seed(K)
            cache[(N, K)] = (codes, gs, w4, torch.randn(128, K, device="cuda", generator=g).bfloat16())
        return cache[(N, K)]
    return get


@pytest.mark.parametrize("n_ctas", [0, 7, 37])
@pytest.mark.parametrize("T", ROWS)
@pytest.mark.parametrize("N,K", SHAPES)
def test_planes_are_the_bf16_kernels_on_w4(lib, operands, N, K, T, n_ctas):
    """every plane of vlo_op_gemm_ws_i4 equals that of the bf16 kernel on W4 (same n_ctas) bit for bit; the same plan;
    the plane past the plan stays NaN"""
    codes, gs, w4, x_all = operands(N, K)
    x = x_all[:T].contiguous()
    ref = _planes_bf16(lib, w4, N, x, T, K, n_ctas)
    out = _planes_i4(lib, codes, gs, N, x, T, K, n_ctas)
    torch.cuda.synchronize()
    assert _same_bits(out, ref), f"N={N} K={K} T={T} n_ctas={n_ctas}"
    assert bool(torch.isnan(out[-1]).all())


@pytest.mark.parametrize("T", [1, 16, 97, 128])
@pytest.mark.parametrize("N,K", [(4096, 4096), (1000, 640)])
def test_planes_eight_planes(lib, operands, N, K, T):
    n_ctas = DK._ctas_for_planes(N, K, 8)
    codes, gs, w4, x_all = operands(N, K)
    x = x_all[:T].contiguous()
    ref = _planes_bf16(lib, w4, N, x, T, K, n_ctas)
    out = _planes_i4(lib, codes, gs, N, x, T, K, n_ctas)
    torch.cuda.synchronize()
    assert out.shape[0] == 9
    assert _same_bits(out, ref)


def test_bad_arguments(lib, operands):
    from videollm_online_b200._lib import VloError
    codes, gs, w4, x = operands(256, 128)
    out = torch.zeros(4, 16, 256, device="cuda")
    with pytest.raises(VloError, match="128"):   # K not a multiple of 128
        _check(lib.vlo_op_gemm_ws_i4(_p(codes), _p(gs), 256, _p(x), 16, 64, _p(out), 16 * 256, 0, None, _st()), "k")
    with pytest.raises(VloError, match="1..128 token rows"):
        _check(lib.vlo_op_gemm_ws_i4(_p(codes), _p(gs), 256, _p(x), 129, 128, _p(out), 16 * 256, 0, None, _st()), "T")
    with pytest.raises(VloError, match="group scales"):
        _check(lib.vlo_op_gemm_ws_i4(_p(codes), None, 256, _p(x), 16, 128, _p(out), 16 * 256, 0, None, _st()), "gs")


@pytest.fixture(scope="module")
def gate_up():
    """interleaved gate|up of Llama-3-8B (28672 x 4096) and a small one, quantized"""
    from videollm_online_b200 import weights as W
    out = {}
    for I, K in ((14336, 4096), (256, 384)):
        g = torch.Generator(device="cuda").manual_seed(I)
        gate = (torch.randn(I, K, device="cuda", generator=g) * 3 / K ** 0.5).bfloat16()
        up = (torch.randn(I, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
        q, s = W.quantize_int4_groups(W.interleave_gate_up(gate, up))
        out[(2 * I, K)] = (W.pack_int4_codes(q), s, W.dequantize_int4_groups(q, s),
                           torch.randn(128, K, device="cuda", generator=g).bfloat16())
    return out


def _swiglu(lib, fn, w, gs, N, x, T, K):
    I = N // 2
    ns = DK._sk_planes(N, K, 0)
    planes = torch.full((max(1, max(ns) - 1) * T * N,), float("nan"), device="cuda")
    flags = torch.zeros(N // 128, dtype=torch.int32, device="cuda")
    act = DK._sentinel(T + 3, I)
    args = (_p(w),) + ((_p(gs),) if gs is not None else ()) + (N, _p(x), T, K, _p(act), _p(planes), planes.numel(),
                                                                _p(flags), flags.numel(), _st())
    _check(fn(*args), "swiglu")
    torch.cuda.synchronize()
    assert int(flags.abs().sum()) == 0
    return act


@pytest.mark.parametrize("T", ROWS)
@pytest.mark.parametrize("N,K", [(28672, 4096), (512, 384)])
def test_fused_gate_up_is_the_bf16_kernel_on_w4(lib, gate_up, N, K, T):
    codes, gs, w4, x_all = gate_up[(N, K)]
    x = x_all[:T].contiguous()
    want = _swiglu(lib, lib.vlo_op_gemm_swiglu, w4, None, N, x, T, K)
    got = _swiglu(lib, lib.vlo_op_gemm_swiglu_i4, codes, gs, N, x, T, K)
    assert DK._same_bits(got, want), f"N={N} K={K} T={T}"


# ============================================================================================ engine
def _w4_state(cfg, llm):
    """the HF-style state with every layer matrix replaced by W4: groups run along K inside one row, so they commute
    with the q|k|v concatenation and the gate|up interleave"""
    from videollm_online_b200 import weights as W
    out = dict(llm)
    for i in range(cfg.num_hidden_layers):
        for m in ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj",
                  "mlp.up_proj", "mlp.down_proj"):
            k = f"model.layers.{i}.{m}.weight"
            out[k] = W.dequantize_int4_groups(*W.quantize_int4_groups(llm[k].cuda())).cpu()
    return out


def _model(cfg, llm, int4, max_streams=3, max_kv_tokens=4096, kv_pool_tokens=None):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=kv_pool_tokens,
                          int4_weights=int4)
    return model


@pytest.fixture(scope="module")
def tiny():
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config()
    llm = W.synthetic_llm_state(cfg, seed=0)
    llm["lm_head.weight"] = (llm["lm_head.weight"].float() * 8).to(torch.bfloat16)
    return cfg, llm


@pytest.fixture(scope="module")
def pair(tiny):
    """(int4 engine on the state, bf16 engine on W4)"""
    cfg, llm = tiny
    e4 = _model(cfg, llm, True).engine
    eb = _model(cfg, _w4_state(cfg, llm), False).engine
    assert e4.int4_weights and not eb.int4_weights and not e4.prefills and eb.prefills
    return e4, eb


def _emb(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()


def _outputs(eng, sid, lg, dc, n):
    return (lg.clone(), dc.clone(), eng.last_step_hidden(n).clone(), FB._kv_all(eng, sid))


def _assert_same(a, b, what):
    assert torch.equal(a[0], b[0]), f"{what}: logits"
    assert torch.equal(a[1], b[1]), f"{what}: decision rows"
    assert torch.equal(a[2], b[2]), f"{what}: final hidden rows"
    assert FB._same_kv(a[3], b[3]), f"{what}: K/V"


@pytest.mark.parametrize("T", [1, 11, 128])
def test_engine_step_equals_bf16_engine_on_w4(tiny, pair, T):
    """one stream, T rows after a 40-row step"""
    cfg, _ = tiny
    res = []
    for eng in pair:
        sid = eng.stream_open()
        eng.step([sid], [40], _emb(cfg, 40, 1))
        lg, dc = eng.step([sid], [T], _emb(cfg, T, 2 + T))
        res.append(_outputs(eng, sid, lg, dc, T))
        eng.stream_close(sid)
    _assert_same(res[0], res[1], f"T={T}")
    assert torch.isfinite(res[0][0].float()).all()


def test_long_input_chunked_equals_bf16_prefill(tiny):
    """a 1000-row input after a 40-row step on fresh engines: the bf16 engine prefills it, the int4 engine cuts it into
    128-row steps; also fed as explicit 128-row steps on both"""
    cfg, llm = tiny
    res = []
    for int4, state in ((True, llm), (False, _w4_state(cfg, llm))):
        eng = _model(cfg, state, int4).engine
        assert eng.prefills != int4
        outs = []
        for cap in (1000, 128):
            sid = eng.stream_open()
            eng.step([sid], [40], _emb(cfg, 40, 1))
            emb = _emb(cfg, 1000, 1002)
            for lo in range(0, 1000, cap):
                n = min(cap, 1000 - lo)
                lg, dc = eng.step([sid], [n], emb[lo:lo + n].contiguous())
            last_rows = 1000 if eng.prefills and cap == 1000 else 1000 % 128   # rows of the last pass
            outs.append((lg.clone(), dc.clone(), eng.last_step_hidden(last_rows)[-1:].clone(), FB._kv_all(eng, sid)))
            eng.stream_close(sid)
        res.append(outs)
        eng.close()
    _assert_same(res[0][0], res[1][0], "one call")
    _assert_same(res[0][1], res[1][1], "128-row steps")
    _assert_same(res[0][0], res[0][1], "int4: one call vs 128-row steps")


def test_segments_on_a_fragmented_pool(tiny, pair):
    cfg, _ = tiny
    res = []
    for eng in pair:
        hold = [eng.stream_open() for _ in range(2)]
        eng.kv_fill_synthetic(hold[0], 70, seed=1)
        eng.kv_fill_synthetic(hold[1], 130, seed=2)
        eng.stream_close(hold[0])   # a hole in the pool
        sid = eng.stream_open()
        eng.kv_fill_synthetic(sid, 100, seed=3)
        emb = _emb(cfg, 22, 5)
        lg, dc = eng.step([sid], [22], emb, segments=[[1, 10, 1, 10]])
        res.append(_outputs(eng, sid, lg, dc, 22))
        eng.stream_close(sid)
        eng.stream_close(hold[1])
    _assert_same(res[0], res[1], "segments [1, 10, 1, 10]")


def test_ragged_three_streams(tiny, pair):
    cfg, _ = tiny
    q = [11, 1, 29]
    res = []
    for eng in pair:
        s = [eng.stream_open() for _ in q]
        for i, sid in enumerate(s):
            eng.kv_fill_synthetic(sid, 100 + 37 * i, seed=i)
        lg, dc = eng.step(s, q, _emb(cfg, sum(q), 9))
        res.append((lg.clone(), dc.clone(), eng.last_step_hidden(sum(q)).clone(), [FB._kv_all(eng, sid) for sid in s]))
        for sid in s:
            eng.stream_close(sid)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])
    assert all(FB._same_kv(a, b) for a, b in zip(res[0][3], res[1][3]))


def test_verify_step_with_drafts(tiny, pair):
    cfg, _ = tiny
    ids = torch.tensor([17, 40, 99, 3, 250, 8], dtype=torch.int64)
    n = ids.numel()
    res = []
    for eng in pair:
        sid = eng.stream_open()
        eng.kv_fill_synthetic(sid, 200, seed=4)
        zeros = torch.zeros(n, cfg.hidden_size, dtype=torch.bfloat16, device="cuda")
        lg, dc = eng.step([sid], [n], zeros, row_ids=ids, segments=[[1] * n])
        res.append(_outputs(eng, sid, lg, dc, n))
        eng.stream_close(sid)
    _assert_same(res[0], res[1], "verify step")


def test_sampled_step(tiny, pair):
    from videollm_online_b200.engine import SampleRow
    cfg, _ = tiny
    draws = []
    for eng in pair:
        sid = eng.stream_open()
        eng.kv_fill_synthetic(sid, 64, seed=2)
        row = SampleRow(seed=1234, position=64, temperature=0.9, top_k=50, top_p=0.95)
        eng.step([sid], [5], _emb(cfg, 5, 3), sample=[row])
        draws.append(eng.read_decisions(1)[0].sampled_id)
        eng.stream_close(sid)
    assert draws[0] is not None and draws[0] == draws[1]


def test_evict_compact_swap_then_step(tiny, pair):
    cfg, _ = tiny
    res = []
    for eng in pair:
        sid = eng.stream_open()
        eng.step([sid], [128], _emb(cfg, 128, 11))
        eng.step([sid], [100], _emb(cfg, 100, 12))
        outs = []
        eng.kv_evict(sid, 64, 64)
        lg, dc = eng.step([sid], [11], _emb(cfg, 11, 13))
        outs.append(_outputs(eng, sid, lg, dc, 11))
        eng.kv_compact(sid, [(0, 20), (40, 50)])
        lg, dc = eng.step([sid], [11], _emb(cfg, 11, 14))
        outs.append(_outputs(eng, sid, lg, dc, 11))
        img = eng.kv_swap_out(sid)
        eng.kv_swap_in(sid, img)
        lg, dc = eng.step([sid], [1], _emb(cfg, 1, 15))
        outs.append(_outputs(eng, sid, lg, dc, 1))
        res.append(outs)
        eng.stream_close(sid)
    for what, a, b in zip(("evict", "compact", "swap"), res[0], res[1]):
        _assert_same(a, b, what)


def test_over_poisoned_pages(tiny, pair):
    """pages that held NaN / +-Inf rows of a closed stream, reused by the next one"""
    cfg, _ = tiny
    res = []
    for eng in pair:
        bad = eng.stream_open()
        eng.kv_fill_synthetic(bad, 300, seed=6)
        for layer in range(cfg.num_hidden_layers):
            for v in (False, True):
                kv = eng.kv_read(bad, layer, v)
                poison = torch.tensor([float("nan"), float("inf"), -float("inf")], dtype=kv.dtype, device=kv.device)
                kv.copy_(poison[torch.arange(kv.numel(), device=kv.device) % 3].view_as(kv))
                eng.kv_write(bad, layer, v, kv)
        eng.stream_close(bad)
        sid = eng.stream_open()
        lg, dc = eng.step([sid], [33], _emb(cfg, 33, 21))
        res.append(_outputs(eng, sid, lg, dc, 33))
        eng.stream_close(sid)
    _assert_same(res[0], res[1], "poisoned pages")
    assert torch.isfinite(res[0][0].float()).all()


def test_two_layer_full_width_stack():
    """Llama-3-8B's layer widths (4096 / 14336, 32 q and 8 kv heads), two layers"""
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config()
    cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.num_key_value_heads = 4096, 14336, 32, 8
    llm = W.synthetic_llm_state(cfg, seed=5, device="cuda")
    res = []
    for int4, state in ((True, llm), (False, _w4_state(cfg, llm))):
        eng = _model(cfg, state, int4, max_streams=1, max_kv_tokens=1024).engine
        sid = eng.stream_open()
        eng.step([sid], [40], _emb(cfg, 40, 1))
        lg, dc = eng.step([sid], [11], _emb(cfg, 11, 2))
        res.append(_outputs(eng, sid, lg, dc, 11))
        eng.close()
    _assert_same(res[0], res[1], "full-width stack")


CHILD = """
import sys, torch
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import vlo_bootstrap
import test_gpu_int4_weights as T
from videollm_online_b200 import tiny_config, weights as W
cfg = tiny_config()
llm = W.synthetic_llm_state(cfg, seed=0)
llm["lm_head.weight"] = (llm["lm_head.weight"].float() * 8).to(torch.bfloat16)
eng = T._model(cfg, llm, True).engine
sid = eng.stream_open()
eng.step([sid], [40], T._emb(cfg, 40, 1))
lg, dc = eng.step([sid], [11], T._emb(cfg, 11, 13))
torch.save({{"lg": lg.cpu(), "dc": dc.cpu(), "kv": [(k.cpu(), v.cpu()) for k, v in T.FB._kv_all(eng, sid)]}}, sys.argv[1])
"""


def test_no_pdl_child_equals_pdl(tiny, pair, tmp_path):
    cfg, _ = tiny
    path = tmp_path / "no_pdl.pt"
    env = dict(os.environ, VLO_NO_PDL="1")
    code = CHILD.format(root=str(ROOT), tests=str(ROOT / "tests"))
    r = subprocess.run([sys.executable, "-c", code, str(path)], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    child = torch.load(path)
    eng = pair[0]
    sid = eng.stream_open()
    eng.step([sid], [40], _emb(cfg, 40, 1))
    lg, dc = eng.step([sid], [11], _emb(cfg, 11, 13))
    assert torch.equal(lg.cpu(), child["lg"]) and torch.equal(dc.cpu(), child["dc"])
    assert all(torch.equal(k.cpu(), k2) and torch.equal(v.cpu(), v2)
               for (k, v), (k2, v2) in zip(FB._kv_all(eng, sid), child["kv"]))
    eng.stream_close(sid)


# ============================================================================================ errors
def test_finalize_rejects_mixed_missing_and_wrong_sizes(tiny):
    """(K % 128 != 0 cannot reach finalize: engine creation needs hidden, intermediate and head_dim multiples of 128;
    the GEMM's own check is test_bad_arguments)"""
    from videollm_online_b200 import weights as W
    from videollm_online_b200._lib import VloError
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    bf = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512)
    i4 = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512, int4_weights=True)
    f8 = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512, fp8_weights=True)

    def attempt(packed, match, fp8_act=False):
        eng = Engine(cfg, "cuda:0", max_streams=1, max_kv_tokens=256, max_step_tokens=32, max_vit_batch=1,
                     fp8_activations=fp8_act)
        try:
            before = eng.device_bytes()
            with pytest.raises(VloError, match=match):
                eng.load_weights(packed)
            assert eng.max_prefill_tokens == 0 and eng.device_bytes() == before
        finally:
            eng.close()

    mixed = {k: v for k, v in bf.items() if not k.startswith("L1.o")}
    mixed["L1.o.i4"], mixed["L1.o.gscale"] = i4["L1.o.i4"], i4["L1.o.gscale"]
    attempt(mixed, "L1.o.i4")
    mixed8 = {k: v for k, v in i4.items() if not k.startswith("L0.down")}
    mixed8["L0.down.f8"], mixed8["L0.down.scale"] = f8["L0.down.f8"], f8["L0.down.scale"]
    attempt(mixed8, "L0.down.f8")
    attempt({k: v for k, v in i4.items() if k != "L0.down.gscale"}, "L0.down.gscale")
    attempt({k: v for k, v in i4.items() if k != "L1.qkv.i4"}, "L1.qkv.i4")
    short = dict(i4)
    short["L0.gate_up.i4"] = i4["L0.gate_up.i4"][:-16].contiguous()
    attempt(short, "L0.gate_up.i4")
    short_s = dict(i4)
    short_s["L1.qkv.gscale"] = i4["L1.qkv.gscale"][:-1].contiguous()
    attempt(short_s, "L1.qkv.gscale")
    both = dict(i4)
    both["L0.o"] = bf["L0.o"]
    attempt(both, "L0.o")
    attempt(i4, "int4", fp8_act=True)


# ============================================================================================ LiveInfer
LIVE_FRAMES = 40
LIVE_SPEAK = {7, 22, 33}


@pytest.fixture(scope="module")
def tiny_vision(tiny):
    from videollm_online_b200 import weights as W
    cfg, llm = tiny
    return cfg, llm, W.synthetic_vision_state(cfg, seed=1)


def _live_model(cfg, llm, vis, int4):
    """the model LiveInfer builds from its LiveArguments (build_model_and_tokenizer with the same keywords), on the given
    weights"""
    from dataclasses import asdict
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.modeling_live import build_model_and_tokenizer
    args = LiveArguments(llm_pretrained="", frame_resolution=cfg.frame_resolution, int4_weights=int4)
    model, tok = build_model_and_tokenizer(is_training=False, set_vision_inside=True, config=cfg, llm_state=llm,
                                           vision_state=vis, max_kv_tokens=2048, max_vit_batch=8, **asdict(args))
    assert model.engine.int4_weights == int4
    return args, model, tok


def test_liveinfer_cli_int4_equals_bf16_on_w4(tiny_vision):
    """cli.main over a seeded clip with LiveArguments(int4_weights=True), and with a bf16 model on W4: the same
    conversation, every decision row as the device wrote it, and the same final cache; the suspended state records
    the form"""
    import test_gpu_ordering as OR
    from videollm_online_b200 import cli
    from videollm_online_b200.inference import LiveInfer
    cfg, llm, vis = tiny_vision
    runs = []
    for int4, state in ((True, llm), (False, _w4_state(cfg, llm))):
        args, model, tok = _live_model(cfg, state, vis, int4)
        li = LiveInfer(args, model=model, tokenizer=tok)
        hook, raw = OR._script(cfg, LIVE_SPEAK)
        mode = {"resp": False}
        respond = li._call_for_response

        def call_for_response(*a, respond=respond, mode=mode):
            mode["resp"] = True
            try:
                return respond(*a)
            finally:
                mode["resp"] = False
        li._call_for_response = call_for_response
        li.decision_hook = lambda dec, n, hook=hook, mode=mode: hook(dec, n, mode["resp"])
        _, history = cli.main(li, video=cli.synthetic_clip(LIVE_FRAMES, cfg.frame_resolution, seed=21),
                              n_iters=LIVE_FRAMES, quiet=True)
        conv = [(c["role"], c["content"]) for c in history["conversation"] if "role" in c]
        runs.append((conv, raw, FB._kv_all(model.engine, li._kv.stream_id)))
        assert li.suspend().int4_weights is int4
    (conv4, raw4, kv4), (conv16, raw16, kv16) = runs
    assert len(conv4) >= 4
    assert conv4 == conv16
    assert raw4 == raw16
    assert FB._same_kv(kv4, kv16)


def test_resume_refuses_a_state_of_another_weight_form(tiny_vision):
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200._lib import VloError
    cfg, llm, vis = tiny_vision
    sessions = {}
    for form in ("bf16", "fp8", "int4"):
        model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                                max_streams=1, max_kv_tokens=512, max_step_tokens=64, max_vit_batch=2,
                                fp8_weights=form == "fp8", int4_weights=form == "int4")
        sessions[form] = LiveInfer(LiveArguments(), model=model, tokenizer=tok)
    states = {f: s.suspend() for f, s in sessions.items()}
    assert states["int4"].int4_weights and not states["int4"].fp8_weights
    assert not states["bf16"].int4_weights and not states["fp8"].int4_weights
    for theirs in states:
        for ours in sessions:
            if theirs != ours:
                with pytest.raises(VloError, match=f"written with {'FP8' if theirs == 'fp8' else theirs} layer weights, "
                                                   f"this model has {'FP8' if ours == 'fp8' else ours} ones"):
                    sessions[ours].resume(states[theirs])
    for f in sessions:
        sessions[f].resume(states[f])


# ============================================================================================ full size, reported
def test_full_size_int4_vs_bf16_and_fp8_report():
    """32-layer Llama-3-8B-width synthetic stack at 12k keys, 11-token frame steps, 64 steps on a bf16, an FP8-weight
    and an int4 engine of the same seed: logit rms / max difference, correlation, argmax and speak / silent agreement of
    int4 against bf16 and against FP8 are printed and appended to VLO_PARITY_LOG; only finiteness is asserted
    (synthetic weights say little about answer quality)."""
    import json
    from videollm_online_b200 import llama3_8b_siglip_l
    from videollm_online_b200.modeling_live import build_live
    cfg = llama3_8b_siglip_l()
    fill, steps, q = 12288, 64, 11
    res = {}
    for form in ("bf16", "fp8", "int4"):
        model, _ = build_live(config=cfg, synthetic_weights=True, seed=0, set_vision_inside=False, device="cuda:0",
                              max_streams=1, max_kv_tokens=fill + steps * q + 64, max_step_tokens=128, max_vit_batch=1,
                              fp8_weights=form == "fp8", int4_weights=form == "int4")
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
        res[form] = (torch.stack(logits), speak)
        eng.close()
        del model, eng
        torch.cuda.empty_cache()
    b = res["int4"][0]
    assert bool(torch.isfinite(b).all())
    log = os.environ.get("VLO_PARITY_LOG")
    for ref in ("bf16", "fp8"):
        a = res[ref][0]
        assert bool(torch.isfinite(a).all())
        d = b - a
        rep = {"test": f"int4_weights_vs_{ref}_full_size", "steps": steps, "keys": fill, "q": q,
               "logit_rms_diff": d.pow(2).mean().sqrt().item(), "logit_max_diff": d.abs().max().item(),
               "logit_rms": a.pow(2).mean().sqrt().item(),
               "corr": torch.corrcoef(torch.stack([a.flatten(), b.flatten()]))[0, 1].item(),
               "argmax_agree": (a.argmax(-1) == b.argmax(-1)).float().mean().item(),
               "speak_agree": sum(x == y for x, y in zip(res[ref][1], res["int4"][1])) / steps,
               "gpu": torch.cuda.get_device_name(0)}
        print(json.dumps(rep))
        if log:
            with open(log, "a") as fh:
                fh.write(json.dumps(rep) + "\n")
