"""FP8 activations (W8A8): the per-token e4m3 quantizers bit for bit against weights.quantize_fp8_rows, the e4m3 x e4m3
GEMM planes exactly where the FP8 tensor cores are exact and within a stated bound elsewhere, the fused gate|up, the
engine against the CPU oracle with both operands quantized, and the engine's exactness promises in this mode.

The FP8 wgmma does not accumulate in full IEEE fp32, so exact checks use codes in {-2 .. 2} and power-of-two scales:
every partial sum is then a small integer, the accumulation is exact, and each plane must equal an fp64 emulation of
fl(fl(P_p * w_s[n]) * a_s[t]) over its own k-blocks.
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
import test_gpu_decoder_kernels as DK  # noqa: E402  (exact SwiGLU emulation, stream-K plane counts, SM count)
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


def _qrows(x):
    """weights.quantize_fp8_rows on the CPU, results on x's device: torch's CUDA division by a Python scalar multiplies
    by the reciprocal, so amax / 448 there can differ from the IEEE quotient the rule (and the kernels) use in the last
    bit; the CPU divides exactly"""
    from videollm_online_b200 import weights as W
    q, s = W.quantize_fp8_rows(x.cpu())
    return q.to(x.device), s.to(x.device)


def _deq(codes):
    return codes.view(torch.float8_e4m3fn).double()


# ============================================================================================ quantizers
def _rows(T, K, seed):
    """bf16 [T, K] cycling through: an all-zero row, one outlier 10^4 x the rest, values that land in the e4m3 subnormal
    range after scaling (amax 448 -> scale 1, the rest below 2^-6), and rows holding +amax and -amax"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(T, K, device="cuda", generator=g)
    for t in range(T):
        kind = (t + 1) % 4
        if kind == 0:
            x[t] = 0
        elif kind == 1:
            x[t, (t * 37) % K] = 1e4
        elif kind == 2:
            x[t] = (torch.rand(K, device="cuda", generator=g) * 2 - 1) * 2.0 ** -6
            x[t, (t * 11) % K] = 448.0
        else:
            m = x[t].abs().max()
            x[t, (t * 13) % K], x[t, (t * 17 + 1) % K] = m, -m
    return x.bfloat16()


QUANT_T = [1, 11, 128]


@pytest.mark.parametrize("T", QUANT_T)
@pytest.mark.parametrize("K", [4096, 14336, 256, 512])
def test_quant_rows_bits(lib, K, T):
    x = _rows(T, K, K + T)
    q = torch.full((T, K), 0x7F, dtype=torch.uint8, device="cuda")
    s = torch.full((T,), float("nan"), device="cuda")
    _check(lib.vlo_op_quant_rows_e4m3(_p(x), T, K, _p(q), _p(s), _st()), "quant_rows")
    torch.cuda.synchronize()
    rq, rs = _qrows(x)
    assert torch.equal(s.view(torch.int32), rs.view(torch.int32))
    assert torch.equal(q, rq)


@pytest.mark.parametrize("T", QUANT_T)
@pytest.mark.parametrize("H", [4096, 256])
@pytest.mark.parametrize("with_part", [False, True])
def test_fused_rmsnorm_quant_bits(lib, H, T, with_part):
    """resid_rmsnorm_q8: h and xn bit-identical to the bf16 instance, xq / xs = quantize_fp8_rows(xn)"""
    g = torch.Generator(device="cuda").manual_seed(H + T)
    h0 = _rows(T, H, 3 * T + H)
    w = (1 + 0.1 * torch.randn(H, device="cuda", generator=g)).bfloat16()
    part, k = None, 4096 if H == 4096 else 512   # the o_proj / down_proj K of the config (<= 8 planes either way)
    if with_part:
        planes = max(DK._sk_planes(H, k, 0))
        part = torch.randn(planes, T, H, device="cuda", generator=g) * 0.1
    outs = []
    for fused in (False, True):
        h = h0.clone()
        xn = DK._sentinel(T, H)
        if fused:
            xq = torch.zeros(T, H, dtype=torch.uint8, device="cuda")
            xs = torch.zeros(T, device="cuda")
            _check(lib.vlo_op_resid_rmsnorm_q8(_p(part), k, 0, _p(h), _p(w), _p(xn), None, None, _p(xq), _p(xs), T, H,
                                               DK.EPS, _st()), "resid_rmsnorm_q8")
        else:
            _check(lib.vlo_op_resid_rmsnorm(_p(part), k, 0, _p(h), _p(w), _p(xn), None, None, T, H, DK.EPS, _st()),
                   "resid_rmsnorm")
        torch.cuda.synchronize()
        outs.append((h, xn))
    assert DK._same_bits(outs[0][0], outs[1][0]) and DK._same_bits(outs[0][1], outs[1][1])
    rq, rs = _qrows(outs[1][1])
    assert torch.equal(xs.view(torch.int32), rs.view(torch.int32))
    assert torch.equal(xq, rq)


# ============================================================================================ GEMM planes
LLAMA_SHAPES = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]   # q|k|v, o, gate|up, down of Llama-3-8B
TINY_SHAPES = [(1024, 256), (256, 512)]                                     # tiny_config: q|k|v / gate|up, o / down
A8_ROWS = [1, 11, 16, 17, 33, 64, 90, 128]                                  # token tiles 16 / 32 / 64 / 96 / 128


def _planes_a8(lib, w8, ws, N, x8, xs, T, K, n_ctas):
    planes = C.c_int(0)
    _check(lib.vlo_op_gemm_ws_a8(_p(w8), _p(ws), N, _p(x8), _p(xs), T, K, None, T * N, n_ctas, C.byref(planes), _st()),
           "plan a8")
    out = torch.zeros(planes.value, T, N, device="cuda")
    _check(lib.vlo_op_gemm_ws_a8(_p(w8), _p(ws), N, _p(x8), _p(xs), T, K, _p(out), T * N, n_ctas, C.byref(planes), _st()),
           "gemm_ws_a8")
    return out


def _plan_ranges(N, K, n_ctas):
    """per 128-row tile: the k-block range [lo, hi) of each of its planes (CTA c owns units [c U / G, (c + 1) U / G))"""
    tiles, kb = (N + 127) // 128, K // 64
    U = tiles * kb
    G = min(n_ctas if n_ctas > 0 else DK._n_sm(), U)
    lo = [(c * U) // G for c in range(G + 1)]
    out = []
    for tile in range(tiles):
        a, b = tile * kb, (tile + 1) * kb
        out.append([(max(lo[c], a) - a, min(lo[c + 1], b) - a) for c in range(G) if lo[c] < b and lo[c + 1] > a])
    return out


def _small_int_operands(N, K, T, seed):
    """codes in {-2 .. 2}: dense weights, activations with about one non-zero in 8, so |P| <= 4 K / 8 < 2^13 stays an
    exactly representable partial sum in any accumulation order; power-of-two scales"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    vals = torch.tensor([-2.0, -1.0, 0.0, 1.0, 2.0], device="cuda")
    w = vals[torch.randint(0, 5, (N, K), device="cuda", generator=g)]
    x = vals[torch.randint(0, 5, (T, K), device="cuda", generator=g)]
    x = x * (torch.rand(T, K, device="cuda", generator=g) < 0.125)
    w8 = w.to(torch.float8_e4m3fn).view(torch.uint8)
    x8 = x.to(torch.float8_e4m3fn).view(torch.uint8)
    ws = 2.0 ** ((torch.arange(N, device="cuda") % 7) - 3).float()
    xs = 2.0 ** ((torch.arange(T, device="cuda") % 5) - 2).float()
    return w8, ws, x8, xs


@pytest.mark.parametrize("n_ctas", [0, 37])
@pytest.mark.parametrize("T", A8_ROWS)
@pytest.mark.parametrize("N,K", LLAMA_SHAPES + TINY_SHAPES)
def test_planes_exact_small_integers(lib, N, K, T, n_ctas):
    w8, ws, x8, xs = _small_int_operands(N, K, T, N + K + T)
    out = _planes_a8(lib, w8, ws, N, x8, xs, T, K, n_ctas)
    ranges = _plan_ranges(N, K, n_ctas)
    assert out.shape[0] == max(len(r) for r in ranges)
    wd, xd = _deq(w8), _deq(x8)
    ref = torch.zeros(out.shape, dtype=torch.float64, device="cuda")
    for tile, rr in enumerate(ranges):
        n0, n1 = tile * 128, min(N, tile * 128 + 128)
        k0 = 0
        for p, (a, b) in enumerate(rr):
            P = xd[:, a * 64:b * 64] @ wd[n0:n1, a * 64:b * 64].t()
            ref[p, :, n0:n1] = P * ws[n0:n1].double() * xs[:, None].double()
            k0 = b
        assert k0 == K // 64
    torch.cuda.synchronize()
    assert torch.equal(out, ref.float()), f"{int((out != ref.float()).sum())} plane entries differ"


def _random_operands(N, K, T, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    w8, ws = _qrows((torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16())
    x8, xs = _qrows(torch.randn(T, K, device="cuda", generator=g).bfloat16())
    return w8, ws, x8, xs


# Bound of the FP8 MMA accumulation: the tensor cores add each k32 product into an accumulator held at reduced
# precision (about 13 mantissa bits kept per addition), so an output's error is a sum of roundings of partial sums, each
# at most 2^-13 of |partial| <= sum |a w|.  Over K / 32 additions the roundings behave like a random walk: 2^-10 of
# sum |a w| is several times the worst error expected at K = 14336 and still below the contribution of one 64-wide
# k-block to some output of a T x N result (checked below), so the bound sees a missing k-block.
A8_REL_BOUND = 2.0 ** -10


@pytest.mark.parametrize("n_ctas", [0, 37])
@pytest.mark.parametrize("N,K", [(6144, 4096), (4096, 14336)])
def test_planes_random_within_bound(lib, N, K, n_ctas):
    T = 11
    w8, ws, x8, xs = _random_operands(N, K, T, N + K)
    out = _planes_a8(lib, w8, ws, N, x8, xs, T, K, n_ctas)
    got = DK._fixup_sum(out, torch.tensor(DK._sk_planes(N, K, n_ctas), device="cuda").repeat_interleave(128)[:N]).double()
    a = _deq(x8) * xs[:, None].double()
    w = _deq(w8) * ws[:, None].double()
    ref = a @ w.t()
    bound = A8_REL_BOUND * (a.abs() @ w.abs().t())
    err = (got - ref).abs()
    assert bool((err <= bound).all()), f"worst err / bound {(err / bound).max().item():.3f}"
    # leaving out any one k-block of the reference exceeds the bound somewhere
    for kb in range(K // 64):
        sl = slice(kb * 64, kb * 64 + 64)
        part = a[:, sl] @ w[:, sl].t()
        assert bool(((got - (ref - part)).abs() > bound).any()), f"k-block {kb} not seen"


# ============================================================================================ fused gate|up
@pytest.fixture(scope="module")
def gate_up_a8():
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


@pytest.mark.parametrize("T", A8_ROWS)
def test_fused_gate_up(lib, gate_up_a8, T):
    """vlo_op_gemm_swiglu_a8 = the exact SwiGLU of g | u = bf16(plane sum) in plane order, the planes being those of
    vlo_op_gemm_ws_a8 on the same operands (same planner, token tile and mainloop); then g, u against the fp64 product
    within the accumulation bound.  Counters back at zero, rows past rows_x untouched."""
    codes, scale, x_all = gate_up_a8
    N, K = codes.shape
    I = N // 2
    x8, xs = _qrows(x_all[:T].contiguous())
    ns = DK._sk_planes(N, K, 0)
    planes_buf = torch.full((max(1, max(ns) - 1) * T * N,), float("nan"), device="cuda")
    flags = torch.zeros(N // 128, dtype=torch.int32, device="cuda")
    act = DK._sentinel(T + 3, I)
    _check(lib.vlo_op_gemm_swiglu_a8(_p(codes), _p(scale), N, _p(x8), _p(xs), T, K, _p(act), _p(planes_buf),
                                     planes_buf.numel(), _p(flags), flags.numel(), _st()), "gemm_swiglu_a8")
    torch.cuda.synchronize()
    assert int(flags.abs().sum()) == 0
    assert DK._same_bits(act[T:], DK._sentinel(3, I))
    act = act[:T]
    ref = _planes_a8(lib, codes, scale, N, x8, xs, T, K, 0)
    torch.cuda.synchronize()
    y = DK._fixup_sum(ref, torch.tensor(ns, device="cuda").repeat_interleave(128))
    exact = (_deq(x8) * xs[:, None].double()) @ (_deq(codes) * scale[:, None].double()).t()
    bound = A8_REL_BOUND * ((_deq(x8).abs() * xs[:, None].double()) @ (_deq(codes).abs() * scale[:, None].double()).t())
    assert bool(((y.double() - exact).abs() <= bound).all())
    y = y.bfloat16().double().view(T, I // 64, 2, 64)
    g, u = y[:, :, 0].reshape(T, I), y[:, :, 1].reshape(T, I)
    e = torch.exp(-g)
    silu = torch.where(e > DK.FLT_MAX, -0.0 * g.abs(), g / (1 + e))
    lo, hi = DK._either(silu, DK._silu_delta())
    DK._assert_in(act, [DK._bf(lo * u), DK._bf(hi * u)], f"SwiGLU a8 T={T}")


# ============================================================================================ engine
def _engine(cfg, llm, a8=True, max_streams=2, max_kv_tokens=2048):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, fp8_weights=True,
                          fp8_activations=a8)
    return model.engine


@pytest.fixture(scope="module")
def tiny():
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config()
    llm = W.synthetic_llm_state(cfg, seed=0)
    llm["lm_head.weight"] = (llm["lm_head.weight"].float() * 8).to(torch.bfloat16)
    return cfg, llm


class _W8A8:
    """oracle Linear of the mode: x quantized per row (quantize_fp8_rows), times the dequantized per-row-quantized
    weight, in fp64; the lm_head stays unquantized"""
    @staticmethod
    def linear(x, sd, module):
        from videollm_online_b200 import weights as W
        w = sd[module + ".weight"]
        if not module.startswith("model.layers."):
            return torch.nn.functional.linear(x, w)
        shp = x.shape
        xq, xs = W.quantize_fp8_rows(x.reshape(-1, shp[-1]))
        wq, ws = W.quantize_fp8_rows(w)
        y = (xq.view(torch.float8_e4m3fn).double() * xs.double()[:, None]) @ \
            (wq.view(torch.float8_e4m3fn).double() * ws.double()[:, None]).t()
        return y.to(x.dtype).reshape(*shp[:-1], w.shape[0])


def test_engine_vs_oracle(tiny):
    """all-position logits of the W8A8 engine vs the CPU oracle with both operands quantized within 0.25 + 0.02 |x|;
    greedy ids exact where the oracle's top-2 margin exceeds 0.5"""
    sys.path.insert(0, str(ROOT / "oracle"))
    import vlo_oracle as O
    cfg, llm = tiny
    eng = _engine(cfg, llm)
    assert eng.fp8_weights and eng.fp8_activations
    sid = eng.stream_open()
    g = torch.Generator().manual_seed(4)
    emb = torch.randn(40, cfg.hidden_size, generator=g).bfloat16()
    eng.step([sid], [40], emb.cuda())
    got = eng.last_step_logits(40).float().cpu()
    ref = O.llama_forward(llm, cfg, emb, O.KVCache(cfg.num_hidden_layers), lora=_W8A8()).float()
    err = (got - ref).abs()
    assert bool((err <= 0.25 + 0.02 * ref.abs()).all()), f"worst {err.max().item()}"
    top2 = ref.topk(2, dim=-1).values
    sure = (top2[:, 0] - top2[:, 1]) > 0.5
    assert int(sure.sum()) > 0
    assert torch.equal(got.argmax(-1)[sure], ref.argmax(-1)[sure])


def test_segmented_backlog_equals_one_frame_per_step(tiny):
    cfg, llm = tiny
    eng = _engine(cfg, llm)
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
    cfg, llm = tiny
    eng = _engine(cfg, llm)
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
    eng = _engine(cfg, llm, max_streams=3)
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
    eng = _engine(cfg, llm)
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


# ============================================================================================ errors / isolation
def test_mode_on_bf16_weights_fails_at_finalize(tiny):
    from videollm_online_b200 import weights as W
    from videollm_online_b200._lib import VloError
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    eng = Engine(cfg, "cuda:0", max_streams=1, max_kv_tokens=256, max_step_tokens=32, max_vit_batch=1,
                 fp8_activations=True)
    try:
        with pytest.raises(VloError, match="fp8_activations needs FP8"):
            eng.load_weights(W.pack_llm_for_engine(cfg, llm, "cuda:0", 512))
    finally:
        eng.close()


def test_mode_after_finalize_fails(tiny):
    from videollm_online_b200._lib import VloError, check
    cfg, llm = tiny
    eng = _engine(cfg, llm, a8=False)
    with pytest.raises(VloError, match="before vlo_finalize_weights"):
        check(eng.lib.vlo_set_fp8_activations(eng._h, 1), "vlo_set_fp8_activations")
    assert not eng.fp8_activations


def test_build_live_needs_fp8_weights(tiny):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm = tiny
    with pytest.raises(ValueError, match="fp8_activations needs fp8_weights"):
        build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=1, max_kv_tokens=256,
                   max_step_tokens=32, max_vit_batch=1, fp8_activations=True)


def test_resume_rejects_a_state_of_the_other_mode(tiny):
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200._lib import VloError
    from videollm_online_b200 import weights as W
    cfg, llm = tiny
    vis = W.synthetic_vision_state(cfg, seed=1)
    sessions = {}
    for a8 in (False, True):
        model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                                max_streams=1, max_kv_tokens=512, max_step_tokens=64, max_vit_batch=2, fp8_weights=True,
                                fp8_activations=a8)
        sessions[a8] = LiveInfer(LiveArguments(), model=model, tokenizer=tok)
    state = sessions[False].suspend()
    assert state.fp8_activations is False
    with pytest.raises(VloError, match="bf16 layer activations"):
        sessions[True].resume(state)
    sessions[False].resume(state)
    state8 = sessions[True].suspend()
    assert state8.fp8_activations is True
    with pytest.raises(VloError, match="FP8 layer activations"):
        sessions[False].resume(state8)


def test_default_engine_bytes_and_launches(tiny):
    """the mode adds exactly its e4m3 copies and scales to the device bytes and two launches per layer to a step; a
    default engine holds neither"""
    from videollm_online_b200 import _lib
    cfg, llm = tiny
    lib = _lib.load()
    engs = {a8: _engine(cfg, llm, a8=a8) for a8 in (False, True)}
    T, H, I, A = 128, cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads * cfg.head_dim
    al = lambda n: (n + 255) // 256 * 256   # noqa: E731
    extra = al(T * H) + al(T * A) + al(T * I) + 3 * al(4 * T)
    assert engs[True].device_bytes() - engs[False].device_bytes() == extra
    launches = {}
    for a8, eng in engs.items():
        sid = eng.stream_open()
        emb = torch.zeros(11, H, dtype=torch.bfloat16, device="cuda")
        eng.step([sid], [11], emb)
        torch.cuda.synchronize()
        n0 = lib.vlo_launch_count()
        eng.step([sid], [11], emb)
        torch.cuda.synchronize()
        launches[a8] = lib.vlo_launch_count() - n0
    assert launches[True] - launches[False] == 2 * cfg.num_hidden_layers


# ============================================================================================ full size, reported
def test_full_size_w8a8_report():
    """32-layer Llama-3-8B-width synthetic stack at 12k keys, 11-token frame steps, 64 steps on a bf16, an FP8-weight and
    a W8A8 engine of the same seed: logit rms / max difference, correlation and speak / silent agreement of W8A8 against
    each are printed and appended to VLO_PARITY_LOG; loose bounds only (synthetic weights say little about answer
    quality, which is not measured on the real checkpoint)."""
    import json
    from videollm_online_b200 import llama3_8b_siglip_l
    from videollm_online_b200.modeling_live import build_live
    cfg = llama3_8b_siglip_l()
    fill, steps, q = 12288, 64, 11
    res = {}
    for mode in ("bf16", "fp8", "w8a8"):
        model, _ = build_live(config=cfg, synthetic_weights=True, seed=0, set_vision_inside=False, device="cuda:0",
                              max_streams=1, max_kv_tokens=fill + steps * q + 64, max_step_tokens=128, max_vit_batch=1,
                              fp8_weights=mode != "bf16", fp8_activations=mode == "w8a8")
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
        res[mode] = (torch.stack(logits), speak)
        del model, eng
        torch.cuda.empty_cache()
    b = res["w8a8"][0]
    assert bool(torch.isfinite(b).all())
    rep = {"test": "w8a8_full_size", "steps": steps, "keys": fill, "q": q, "gpu": torch.cuda.get_device_name(0)}
    for ref in ("bf16", "fp8"):
        a = res[ref][0]
        d = b - a
        rep[ref] = {"logit_rms_diff": d.pow(2).mean().sqrt().item(), "logit_max_diff": d.abs().max().item(),
                    "logit_rms": a.pow(2).mean().sqrt().item(),
                    "corr": torch.corrcoef(torch.stack([a.flatten(), b.flatten()]))[0, 1].item(),
                    "speak_agree": sum(x == y for x, y in zip(res[ref][1], res["w8a8"][1])) / steps}
        assert rep[ref]["corr"] > 0.5 and rep[ref]["logit_rms_diff"] < rep[ref]["logit_rms"]
    print(json.dumps(rep))
    log = os.environ.get("VLO_PARITY_LOG")
    if log:
        with open(log, "a") as fh:
            fh.write(json.dumps(rep) + "\n")
