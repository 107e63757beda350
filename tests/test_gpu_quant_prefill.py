"""Prefill on quantized layer matrices (vlo_set_quantized_prefill, gemm_prefill_q_kernel) against the chunked path of
the same weight format, bit for bit.

A.  gemm_prefill_q_kernel: int4 against the bf16 prefill kernel on W4 = dequantize_int4_groups(q, s); e4m3 weights and
    W8A8 against vlo_op_gemm_ws_{f8,a8} mode 0 on each 128-token chunk followed by the fix-up kernels' plane sum (one
    fp32 plane), and against vlo_op_gemm_swiglu_{f8,a8} on each chunk.  Llama-3-8B widths, the tiny and odd shapes,
    T = 129 .. 1024, plans of 7, 37 and all SMs and one with 8 planes.  Rows past T hold NaN and must keep it.
B.  An engine of each form with quantized_prefill: one stream's long input (prefill) against the same input fed as
    explicit max_step_tokens steps on the same engine, from kv_len 0, from an unaligned kv_len on a fragmented pool and
    after kv_evict, with and without quantized vocabulary matrices; a 2-layer full-width stack, PDL off, pages that held
    non-finite values, pool exhaustion, bad arguments, the finalize rules and the device memory the flag adds.
C.  forward_all_logits, stream_evaluate and fast_greedy_generate on int4 and W8A8 engines with the flag against the same
    engines without it; StreamScheduler's ticks; SessionState round trips between the two.
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
import test_gpu_decoder_kernels as DK  # noqa: E402  (stream-K plane counts, SM count)

FMT_E4M3, FMT_E4M3_A8, FMT_I4 = 2, 3, 4
FIX_MAX_PLANES = 8
PREFILL_PLANE, PREFILL_SWIGLU = 0, 1
FORMS = ["fp8", "w8a8", "int4"]


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


def _same_bits(got, want, what):
    ok = (got.view(torch.int32 if got.dtype == torch.float32 else torch.int16) ==
          want.view(torch.int32 if want.dtype == torch.float32 else torch.int16))
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:4].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} entries differ; at {bad} got "
                             f"{[got[tuple(i)].item() for i in bad]}, want {[want[tuple(i)].item() for i in bad]}")


# ============================================================================================ A: the kernel
PREFILL_T = [129, 200, 1000, 1024]
LLAMA_SHAPES = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]  # q|k|v, o_proj, gate|up, down of Llama-3-8B
TINY_SHAPES = [(1024, 256), (256, 512)]
ODD_SHAPE = (1000, 1024)


@pytest.fixture(scope="module")
def operands():
    """per (form, N, K): the weight operand and 1024 token rows (e4m3 codes + scales for W8A8); the sums are inexact, so
    any change of order shows"""
    from videollm_online_b200 import weights as W
    cache = {}

    def get(form, N, K):
        key = (form, N, K)
        if key not in cache:
            g = torch.Generator(device="cuda").manual_seed(N * 3 + K)
            w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
            x = torch.randn(1024, K, device="cuda", generator=g).bfloat16()
            if form == "int4":
                q, s = W.quantize_int4_groups(w)
                cache[key] = dict(w=W.pack_int4_codes(q), gs=s, w4=W.dequantize_int4_groups(q, s), x=x)
            else:
                codes, scale = W.quantize_fp8_rows(w)
                d = dict(w=codes, scale=scale, x=x)
                if form == "w8a8":
                    d["x8"], d["xs"] = W.quantize_fp8_rows(x)
                cache[key] = d
        return cache[key]
    return get


def _fmt(form):
    return {"fp8": FMT_E4M3, "w8a8": FMT_E4M3_A8, "int4": FMT_I4}[form]


def _x(form, op, T):
    if form == "w8a8":
        return op["x8"][:T].contiguous(), op["xs"][:T].contiguous()
    return op["x"][:T].contiguous(), None


def _prefill_q(lib, form, epi, op, N, K, T, n_ctas, pad=37):
    """gemm_prefill_q into an output with `pad` NaN rows past T, which must keep their NaN"""
    x, xs = _x(form, op, T)
    if epi == PREFILL_PLANE:
        out = torch.full((T + pad, N), float("nan"), device="cuda")
    else:
        out = torch.full((T + pad, N // 2), float("nan"), device="cuda", dtype=torch.bfloat16)
    _check(lib.vlo_op_gemm_prefill_q(_fmt(form), epi, _p(op["w"]), _p(op.get("scale")), _p(op.get("gs")), N, _p(x), _p(xs),
                                     T, K, n_ctas, _p(out), _st()), "gemm_prefill_q")
    torch.cuda.synchronize()
    assert out[T:].isnan().all(), "rows past T were written"
    return out[:T]


def _chunked_plane(lib, form, op, N, K, T, n_ctas):
    """the reference of PREFILL_PLANE: int4, the bf16 prefill on W4 (itself held to the chunked path); e4m3 / W8A8,
    vlo_op_gemm_ws_{f8,a8} mode 0 on each <= 128-row chunk, planes summed as the fix-up kernels do: 0 + P0 + P1 + ..."""
    x, xs = _x(form, op, T)
    if form == "int4":
        out = torch.empty(T, N, device="cuda")
        _check(lib.vlo_op_gemm_prefill(PREFILL_PLANE, _p(op["w4"]), N, _p(x), T, K, n_ctas, _p(out), _st()), "bf16 prefill")
        return out
    ns = torch.tensor(DK._sk_planes(N, K, n_ctas), device="cuda").repeat_interleave(128)[:N]
    outs = []
    for lo in range(0, T, 128):
        xc = x[lo:lo + 128].contiguous()
        t = xc.shape[0]
        planes = C.c_int(0)

        def call(out):
            if form == "fp8":
                return lib.vlo_op_gemm_ws_f8(_p(op["w"]), _p(op["scale"]), N, _p(xc), t, K, _p(out), t * N, n_ctas,
                                             C.byref(planes), _st())
            return lib.vlo_op_gemm_ws_a8(_p(op["w"]), _p(op["scale"]), N, _p(xc), _p(xs[lo:lo + t].contiguous()), t, K,
                                         _p(out), t * N, n_ctas, C.byref(planes), _st())
        _check(call(None), "plan")
        buf = torch.full((planes.value, t, N), float("nan"), device="cuda")
        _check(call(buf), "gemm_ws")
        y = torch.zeros(t, N, device="cuda")
        for s in range(planes.value):
            y = y + torch.where((s < ns)[None, :], buf[s], torch.zeros_like(y))
        outs.append(y)
    return torch.cat(outs, 0)


def _chunked_swiglu(lib, form, op, N, K, T):
    x, xs = _x(form, op, T)
    if form == "int4":
        out = torch.empty(T, N // 2, device="cuda", dtype=torch.bfloat16)
        _check(lib.vlo_op_gemm_prefill(PREFILL_SWIGLU, _p(op["w4"]), N, _p(x), T, K, 0, _p(out), _st()), "bf16 prefill")
        return out
    outs = []
    planes = torch.empty(FIX_MAX_PLANES * 128 * N, device="cuda")
    flags = torch.zeros(N // 128, dtype=torch.int32, device="cuda")
    for lo in range(0, T, 128):
        xc = x[lo:lo + 128].contiguous()
        t = xc.shape[0]
        act = torch.empty(t, N // 2, dtype=torch.bfloat16, device="cuda")
        if form == "fp8":
            rc = lib.vlo_op_gemm_swiglu_f8(_p(op["w"]), _p(op["scale"]), N, _p(xc), t, K, _p(act), _p(planes),
                                           planes.numel(), _p(flags), flags.numel(), _st())
        else:
            rc = lib.vlo_op_gemm_swiglu_a8(_p(op["w"]), _p(op["scale"]), N, _p(xc), _p(xs[lo:lo + t].contiguous()), t, K,
                                           _p(act), _p(planes), planes.numel(), _p(flags), flags.numel(), _st())
        _check(rc, "gemm_swiglu")
        outs.append(act)
    return torch.cat(outs, 0)


@pytest.mark.parametrize("n_ctas", [0, 37, 7])
@pytest.mark.parametrize("T", PREFILL_T)
@pytest.mark.parametrize("N,K", LLAMA_SHAPES + TINY_SHAPES + [ODD_SHAPE])
@pytest.mark.parametrize("form", FORMS)
def test_prefill_q_plane_matches_chunked(lib, operands, form, N, K, T, n_ctas):
    op = operands(form, N, K)
    got = _prefill_q(lib, form, PREFILL_PLANE, op, N, K, T, n_ctas)
    _same_bits(got, _chunked_plane(lib, form, op, N, K, T, n_ctas), f"{form} N={N} K={K} T={T} n_ctas={n_ctas}")


@pytest.mark.parametrize("T", [129, 1000])
@pytest.mark.parametrize("N,K", [(4096, 4096), (256, 512), ODD_SHAPE])
@pytest.mark.parametrize("form", FORMS)
def test_prefill_q_plane_eight_planes(lib, operands, form, N, K, T):
    n_ctas = DK._ctas_for_planes(N, K, FIX_MAX_PLANES)
    op = operands(form, N, K)
    got = _prefill_q(lib, form, PREFILL_PLANE, op, N, K, T, n_ctas)
    _same_bits(got, _chunked_plane(lib, form, op, N, K, T, n_ctas), f"{form} N={N} K={K} T={T} (8 planes)")


@pytest.mark.parametrize("T", PREFILL_T)
@pytest.mark.parametrize("N,K", [(28672, 4096), (1024, 256), (256, 512)])
@pytest.mark.parametrize("form", FORMS)
def test_prefill_q_swiglu_matches_fused_gate_up(lib, operands, form, N, K, T):
    op = operands(form, N, K)
    got = _prefill_q(lib, form, PREFILL_SWIGLU, op, N, K, T, 0)
    _same_bits(got, _chunked_swiglu(lib, form, op, N, K, T), f"{form} gate|up N={N} K={K} T={T}")


def test_prefill_q_bad_arguments(lib, operands):
    from videollm_online_b200._lib import VloError
    f8, a8, i4 = operands("fp8", 256, 512), operands("w8a8", 256, 512), operands("int4", 256, 512)
    out = torch.empty(1024, 256, device="cuda")
    x, x8, xs = f8["x"], a8["x8"], a8["xs"]
    cases = [
        (1, PREFILL_PLANE, f8["w"], f8["scale"], None, 256, x, None, 128, 512),     # bf16 is vlo_op_gemm_prefill's
        (FMT_E4M3, 2, f8["w"], f8["scale"], None, 256, x, None, 128, 512),          # epilogue
        (FMT_E4M3, PREFILL_PLANE, f8["w"], None, None, 256, x, None, 128, 512),     # no row scales
        (FMT_E4M3_A8, PREFILL_PLANE, a8["w"], a8["scale"], None, 256, x8, None, 128, 512),   # no token scales
        (FMT_I4, PREFILL_PLANE, i4["w"], None, None, 256, x, None, 128, 512),       # no group scales
        (FMT_I4, PREFILL_PLANE, i4["w"], None, i4["gs"], 256, x, None, 128, 448),   # K not a multiple of 128
        (FMT_E4M3, PREFILL_PLANE, f8["w"], f8["scale"], None, 256, x, None, 0, 512),     # no rows
        (FMT_E4M3, PREFILL_SWIGLU, f8["w"], f8["scale"], None, 200, x, None, 128, 512),  # SwiGLU on a partial tile
    ]
    for fmt, epi, w, sc, gs, N, xx, xsc, T, K in cases:
        with pytest.raises(VloError):
            _check(lib.vlo_op_gemm_prefill_q(fmt, epi, _p(w), _p(sc), _p(gs), N, _p(xx), _p(xsc), T, K, 0, _p(out), _st()),
                   f"fmt {fmt} epi {epi}")
    _check(lib.vlo_op_gemm_prefill_q(FMT_E4M3_A8, PREFILL_PLANE, _p(a8["w"]), _p(a8["scale"]), None, 256, _p(x8), _p(xs),
                                     128, 512, 0, _p(out), _st()), "the good call")


# ============================================================================================ B: the engine
def _model(cfg, llm, form, max_step_tokens=128, qp=True, vocab=False, max_streams=4, max_kv_tokens=4096,
           kv_pool_tokens=None, vit_batch=1):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=max_step_tokens, max_vit_batch=vit_batch,
                          kv_pool_tokens=kv_pool_tokens, fp8_weights=form in ("fp8", "w8a8"),
                          fp8_activations=form == "w8a8", int4_weights=form == "int4", quantize_vocab=vocab,
                          quantized_prefill=qp)
    return model


@pytest.fixture(scope="module")
def tiny():
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config()
    return cfg, W.synthetic_llm_state(cfg, seed=11)


@pytest.fixture(scope="module")
def models(tiny):
    cfg, llm = tiny
    cache = {}

    def get(form, mst=128, vocab=False):
        key = (form, mst, vocab)
        if key not in cache:
            cache[key] = _model(cfg, llm, form, mst, vocab=vocab)
        return cache[key]
    return get


def _emb(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _feed(eng, sid, emb, cap, ids=None):
    """emb in calls of at most `cap` rows; all-position logits and final hidden rows, then the last call's logits and
    decision row"""
    lg_all, hid, last = [], [], None
    for lo in range(0, emb.shape[0], cap):
        n = min(cap, emb.shape[0] - lo)
        lg, dc = eng.step([sid], [n], emb[lo:lo + n].contiguous(), row_ids=None if ids is None else ids[lo:lo + n])
        last = (lg[0].clone(), dc[0].clone())
        lg_all.append(eng.last_step_logits(n))
        hid.append(eng.last_step_hidden(n))
    return torch.cat(lg_all), torch.cat(hid), last


def _compare_streams(eng, a, b, emb, ids=None):
    """stream a: emb as prefills (calls of max_pass_tokens rows); stream b: the same as max_step_tokens steps"""
    assert eng.prefills and eng.max_pass_tokens == eng.max_prefill_tokens > eng.max_step_tokens
    la, ha, (lga, dca) = _feed(eng, a, emb, eng.max_pass_tokens, ids)
    lb, hb, (lgb, dcb) = _feed(eng, b, emb, eng.max_step_tokens, ids)
    assert eng.kv_len(a) == eng.kv_len(b)
    assert torch.equal(lga, lgb), "last logits"
    assert torch.equal(dca, dcb), "decision row"
    assert torch.equal(la, lb), "all-position logits"
    assert torch.equal(ha, hb), "final hidden rows"
    for l, (x, y) in enumerate(zip(_kv_all(eng, a), _kv_all(eng, b))):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]), f"layer {l} K/V"


@pytest.mark.parametrize("vocab", [False, True])
@pytest.mark.parametrize("L", [129, 1024, 2500])
@pytest.mark.parametrize("form", FORMS)
def test_engine_prefill_from_empty(models, tiny, form, L, vocab):
    cfg, _ = tiny
    eng = models(form, vocab=vocab).engine
    assert eng.max_prefill_tokens == FIX_MAX_PLANES * 128 and eng.quantized_vocab == vocab
    a, b = eng.stream_open(), eng.stream_open()
    try:
        _compare_streams(eng, a, b, _emb(cfg, L, L))
    finally:
        eng.stream_close(a)
        eng.stream_close(b)


@pytest.mark.parametrize("mst", [128, 32])
@pytest.mark.parametrize("form", FORMS)
def test_engine_prefill_unaligned_fragmented(models, tiny, form, mst):
    """after a 37-token step (kv_len not page-aligned), on a pool fragmented by other streams' pages, with row ids"""
    cfg, _ = tiny
    eng = models(form, mst).engine
    a, b, c = eng.stream_open(), eng.stream_open(), eng.stream_open()
    try:
        head = _emb(cfg, 37, 1)
        for s in (a, c, b, c):
            eng.step([s], [37], head)
        eng.stream_close(c)
        c = None
        L = 1025
        emb = _emb(cfg, L, 2)
        ids = torch.full((L,), -1, dtype=torch.int64)
        ids[::7] = torch.arange(0, L, 7) % cfg.vocab_size
        _compare_streams(eng, a, b, emb, ids.cuda())
    finally:
        for s in (a, b, c):
            if s is not None:
                eng.stream_close(s)


@pytest.mark.parametrize("form", FORMS)
def test_engine_prefill_after_evict(models, tiny, form):
    cfg, _ = tiny
    eng = models(form).engine
    a, b = eng.stream_open(), eng.stream_open()
    try:
        eng.kv_fill_synthetic(a, 300, seed=4)
        eng.kv_copy_prefix(a, b, 300)
        for s in (a, b):
            eng.kv_evict(s, 64, 128)
        _compare_streams(eng, a, b, _emb(cfg, 1025, 3))
    finally:
        eng.stream_close(a)
        eng.stream_close(b)


@pytest.mark.parametrize("form", FORMS)
def test_engine_prefill_full_width(form):
    """two full-width Llama-3-8B decoder layers (hidden 4096, 32 / 8 heads, intermediate 14336)"""
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config(hidden_size=4096, num_attention_heads=32, num_key_value_heads=8, intermediate_size=14336)
    eng = _model(cfg, W.synthetic_llm_state(cfg, seed=5), form, max_streams=2, max_kv_tokens=2048).engine
    a, b = eng.stream_open(), eng.stream_open()
    for s in (a, b):
        eng.step([s], [37], _emb(cfg, 37, 8))
    _compare_streams(eng, a, b, _emb(cfg, 1300, 9))


@pytest.mark.parametrize("form", FORMS)
def test_engine_prefill_poisoned_pages(tiny, form):
    """pages that held NaN / +-Inf rows of an earlier stream change nothing"""
    cfg, llm = tiny
    clean = _model(cfg, llm, form, max_streams=2, kv_pool_tokens=4096).engine
    dirty = _model(cfg, llm, form, max_streams=2, kv_pool_tokens=4096).engine
    s = dirty.stream_open()
    n = 4096 - 64
    bad = torch.tensor([float("nan"), float("inf"), float("-inf")]).repeat(n * 128 // 3 + 1)[:n * 128]
    rows = bad.view(n, 128).to(torch.bfloat16).cuda()
    for l in range(cfg.num_hidden_layers):
        for v in (False, True):
            dirty.kv_write(s, l, v, rows.repeat(cfg.num_key_value_heads, 1, 1).view(cfg.num_key_value_heads, n, 128))
    dirty.stream_close(s)
    emb = _emb(cfg, 1025, 12)
    outs = []
    for eng in (clean, dirty):
        sid = eng.stream_open()
        outs.append(_feed(eng, sid, emb, eng.max_pass_tokens) + (_kv_all(eng, sid),))
    (la, ha, (lga, dca), kva), (lb, hb, (lgb, dcb), kvb) = outs
    assert torch.equal(la, lb) and torch.equal(ha, hb) and torch.equal(lga, lgb) and torch.equal(dca, dcb)
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(kva, kvb))


class _CountPrefills:
    def __init__(self, lib):
        self._lib, self.rcs = lib, []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def vlo_prefill(self, *args):
        rc = self._lib.vlo_prefill(*args)
        self.rcs.append(rc)
        return rc


@pytest.mark.parametrize("form", FORMS)
def test_engine_prefill_pool_exhaustion(tiny, form):
    """a 2100-row input is two prefill calls; the second runs out of pages: the stream, its K/V and the free pages are
    as before the call"""
    from videollm_online_b200._lib import VloError
    cfg, llm = tiny
    eng = _model(cfg, llm, form, max_streams=2, kv_pool_tokens=80 * 64).engine
    a, hog = eng.stream_open(), eng.stream_open()
    eng.step([a], [37], _emb(cfg, 37, 1))
    eng.kv_fill_synthetic(hog, 59 * 64, seed=1)
    kv0, free0 = _kv_all(eng, a), eng.kv_pool_info()["free_pages"]
    assert free0 == 20
    spy = _CountPrefills(eng.lib)
    eng.lib = spy
    try:
        with pytest.raises(VloError):
            eng.step([a], [2100], _emb(cfg, 2100, 2))
    finally:
        eng.lib = spy._lib
    assert spy.rcs[0] == 0 and spy.rcs[1] != 0, spy.rcs
    assert eng.kv_len(a) == 37 and eng.kv_pool_info()["free_pages"] == free0
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(kv0, _kv_all(eng, a)))


def test_engine_prefill_bad_arguments(models, tiny):
    from videollm_online_b200._lib import VloError, check
    cfg, _ = tiny
    eng = models("int4").engine
    sid = eng.stream_open()
    emb = _emb(cfg, 1025, 1)
    st = eng._stream()
    try:
        for s, n, e, what in [(sid, 0, emb, "n_tokens 0"), (sid, 1025, emb, "past max_prefill_tokens"),
                              (99, 300, emb, "stream id"), (sid, 300, None, "null embeddings")]:
            with pytest.raises(VloError):
                check(eng.lib.vlo_prefill(eng._h, s, n, None, _p(e), None, None, -1, st), what)
        assert eng.kv_len(sid) == 0
    finally:
        eng.stream_close(sid)


@pytest.mark.parametrize("form", FORMS)
def test_flag_rules(tiny, form):
    """vlo_prefill needs the flag on a quantized engine; the setter fails after finalize; the flag fails on bf16 layers"""
    from videollm_online_b200 import weights as W
    from videollm_online_b200.engine import Engine
    from videollm_online_b200._lib import VloError, check
    cfg, llm = tiny
    eng = _model(cfg, llm, form, max_streams=1, qp=False).engine
    assert not eng.prefills and eng.max_prefill_tokens == 0
    sid = eng.stream_open()
    with pytest.raises(VloError, match="quantized_prefill"):
        check(eng.lib.vlo_prefill(eng._h, sid, 300, None, _p(_emb(cfg, 300, 1)), None, None, -1, eng._stream()), "prefill")
    assert eng.kv_len(sid) == 0
    with pytest.raises(VloError, match="before vlo_finalize_weights"):
        check(eng.lib.vlo_set_quantized_prefill(eng._h, 1), "set_quantized_prefill")
    bf = Engine(cfg, "cuda:0", max_streams=1, max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=1,
                quantized_prefill=True)
    with pytest.raises(VloError, match="bf16"):
        bf.load_weights(W.pack_llm_for_engine(cfg, llm, bf.device, 4096))
    bf.close()


def _act_bytes(cfg, rows):
    """the e4m3 copies of xn, attn_out and act and their three fp32 token scales, 256-byte aligned as allocated"""
    a = lambda n: (n + 255) // 256 * 256
    H, A, I = cfg.hidden_size, cfg.num_attention_heads * cfg.head_dim, cfg.intermediate_size
    return a(rows * H) + a(rows * A) + a(rows * I) + 3 * a(4 * rows)


def test_workspace_growth(tiny):
    """the flag grows a quantized engine's device memory by what bf16 weights grow a bf16 engine's; under W8A8 also by
    the e4m3 activation copies at max_prefill_tokens rows instead of max_step_tokens"""
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    kw = dict(max_streams=2, max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=1)

    def created(**k):
        e = Engine(cfg, "cuda:0", **kw, **k)
        b = e.device_bytes()
        e.close()
        return b
    plain, a8 = created(), created(fp8_activations=True)
    assert _model(cfg, llm, "int4", max_streams=2, qp=False).engine.device_bytes() == plain
    from videollm_online_b200.modeling_live import build_live
    bf, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", **kw)
    growth = bf.engine.device_bytes() - plain
    assert growth > 0
    for form in FORMS:
        eng = _model(cfg, llm, form, max_streams=2).engine
        if form == "w8a8":
            assert eng.device_bytes() - a8 == growth + _act_bytes(cfg, 1024) - _act_bytes(cfg, 128), form
        else:
            assert eng.device_bytes() - plain == growth, form
        assert eng.max_prefill_tokens == 1024


_CHILD = r"""
import sys, torch
sys.path.insert(0, {root!r})
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import tiny_config, weights as W
from videollm_online_b200.modeling_live import build_live
cfg = tiny_config()
out = {{}}
for form in ("fp8", "w8a8", "int4"):
    model, _ = build_live(config=cfg, llm_state=W.synthetic_llm_state(cfg, seed=11), set_vision_inside=False,
                          device="cuda:0", max_streams=1, max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=1,
                          fp8_weights=form != "int4", fp8_activations=form == "w8a8", int4_weights=form == "int4",
                          quantized_prefill=True)
    eng = model.engine
    g = torch.Generator().manual_seed(21)
    emb = torch.randn(2500, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
    sid = eng.stream_open()
    lg, dc = eng.step([sid], [2500], emb)
    out[form] = dict(lg=lg[0].cpu(), dc=dc[0].cpu(), hid=eng.last_step_hidden(2500 - 2048).cpu(),
                     kv=[(eng.kv_read(sid, l, False).cpu(), eng.kv_read(sid, l, True).cpu())
                         for l in range(cfg.num_hidden_layers)])
    del model, eng
torch.save(out, sys.argv[1])
"""


def test_engine_prefill_without_pdl(tmp_path):
    """the same results with PDL off (VLO_NO_PDL=1) and on, for every form"""
    script = tmp_path / "child.py"
    script.write_text(_CHILD.format(root=str(ROOT)))
    res = {}
    for off in (True, False):
        env = dict(os.environ)
        env.pop("VLO_NO_PDL", None)
        if off:
            env["VLO_NO_PDL"] = "1"
        path = tmp_path / f"out{int(off)}.pt"
        r = subprocess.run([sys.executable, str(script), str(path)], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        res[off] = torch.load(path)
    for form in FORMS:
        a, b = res[True][form], res[False][form]
        assert torch.equal(a["lg"], b["lg"]) and torch.equal(a["dc"], b["dc"]) and torch.equal(a["hid"], b["hid"]), form
        assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a["kv"], b["kv"])), form


# ============================================================================================ C: host paths
@pytest.mark.parametrize("form", ["int4", "w8a8"])
def test_forward_all_logits_and_generate(tiny, form):
    from videollm_online_b200.modeling_live import fast_greedy_generate
    cfg, llm = tiny
    emb = _emb(cfg, 700, 5)
    res = []
    for qp in (True, False):
        model = _model(cfg, llm, form, 32, qp=qp, max_streams=2)
        assert model.engine.prefills == qp
        kv = model.new_stream()
        lg = model.forward_all_logits(emb, kv)
        kv2 = model.new_stream()
        buf = torch.zeros(1, 20, dtype=torch.long)
        ids, _ = fast_greedy_generate(model=model, inputs_embeds=emb[None], past_key_values=kv2,
                                      eos_token_id=cfg.eos_token_id, inplace_output_ids=buf)
        res.append((lg, ids.clone(), _kv_all(model.engine, kv2.stream_id)))
        del model
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(res[0][2], res[1][2]))


@pytest.mark.parametrize("form", ["int4", "w8a8"])
def test_stream_evaluate(tiny, form, monkeypatch):
    """tests/test_gpu_prefill.py's conversation (60 frames in 4 turns, the interval id's lm_head row aligned with turn 0's
    frame rows so that the look-ahead branch runs) on an engine with the flag and one without"""
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    g = torch.Generator().manual_seed(7)
    fnt, v = cfg.frame_num_tokens, cfg.v_placeholder_id
    ids, labels, silent = [], [], []
    for turn in range(4):
        for f in range(15):
            ids += [v] * fnt
            labels += [-100] * (fnt - 1) + [cfg.frame_token_interval_id if f < 14 else 5 + turn]
            if turn == 0:
                silent.append(len(ids) - 1)
        words = torch.randint(10, 200, (9,), generator=g).tolist() + [cfg.eos_token_id]
        ids += words
        labels += words[1:] + [-100]
    input_ids = torch.tensor([ids])
    label_ids = torch.tensor([labels])
    feats = torch.randn(60, cfg.frame_num_tokens, cfg.vision_hidden_size, generator=g)

    probe = _model(cfg, llm, form, 32, max_streams=2, vit_batch=60)
    emb = probe.joint_embed(input_ids[0].cuda(), feats.cuda())
    sid = probe.engine.stream_open()
    _, hid, _ = _feed(probe.engine, sid, emb, probe.engine.max_pass_tokens)
    row = hid[silent].float().sum(0)
    sd = dict(llm)
    w = sd["lm_head.weight"].clone()
    w[cfg.frame_token_interval_id] = (row / row.norm() * 40.0).to(w.dtype).to(w.device)
    sd["lm_head.weight"] = w
    del probe

    copies, prefills = [], []
    orig_copy, orig_prefill = Engine.kv_copy_prefix, Engine._prefill
    monkeypatch.setattr(Engine, "kv_copy_prefix", lambda self, *a: (copies.append(a), orig_copy(self, *a))[1])
    monkeypatch.setattr(Engine, "_prefill", lambda self, *a: (prefills.append(a[1]), orig_prefill(self, *a))[1])
    res = []
    for qp in (True, False):
        model = _model(cfg, sd, form, 32, qp=qp, max_streams=2, vit_batch=60)
        out = []
        for thr in (0.0, 0.9):
            n, p = len(copies), len(prefills)
            out.append(model.stream_evaluate(input_ids.cuda(), label_ids.cuda(), feats.cuda(),
                                             frame_token_interval_threshold=thr).cpu())
            assert len(copies) > n, f"the look-ahead branch did not run (thr {thr})"
            assert (len(prefills) > p) == qp
        res.append(out)
        del model
    for a, b in zip(*res):
        assert torch.equal(a, b), (a, b)


def test_scheduler_ticks_and_session_states(tiny):
    """StreamScheduler over an int4 engine with the flag and one without: ragged multi-stream ticks step as before
    (never _prefill), each session's long first prompt prefills alone, and every session ends with the same cache.  A
    LiveInfer state saved on either engine resumes on the other."""
    from videollm_online_b200 import weights as W
    from videollm_online_b200.engine import Engine
    from videollm_online_b200.modeling_live import build_live
    from videollm_online_b200.multistream import StreamScheduler
    from videollm_online_b200.cli import synthetic_clip
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.config import LiveArguments
    cfg, llm = tiny
    vis = W.synthetic_vision_state(cfg, seed=1)
    seen = []
    orig = Engine._step

    def spy(self, stream_ids, q_lens, *a, **k):
        seen.append((self.prefills, len(stream_ids), int(sum(q_lens))))
        return orig(self, stream_ids, q_lens, *a, **k)
    def silent(dec):   # the random model's speak / silent decisions would start responses at arbitrary points
        dec.argmax_id = dec.argmax_prob_id = cfg.frame_token_interval_id
        dec.p_interval = 1.0
        return dec
    caches, states = [], []
    Engine._step = spy
    try:
        for qp in (True, False):
            model, tok = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                                    max_streams=4, max_kv_tokens=2048, max_step_tokens=32, max_vit_batch=8,
                                    int4_weights=True, quantized_prefill=qp)
            sched = StreamScheduler(model, tok, 3, frame_fps=2, system_prompt="a long system prompt " * 12)
            sched.decision_hook = lambda i, dec, n: silent(dec)
            for i, s in enumerate(sched.sessions):
                s.load_video(synthetic_clip(6, cfg.frame_resolution, seed=i))
            for f in range(6):
                for s in sched.sessions:
                    s.input_video_stream(f / 2)
                while sched.tick():
                    pass
            caches.append([_kv_all(model.engine, s.stream_id) for s in sched.sessions])
            inf = LiveInfer(LiveArguments(), model=model, tokenizer=tok)
            inf.decision_hook = lambda dec, n: silent(dec)
            inf.load_video(synthetic_clip(4, cfg.frame_resolution, seed=9))
            for f in range(3):
                inf.input_video_stream(f / 2)
                inf()
            states.append((inf.suspend(), inf))
    finally:
        Engine._step = orig
    assert any(p and n == 1 and t > 32 for p, n, t in seen), "no session prompt prefilled"
    assert any(n > 1 for p, n, t in seen if p), "no ragged tick on the prefilling engine"
    for a, b in zip(*caches):
        assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))
    for (state, _), (_, inf) in ((states[0], states[1]), (states[1], states[0])):
        inf.resume(state)     # no field of the state tells the two engines apart
        inf.load_video(synthetic_clip(4, cfg.frame_resolution, seed=9))   # the video is not part of a state
        inf.input_video_stream(1.5)
        inf()
