"""Prefill (vlo_prefill, gemm_prefill_kernel) against the chunked path, bit for bit.

A.  gemm_prefill_kernel against gemm_ws_kernel mode 0 on each 128-token chunk followed by the fix-up kernels' plane sum
    (one fp32 plane), and against the fused gate|up GEMM + SwiGLU on each chunk (act): Llama-3-8B widths, the tiny and
    odd shapes, T = 129 .. 1024, plans of 7, 37 and all SMs and one with 8 planes.  Rows past T hold NaN and must keep it.
B.  An engine's one-stream input longer than max_step_tokens (prefill) against the same input fed as explicit steps of
    max_step_tokens: last logits, decision rows, all-position logits, final hidden rows and every layer's K and V, from
    kv_len 0, from a kv_len that is not page-aligned, on a fragmented pool and after kv_evict; also a 2-layer full-width
    stack, with PDL off, over a pool whose pages held non-finite values, on pool exhaustion and on bad arguments.
C.  forward_all_logits, stream_evaluate and fast_greedy_generate against the explicit-step loop; e4m3-weight engines and
    ragged multi-stream inputs still take the chunked path.
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

FMT_BF16 = 1
ACT_NONE = 0
WS_TILE_FIT = 0
FIX_MAX_PLANES = 8
PREFILL_PLANE, PREFILL_SWIGLU = 0, 1


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


# ============================================================================================ A: the kernel
PREFILL_T = [129, 200, 256, 1000, 1024]
LLAMA_SHAPES = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]  # q|k|v, o_proj, gate|up, down of Llama-3-8B
TINY_SHAPES = [(1024, 256), (256, 512)]
ODD_SHAPE = (1000, 1024)


@pytest.fixture(scope="module")
def operands():
    """per (N, K): random bf16 w [N, K] and 1024 token rows; the sums are inexact, so any change of order shows"""
    cache = {}

    def get(N, K):
        if (N, K) not in cache:
            g = torch.Generator(device="cuda").manual_seed(N * 3 + K)
            w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
            x = torch.randn(1024, K, device="cuda", generator=g).bfloat16()
            cache[(N, K)] = (w, x)
        return cache[(N, K)]
    return get


def _chunked_plane(lib, w, x, n_ctas):
    """gemm_ws mode 0 on each <= 128-row chunk, planes summed as the fix-up kernels do: 0 + P0 + P1 + ... in fp32"""
    N, K = w.shape
    ns = torch.tensor(DK._sk_planes(N, K, n_ctas), device="cuda").repeat_interleave(128)[:N]
    outs = []
    for lo in range(0, x.shape[0], 128):
        xc = x[lo:lo + 128].contiguous()
        t = xc.shape[0]
        plan = (C.c_int32 * 3)()
        _check(lib.vlo_op_gemm_ws_tiled(FMT_BF16, 0, _p(w), N, _p(xc), t, K, None, N, t * N, None, ACT_NONE, n_ctas, 0,
                                        WS_TILE_FIT, plan, _st()), "plan")
        planes = torch.full((plan[2], t, N), float("nan"), device="cuda")
        _check(lib.vlo_op_gemm_ws_tiled(FMT_BF16, 0, _p(w), N, _p(xc), t, K, _p(planes), N, t * N, None, ACT_NONE,
                                        n_ctas, 0, WS_TILE_FIT, plan, _st()), "gemm_ws")
        y = torch.zeros(t, N, device="cuda")
        for s in range(plan[2]):
            y = y + torch.where((s < ns)[None, :], planes[s], torch.zeros_like(y))
        outs.append(y)
    return torch.cat(outs, 0)


def _chunked_swiglu(lib, w, x):
    N, K = w.shape
    outs = []
    planes = torch.empty(FIX_MAX_PLANES * 128 * N, device="cuda")
    flags = torch.zeros(N // 128, dtype=torch.int32, device="cuda")
    for lo in range(0, x.shape[0], 128):
        xc = x[lo:lo + 128].contiguous()
        act = torch.empty(xc.shape[0], N // 2, dtype=torch.bfloat16, device="cuda")
        _check(lib.vlo_op_gemm_swiglu(_p(w), N, _p(xc), xc.shape[0], K, _p(act), _p(planes), planes.numel(), _p(flags),
                                      flags.numel(), _st()), "gemm_swiglu")
        outs.append(act)
    return torch.cat(outs, 0)


def _prefill(lib, epi, w, x, n_ctas, pad=37):
    """gemm_prefill into an output with `pad` NaN rows past T, which must keep their NaN"""
    N, K = w.shape
    T = x.shape[0]
    if epi == PREFILL_PLANE:
        out = torch.full((T + pad, N), float("nan"), device="cuda")
    else:
        out = torch.full((T + pad, N // 2), float("nan"), device="cuda", dtype=torch.bfloat16)
    _check(lib.vlo_op_gemm_prefill(epi, _p(w), N, _p(x), T, K, n_ctas, _p(out), _st()), "gemm_prefill")
    torch.cuda.synchronize()
    assert out[T:].isnan().all(), "rows past T were written"
    return out[:T]


def _same_bits(got, want, what):
    ok = (got.view(torch.int32 if got.dtype == torch.float32 else torch.int16) ==
          want.view(torch.int32 if want.dtype == torch.float32 else torch.int16))
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:4].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} entries differ; at {bad} got "
                             f"{[got[tuple(i)].item() for i in bad]}, want {[want[tuple(i)].item() for i in bad]}")


@pytest.mark.parametrize("n_ctas", [0, 37, 7])
@pytest.mark.parametrize("T", PREFILL_T)
@pytest.mark.parametrize("N,K", LLAMA_SHAPES + TINY_SHAPES + [ODD_SHAPE])
def test_prefill_plane_matches_chunked(lib, operands, N, K, T, n_ctas):
    w, x_all = operands(N, K)
    x = x_all[:T].contiguous()
    got = _prefill(lib, PREFILL_PLANE, w, x, n_ctas)
    _same_bits(got, _chunked_plane(lib, w, x, n_ctas), f"N={N} K={K} T={T} n_ctas={n_ctas}")


@pytest.mark.parametrize("T", [129, 1000])
@pytest.mark.parametrize("N,K", [(4096, 4096), (256, 512), ODD_SHAPE])
def test_prefill_plane_eight_planes(lib, operands, N, K, T):
    n_ctas = DK._ctas_for_planes(N, K, FIX_MAX_PLANES)
    w, x_all = operands(N, K)
    x = x_all[:T].contiguous()
    got = _prefill(lib, PREFILL_PLANE, w, x, n_ctas)
    _same_bits(got, _chunked_plane(lib, w, x, n_ctas), f"N={N} K={K} T={T} n_ctas={n_ctas} (8 planes)")


@pytest.mark.parametrize("T", PREFILL_T)
@pytest.mark.parametrize("N,K", [(28672, 4096), (1024, 256), (256, 512)])
def test_prefill_swiglu_matches_fused_gate_up(lib, operands, N, K, T):
    w, x_all = operands(N, K)
    x = x_all[:T].contiguous()
    got = _prefill(lib, PREFILL_SWIGLU, w, x, 0)
    _same_bits(got, _chunked_swiglu(lib, w, x), f"gate|up N={N} K={K} T={T}")


def test_prefill_op_bad_arguments(lib, operands):
    from videollm_online_b200._lib import VloError
    w, x = operands(256, 512)
    out = torch.empty(1024, 256, device="cuda")
    for args in [(2, 256, 128, 512, 0), (PREFILL_PLANE, 256, 0, 512, 0), (PREFILL_PLANE, 256, 128, 500, 0),
                 (PREFILL_SWIGLU, 200, 128, 512, 0)]:
        epi, N, T, K, n = args
        with pytest.raises(VloError):
            _check(lib.vlo_op_gemm_prefill(epi, _p(w), N, _p(x), T, K, n, _p(out), _st()), "gemm_prefill")


# ============================================================================================ B: the engine
def _model(cfg, llm, max_step_tokens, max_streams=4, max_kv_tokens=4096, kv_pool_tokens=None, fp8=False, vit_batch=1,
           a8=False):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=max_step_tokens, max_vit_batch=vit_batch,
                          kv_pool_tokens=kv_pool_tokens, fp8_weights=fp8, fp8_activations=a8)
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

    def get(mst):
        if mst not in cache:
            cache[mst] = _model(cfg, llm, mst)
        return cache[mst]
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


def _one_call_vs_steps(eng, a, b, emb):
    """one step call of the whole input (prefill route) against explicit max_step_tokens steps"""
    lga, dca = eng.step([a], [emb.shape[0]], emb)
    lga, dca = lga[0].clone(), dca[0].clone()
    for lo in range(0, emb.shape[0], eng.max_step_tokens):
        piece = emb[lo:lo + eng.max_step_tokens].contiguous()
        lgb, dcb = eng.step([b], [piece.shape[0]], piece)
    assert torch.equal(lga, lgb[0]) and torch.equal(dca, dcb[0])
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(_kv_all(eng, a), _kv_all(eng, b)))


LENGTHS = [129, 300, 1024, 1025, 2500]


@pytest.mark.parametrize("L", LENGTHS)
@pytest.mark.parametrize("mst", [128, 32])
def test_engine_prefill_from_empty(models, tiny, mst, L):
    cfg, _ = tiny
    eng = models(mst).engine
    assert eng.max_prefill_tokens == FIX_MAX_PLANES * mst
    a, b = eng.stream_open(), eng.stream_open()
    try:
        emb = _emb(cfg, L, L + mst)
        _compare_streams(eng, a, b, emb)
        eng.stream_reset(a)
        eng.stream_reset(b)
        _one_call_vs_steps(eng, a, b, emb)
    finally:
        eng.stream_close(a)
        eng.stream_close(b)


@pytest.mark.parametrize("L", [300, 1025])
@pytest.mark.parametrize("mst", [128, 32])
def test_engine_prefill_unaligned_fragmented(models, tiny, mst, L):
    """after a 37-token step (kv_len not page-aligned), on a pool fragmented by other streams' pages, with row ids"""
    cfg, _ = tiny
    eng = models(mst).engine
    a, b, c = eng.stream_open(), eng.stream_open(), eng.stream_open()
    try:
        head = _emb(cfg, 37, 1)
        for s in (a, c, b, c):
            eng.step([s], [37], head)
        eng.stream_close(c)
        c = None
        emb = _emb(cfg, L, 2)
        ids = torch.full((L,), -1, dtype=torch.int64)
        ids[::7] = torch.arange(0, L, 7) % cfg.vocab_size
        _compare_streams(eng, a, b, emb, ids.cuda())
    finally:
        for s in (a, b, c):
            if s is not None:
                eng.stream_close(s)


@pytest.mark.parametrize("mst", [128, 32])
def test_engine_prefill_after_evict(models, tiny, mst):
    cfg, _ = tiny
    eng = models(mst).engine
    a, b = eng.stream_open(), eng.stream_open()
    try:
        eng.kv_fill_synthetic(a, 300, seed=4)
        eng.kv_copy_prefix(a, b, 300)      # the synthetic fill depends on the stream: copy it to have two equal caches
        for s in (a, b):
            eng.kv_evict(s, 64, 128)
        _compare_streams(eng, a, b, _emb(cfg, 1025, 3))
    finally:
        eng.stream_close(a)
        eng.stream_close(b)


def test_engine_prefill_full_width(lib):
    """two full-width Llama-3-8B decoder layers (hidden 4096, 32 / 8 heads, intermediate 14336)"""
    from videollm_online_b200 import tiny_config, weights as W
    cfg = tiny_config(hidden_size=4096, num_attention_heads=32, num_key_value_heads=8, intermediate_size=14336)
    eng = _model(cfg, W.synthetic_llm_state(cfg, seed=5), 128, max_streams=2, max_kv_tokens=2048).engine
    a, b = eng.stream_open(), eng.stream_open()
    for s in (a, b):
        eng.step([s], [37], _emb(cfg, 37, 8))
    _compare_streams(eng, a, b, _emb(cfg, 1300, 9))


def test_engine_prefill_poisoned_pages(tiny):
    """pages that held NaN / +-Inf rows of an earlier stream change nothing: a fresh engine over a clean pool gives the
    same bits"""
    cfg, llm = tiny
    clean = _model(cfg, llm, 128, max_streams=2, kv_pool_tokens=4096).engine
    dirty = _model(cfg, llm, 128, max_streams=2, kv_pool_tokens=4096).engine
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
    """the engine's library with its vlo_prefill calls and their return codes recorded"""

    def __init__(self, lib):
        self._lib, self.rcs = lib, []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def vlo_prefill(self, *args):
        rc = self._lib.vlo_prefill(*args)
        self.rcs.append(rc)
        return rc


def test_engine_prefill_pool_exhaustion(tiny):
    """a 2100-row input is two prefill calls: the first takes 16 of the 20 free pages and commits, the second needs 16
    more and fails; the call then gives the first call's pages back, so neither the stream, its K/V nor the free pages
    change, and the same call runs once the pool has room"""
    from videollm_online_b200._lib import VloError
    cfg, llm = tiny
    eng = _model(cfg, llm, 128, max_streams=2, kv_pool_tokens=80 * 64).engine
    a, hog = eng.stream_open(), eng.stream_open()
    eng.step([a], [37], _emb(cfg, 37, 1))
    eng.kv_fill_synthetic(hog, 59 * 64, seed=1)
    kv0, free0 = _kv_all(eng, a), eng.kv_pool_info()["free_pages"]
    assert free0 == 20
    emb = _emb(cfg, 2100, 2)
    spy = _CountPrefills(eng.lib)
    eng.lib = spy
    try:
        with pytest.raises(VloError):
            eng.step([a], [2100], emb)
    finally:
        eng.lib = spy._lib
    assert spy.rcs[0] == 0 and spy.rcs[1] != 0, spy.rcs     # the first call ran, the second one ran out of pages
    assert eng.kv_len(a) == 37 and eng.kv_pool_info()["free_pages"] == free0
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(kv0, _kv_all(eng, a)))
    eng.stream_close(hog)
    b = eng.stream_open()     # room for both: 34 pages each
    eng.step([b], [37], _emb(cfg, 37, 1))
    for lo in range(0, 2100, 128):      # the reference: the same rows as explicit steps on a second stream
        eng.step([b], [min(128, 2100 - lo)], emb[lo:lo + 128].contiguous())
    lg, dc = eng.step([a], [2100], emb)
    assert eng.kv_len(a) == 2137
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(_kv_all(eng, a), _kv_all(eng, b)))


def test_engine_prefill_bad_arguments(models, tiny):
    from videollm_online_b200._lib import VloError, check
    cfg, _ = tiny
    eng = models(128).engine
    sid = eng.stream_open()
    emb = _emb(cfg, 1025, 1)
    lib = eng.lib
    st = eng._stream()
    try:
        for args, what in [((sid, 0), "n_tokens 0"), ((sid, 1025), "past max_prefill_tokens"), ((99, 300), "stream id"),
                           ((sid, 300, False), "null embeddings")]:
            s, n = args[0], args[1]
            e = None if len(args) > 2 else _p(emb)
            with pytest.raises(VloError):
                check(lib.vlo_prefill(eng._h, s, n, None, e, None, None, -1, st), what)
        assert eng.kv_len(sid) == 0
    finally:
        eng.stream_close(sid)


_CHILD = r"""
import sys, torch
sys.path.insert(0, {root!r})
import vlo_bootstrap  # noqa: F401
from videollm_online_b200 import tiny_config, weights as W
from videollm_online_b200.modeling_live import build_live
cfg = tiny_config()
model, _ = build_live(config=cfg, llm_state=W.synthetic_llm_state(cfg, seed=11), set_vision_inside=False, device="cuda:0",
                      max_streams=1, max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=1)
eng = model.engine
g = torch.Generator().manual_seed(21)
emb = torch.randn(2500, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()
sid = eng.stream_open()
lg, dc = eng.step([sid], [2500], emb)
out = dict(lg=lg[0].cpu(), dc=dc[0].cpu(), hid=eng.last_step_hidden(2500 - 2048).cpu(),
           kv=[(eng.kv_read(sid, l, False).cpu(), eng.kv_read(sid, l, True).cpu()) for l in range(cfg.num_hidden_layers)])
torch.save(out, sys.argv[1])
"""


def test_engine_prefill_without_pdl(tmp_path):
    """the same results with PDL off (VLO_NO_PDL=1) and on"""
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
    a, b = res[True], res[False]
    assert torch.equal(a["lg"], b["lg"]) and torch.equal(a["dc"], b["dc"]) and torch.equal(a["hid"], b["hid"])
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a["kv"], b["kv"]))


# ============================================================================================ C: host paths
@pytest.fixture
def no_prefill(monkeypatch):
    """the explicit-step loop: the engine chunks every long input into max_step_tokens steps"""
    from videollm_online_b200.engine import Engine

    def off():
        monkeypatch.setattr(Engine, "prefills", property(lambda self: False))
    return off


def test_forward_all_logits_and_generate(models, tiny, no_prefill):
    from videollm_online_b200.modeling_live import fast_greedy_generate
    cfg, _ = tiny
    model = models(32)
    emb = _emb(cfg, 700, 5)
    res = []
    for run in range(2):
        if run == 1:
            no_prefill()
        kv = model.new_stream()
        lg = model.forward_all_logits(emb, kv)
        kv2 = model.new_stream()
        buf = torch.zeros(1, 20, dtype=torch.long)
        ids, _ = fast_greedy_generate(model=model, inputs_embeds=emb[None], past_key_values=kv2,
                                      eos_token_id=cfg.eos_token_id, inplace_output_ids=buf)
        res.append((lg, ids.clone(), _kv_all(model.engine, kv2.stream_id)))
        model.engine.stream_close(kv.stream_id)
        model.engine.stream_close(kv2.stream_id)
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])
    assert all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(res[0][2], res[1][2]))


def test_stream_evaluate(tiny, no_prefill, monkeypatch):
    """a synthetic conversation of 60 frames in 4 turns, with and without the look-ahead threshold.  Random weights never
    predict the interval id, so the interval id's lm_head row is aligned with the final hidden states of turn 0's frame
    rows (as tests/golden/make_golden.py does): turn 0 reads as silent and takes the look-ahead branch, which copies the
    cache prefix to a scratch stream and appends the next turn's 14 frames (154 rows: a prefill at max_step_tokens 32)"""
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
    assert 14 * (fnt + 1) > 32 and input_ids.shape[1] > 8 * 32

    # the final hidden states of the conversation under the given weights (the lm_head row does not change them)
    probe = _model(cfg, llm, 32, max_streams=2, vit_batch=60)
    emb = probe.joint_embed(input_ids[0].cuda(), feats.cuda())
    sid = probe.engine.stream_open()
    _, hid, _ = _feed(probe.engine, sid, emb, probe.engine.max_pass_tokens)
    row = hid[silent].float().sum(0)
    sd = dict(llm)
    w = sd["lm_head.weight"].clone()
    w[cfg.frame_token_interval_id] = (row / row.norm() * 40.0).to(w.dtype).to(w.device)
    sd["lm_head.weight"] = w
    del probe
    model = _model(cfg, sd, 32, max_streams=2, vit_batch=60)

    copies = []
    orig = Engine.kv_copy_prefix
    monkeypatch.setattr(Engine, "kv_copy_prefix", lambda self, *a: (copies.append(a), orig(self, *a))[1])
    res = []
    for run in range(2):
        if run == 1:
            no_prefill()
        out = []
        for thr in (0.0, 0.9):
            n = len(copies)
            out.append(model.stream_evaluate(input_ids.cuda(), label_ids.cuda(), feats.cuda(),
                                             frame_token_interval_threshold=thr).cpu())
            assert len(copies) > n, f"the look-ahead branch did not run (thr {thr})"
        res.append(out)
    for a, b in zip(*res):
        assert torch.equal(a, b), (a, b)


def test_fp8_and_ragged_take_the_chunked_path(tiny, monkeypatch):
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    calls = []
    orig = Engine._step_chunked

    def spy(self, *a, **k):
        calls.append(len(a[0]))
        return orig(self, *a, **k)
    monkeypatch.setattr(Engine, "_step_chunked", spy)
    for a8 in (False, True):     # e4m3 weights, then W8A8
        f8 = _model(cfg, llm, 128, max_streams=2, fp8=True, a8=a8).engine
        assert not f8.prefills and f8.max_prefill_tokens == 0 and f8.max_pass_tokens == 128
        s = f8.stream_open()
        f8.step([s], [300], _emb(cfg, 300, 1))
        assert f8.kv_len(s) == 300
        del f8
    assert calls == [1, 1]
    bf = _model(cfg, llm, 128, max_streams=2).engine
    a, b = bf.stream_open(), bf.stream_open()
    bf.step([a, b], [150, 100], _emb(cfg, 250, 2))
    assert calls == [1, 1, 2]
    bf.step([a], [300], _emb(cfg, 300, 3))
    assert calls == [1, 1, 2]


def test_workspaces_grow_only_on_prefilling_engines(tiny):
    """loading bf16 weights grows an engine's token-row workspaces to max_prefill_tokens rows; an engine with e4m3
    weights keeps the device memory it was created with"""
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    fresh = Engine(cfg, "cuda:0", max_streams=2, max_kv_tokens=4096, max_step_tokens=128, max_vit_batch=1)
    before = fresh.device_bytes()
    assert fresh.max_prefill_tokens == 0 and not fresh.prefills
    fresh.close()
    bf = _model(cfg, llm, 128, max_streams=2).engine
    assert bf.max_prefill_tokens == 1024 and bf.device_bytes() > before
    f8 = _model(cfg, llm, 128, max_streams=2, fp8=True).engine
    assert f8.max_prefill_tokens == 0 and f8.device_bytes() == before
