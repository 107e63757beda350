"""Quantized vocabulary matrices (embed and lm_head in the layer matrices' int4 or e4m3 form), all bit for bit:

* the whole-tile int4 GEMM equals the bf16 whole-tile GEMM on W4 = dequantize_int4_groups(q, s);
* the whole-tile e4m3 GEMM equals bf16(fl(P * s[n])), P the bf16 kernel's fp32 result on the upcast codes;
* a logits row does not depend on the other rows or on the token tile;
* the gathers equal the host rules (weights.dequantized_vocab_matrix);
* an int4 engine with quantized vocabulary matrices equals an int4 engine loaded with them dequantized in bf16;
* FP8 and W8A8 engines: the hidden rows equal those of the same form on the dequantized embedding table, and the logits
  are the e4m3 rule applied to the engine's own final-normed rows.
"""
import ctypes as C
import pathlib
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import test_gpu_frame_backlog as FB     # noqa: E402  (K/V of every layer)

FMT_BF16, FMT_E4M3, FMT_I4 = 1, 2, 4


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


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


# ============================================================================================ kernels
VS = [(128256, 4096), (1024, 4096), (1000, 640)]   # Llama-3-8B lm_head, a small and an odd shape
ROWS = [1, 11, 16, 17, 31, 32, 33, 64, 65, 96, 97, 128]   # every token tile with a full last tile and a one-row spill
PAD_COLS, PAD_ROWS = 8, 3


@pytest.fixture(scope="module")
def operands():
    from videollm_online_b200 import weights as W
    cache = {}

    def get(V, K):
        if (V, K) not in cache:
            g = torch.Generator(device="cuda").manual_seed(V + K)
            w = (torch.randn(V, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
            q, s = W.quantize_int4_groups(w)
            f8, sc = W.quantize_fp8_rows(w)
            x = torch.randn(128, K, device="cuda", generator=g).bfloat16()
            cache[(V, K)] = dict(i4=W.pack_int4_codes(q), gs=s, w4=W.dequantize_int4_groups(q, s), f8=f8, sc=sc,
                                 up=f8.view(torch.float8_e4m3fn).bfloat16(), x=x)
        return cache[(V, K)]
    return get


def _sentinel(T, V):
    return torch.full((T + PAD_ROWS, V + PAD_COLS), float("nan"), dtype=torch.bfloat16, device="cuda")


def _tiles_bf16(lib, w, V, x, T, K):
    out = _sentinel(T, V)
    _check(lib.vlo_op_gemm_ws(FMT_BF16, 1, _p(w), V, _p(x), T, K, _p(out), V + PAD_COLS, 0, None, 0, 0, 0, None, _st()),
           "bf16 tiles")
    return out


def _tiles_q(lib, fmt, w, scale, V, x, T, K, n_ctas=0):
    out = _sentinel(T, V)
    plan = (C.c_int32 * 3)()
    _check(lib.vlo_op_gemm_ws_tiles_q(fmt, _p(w), _p(scale), V, _p(x), T, K, _p(out), V + PAD_COLS, n_ctas, plan, _st()),
           "quantized tiles")
    return out, list(plan)


def _sentinels_kept(out, T, V):
    return bool(torch.isnan(out[T:].float()).all()) and bool(torch.isnan(out[:, V:].float()).all())


def _e4m3_rule(lib, up, sc, V, x, T, K):
    """bf16(fl(P * s)), P the fp32 result of the bf16 kernel on the upcast codes: mode 0 with one CTA per weight tile
    gives one plane per tile, the whole k chain of one CTA"""
    tiles = (V + 127) // 128
    planes = C.c_int(0)
    P = torch.full((2, T, V), float("nan"), device="cuda")
    _check(lib.vlo_op_gemm_ws(FMT_BF16, 0, _p(up), V, _p(x), T, K, _p(P), V, T * V, None, 0, tiles, 0, C.byref(planes),
                              _st()), "one-plane bf16")
    torch.cuda.synchronize()
    assert planes.value == 1
    return (P[0] * sc[None, :]).bfloat16()


@pytest.mark.parametrize("T", ROWS)
@pytest.mark.parametrize("V,K", VS)
def test_int4_tiles_are_the_bf16_tiles_on_w4(lib, operands, V, K, T):
    o = operands(V, K)
    x = o["x"][:T].contiguous()
    want = _tiles_bf16(lib, o["w4"], V, x, T, K)
    got, plan = _tiles_q(lib, FMT_I4, o["i4"], o["gs"], V, x, T, K)
    torch.cuda.synchronize()
    assert plan[1] == 1 and plan[0] >= T
    assert _same_bits(got, want), f"V={V} K={K} T={T}"
    assert _sentinels_kept(got, T, V)


@pytest.mark.parametrize("T", ROWS)
@pytest.mark.parametrize("V,K", VS)
def test_e4m3_tiles_are_the_rule(lib, operands, V, K, T):
    o = operands(V, K)
    x = o["x"][:T].contiguous()
    want = _e4m3_rule(lib, o["up"], o["sc"], V, x, T, K)
    got, _ = _tiles_q(lib, FMT_E4M3, o["f8"], o["sc"], V, x, T, K)
    torch.cuda.synchronize()
    assert _same_bits(got[:T, :V].contiguous(), want), f"V={V} K={K} T={T}"
    assert _sentinels_kept(got, T, V)


@pytest.mark.parametrize("fmt", [FMT_I4, FMT_E4M3])
def test_rows_are_independent_of_the_token_tile(lib, operands, fmt):
    """the first row's logits, and row 10's, at every token tile and CTA count"""
    V, K = 1000, 640
    o = operands(V, K)
    w, s = (o["i4"], o["gs"]) if fmt == FMT_I4 else (o["f8"], o["sc"])
    ref, _ = _tiles_q(lib, fmt, w, s, V, o["x"][:11].contiguous(), 11, K)
    seen = set()
    for T in ROWS:
        if T < 11:
            continue
        for n_ctas in (0, 5):
            got, plan = _tiles_q(lib, fmt, w, s, V, o["x"][:T].contiguous(), T, K, n_ctas)
            seen.add(plan[0])
            torch.cuda.synchronize()
            assert _same_bits(got[:11, :V].contiguous(), ref[:11, :V].contiguous()), f"T={T} n_ctas={n_ctas}"
    assert seen == {16, 32, 64, 96, 128}


def test_bad_arguments(lib, operands):
    from videollm_online_b200._lib import VloError
    o = operands(1000, 640)
    out = torch.zeros(256, 1000, dtype=torch.bfloat16, device="cuda")
    x = torch.zeros(256, 640, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(VloError, match="1..128 token rows"):
        _check(lib.vlo_op_gemm_ws_tiles_q(FMT_I4, _p(o["i4"]), _p(o["gs"]), 1000, _p(x), 129, 640, _p(out), 1000, 0, None,
                                          _st()), "T")
    with pytest.raises(VloError, match="fmt"):
        _check(lib.vlo_op_gemm_ws_tiles_q(3, _p(o["f8"]), _p(o["sc"]), 1000, _p(x), 16, 640, _p(out), 1000, 0, None,
                                          _st()), "W8A8")
    with pytest.raises(VloError, match="null scales"):
        _check(lib.vlo_op_gemm_ws_tiles_q(FMT_E4M3, _p(o["f8"]), None, 1000, _p(x), 16, 640, _p(out), 1000, 0, None,
                                          _st()), "scales")


def test_e4m3_tiles_beyond_one_token_tile(lib, operands):
    """rows past 128 run as several 128-wide token tiles; every row is still the rule"""
    V, K = 1024, 4096
    o = operands(V, K)
    x = torch.cat([o["x"], o["x"][:72]]).contiguous()
    got, plan = _tiles_q(lib, FMT_E4M3, o["f8"], o["sc"], V, x, 200, K)
    torch.cuda.synchronize()
    assert plan[:2] == [128, 2]
    want = torch.cat([_e4m3_rule(lib, o["up"], o["sc"], V, x[:128].contiguous(), 128, K),
                      _e4m3_rule(lib, o["up"], o["sc"], V, x[128:].contiguous(), 72, K)])
    assert _same_bits(got[:200, :V].contiguous(), want)
    assert _sentinels_kept(got, 200, V)


IDS = [0, 1023, 5, 5, 13, 21, 517, -1, 5000]   # first and last row, a repeated id, rows 8 apart in one tile, <0, > V-1


@pytest.mark.parametrize("fmt", [FMT_I4, FMT_E4M3])
def test_gathers_equal_the_host_rules(lib, operands, fmt):
    from videollm_online_b200 import weights as W
    V, K = 1024, 4096
    o = operands(V, K)
    if fmt == FMT_I4:
        table, scale, deq = o["i4"], o["gs"], W.dequantized_vocab_matrix({"e.i4": o["i4"], "e.gscale": o["gs"]}, "e", V, K)
    else:
        table, scale, deq = o["f8"], o["sc"], W.dequantized_vocab_matrix({"e.f8": o["f8"], "e.scale": o["sc"]}, "e", V, K)
    ids = torch.tensor(IDS, dtype=torch.int64, device="cuda")
    got = torch.full((len(IDS), K), float("nan"), dtype=torch.bfloat16, device="cuda")
    _check(lib.vlo_op_embed_rows_q(fmt, _p(table), _p(scale), V, K, _p(ids), len(IDS), _p(got), _st()), "gather")
    want = torch.full_like(got, float("nan"))   # the bf16 gather on the dequantized table: the same out-of-range handling
    _check(lib.vlo_op_embed_rows_q(FMT_BF16, _p(deq), None, V, K, _p(ids), len(IDS), _p(want), _st()), "bf16 gather")
    torch.cuda.synchronize()
    assert _same_bits(got, want)
    assert bool(torch.isnan(got[IDS.index(-1)].float()).all())
    rows = torch.tensor([min(i, V - 1) for i in IDS if i >= 0])
    assert _same_bits(got[[j for j, i in enumerate(IDS) if i >= 0]], deq[rows.cuda()])


# ============================================================================================ int4 engine
def _deq_vocab_state(llm, fmt):
    """the HF-style state with embed_tokens and lm_head replaced by what the quantized engine multiplies or gathers"""
    from videollm_online_b200 import weights as W
    out = dict(llm)
    for k in ("model.embed_tokens.weight", "lm_head.weight"):
        w = llm[k].cuda()
        out[k] = (W.dequantize_int4_groups(*W.quantize_int4_groups(w)) if fmt == "int4"
                  else W.dequantize_fp8_rows_bf16(*W.quantize_fp8_rows(w))).cpu()
    return out


def _model(cfg, llm, quantize_vocab, fp8=False, int4=True, fp8_act=False, max_streams=3, max_kv_tokens=4096):
    from videollm_online_b200.modeling_live import build_live
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, int4_weights=int4,
                          fp8_weights=fp8, fp8_activations=fp8_act, quantize_vocab=quantize_vocab)
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
    """(int4 engine with quantized vocabulary matrices, int4 engine with them dequantized in bf16)"""
    cfg, llm = tiny
    eq = _model(cfg, llm, True).engine
    eb = _model(cfg, _deq_vocab_state(llm, "int4"), False).engine
    assert eq.quantized_vocab and not eb.quantized_vocab and eq.int4_weights and eb.int4_weights
    assert eq.lib.vlo_vocab_format(eq._h) == FMT_I4 and eb.lib.vlo_vocab_format(eb._h) == FMT_BF16
    return eq, eb


def _emb(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()


def _ids(cfg, n, seed):
    """token ids for every other row (the gather) and -1 (the given embedding) for the rest; one past the vocabulary"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, cfg.vocab_size, (n,), generator=g)
    ids[1::2] = -1
    ids[-1] = cfg.vocab_size + 3 if n > 2 else ids[-1]
    return ids


def _outputs(eng, sid, lg, dc, n):
    return (lg.clone(), dc.clone(), eng.last_step_hidden(n).clone(), FB._kv_all(eng, sid))


def _assert_same(a, b, what):
    assert torch.equal(a[0], b[0]), f"{what}: logits"
    assert torch.equal(a[1], b[1]), f"{what}: decision rows"
    assert torch.equal(a[2], b[2]), f"{what}: final hidden rows"
    assert FB._same_kv(a[3], b[3]), f"{what}: K/V"


@pytest.mark.parametrize("T", [1, 11, 128])
def test_engine_step_equals_dequantized_bf16_vocab(tiny, pair, T):
    """one stream, T rows (half of them gathered by id) after a 40-row step; then last_step_logits over all rows"""
    cfg, _ = tiny
    res = []
    for eng in pair:
        sid = eng.stream_open()
        eng.step([sid], [40], _emb(cfg, 40, 1), row_ids=_ids(cfg, 40, 1))
        lg, dc = eng.step([sid], [T], _emb(cfg, T, 2 + T), row_ids=_ids(cfg, T, 2 + T))
        res.append(_outputs(eng, sid, lg, dc, T) + (eng.last_step_logits(T).clone(),))
        eng.stream_close(sid)
    _assert_same(res[0], res[1], f"T={T}")
    assert torch.equal(res[0][4], res[1][4]), "last_step_logits"
    assert torch.equal(res[0][4][-1:], res[0][0])
    assert torch.isfinite(res[0][0].float()).all()


def test_embed_tokens_equal(tiny, pair):
    cfg, _ = tiny
    ids = torch.tensor([0, cfg.vocab_size - 1, 7, 7, 15, 23, cfg.vocab_size + 100], dtype=torch.int64)
    a, b = (eng.embed_tokens(ids) for eng in pair)
    assert torch.equal(a, b)
    from videollm_online_b200.modeling_live import _Embedding
    assert torch.equal(_Embedding(pair[0]).weight, pair[1].weights["embed"])


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
        lg, dc = eng.step([sid], [22], _emb(cfg, 22, 5), row_ids=_ids(cfg, 22, 5), segments=[[1, 10, 1, 10]])
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
        lg, dc = eng.step(s, q, _emb(cfg, sum(q), 9), row_ids=_ids(cfg, sum(q), 9))
        res.append((lg.clone(), dc.clone(), eng.last_step_hidden(sum(q)).clone(), [FB._kv_all(eng, sid) for sid in s]))
        for sid in s:
            eng.stream_close(sid)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])
    assert all(FB._same_kv(a, b) for a, b in zip(res[0][3], res[1][3]))


def test_verify_step_with_drafts_and_sampling(tiny, pair):
    from videollm_online_b200.engine import SampleRow
    cfg, _ = tiny
    ids = torch.tensor([17, 40, 99, 3, 250, 8], dtype=torch.int64)
    n = ids.numel()
    res, draws = [], []
    for eng in pair:
        sid = eng.stream_open()
        eng.kv_fill_synthetic(sid, 200, seed=4)
        zeros = torch.zeros(n, cfg.hidden_size, dtype=torch.bfloat16, device="cuda")
        lg, dc = eng.step([sid], [n], zeros, row_ids=ids, segments=[[1] * n])
        res.append(_outputs(eng, sid, lg, dc, n))
        row = SampleRow(seed=1234, position=206, temperature=0.9, top_k=50, top_p=0.95)
        eng.step([sid], [1], zeros[:1], row_ids=ids[:1], sample=[row])
        d = eng.read_decisions(1)[0]
        draws.append((d.sampled_id, d.argmax_id))
        eng.stream_close(sid)
    _assert_same(res[0], res[1], "verify step")
    assert draws[0][0] is not None and draws[0] == draws[1]


def test_evict_compact_swap_then_step(tiny, pair):
    cfg, _ = tiny
    res = []
    for eng in pair:
        sid = eng.stream_open()
        eng.step([sid], [128], _emb(cfg, 128, 11), row_ids=_ids(cfg, 128, 11))
        eng.step([sid], [100], _emb(cfg, 100, 12))
        outs = []
        eng.kv_evict(sid, 64, 64)
        lg, dc = eng.step([sid], [11], _emb(cfg, 11, 13), row_ids=_ids(cfg, 11, 13))
        outs.append(_outputs(eng, sid, lg, dc, 11))
        eng.kv_compact(sid, [(0, 20), (40, 50)])
        lg, dc = eng.step([sid], [11], _emb(cfg, 11, 14))
        outs.append(_outputs(eng, sid, lg, dc, 11))
        img = eng.kv_swap_out(sid)
        eng.kv_swap_in(sid, img)
        lg, dc = eng.step([sid], [1], _emb(cfg, 1, 15), row_ids=_ids(cfg, 1, 15))
        outs.append(_outputs(eng, sid, lg, dc, 1))
        res.append(outs)
        eng.stream_close(sid)
    for what, a, b in zip(("evict", "compact", "swap"), res[0], res[1]):
        _assert_same(a, b, what)


def test_finalize_rejects_bad_vocabulary_forms(tiny):
    from videollm_online_b200 import weights as W
    from videollm_online_b200._lib import VloError
    from videollm_online_b200.engine import Engine
    cfg, llm = tiny
    i4q = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512, int4_weights=True, quantize_vocab=True)
    f8q = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512, fp8_weights=True, quantize_vocab=True)
    bf = W.pack_llm_for_engine(cfg, llm, "cuda:0", 512)
    vocab = ("embed", "lm_head")

    def swap_vocab(base, src, which=vocab):
        out = {k: v for k, v in base.items() if k.split(".")[0] not in which}
        out.update({k: v for k, v in src.items() if k.split(".")[0] in which})
        return out

    def attempt(packed, match):
        eng = Engine(cfg, "cuda:0", max_streams=1, max_kv_tokens=256, max_step_tokens=32, max_vit_batch=1)
        try:
            before = eng.device_bytes()
            with pytest.raises(VloError, match=match):
                eng.load_weights(packed)
            assert eng.device_bytes() == before
        finally:
            eng.close()

    attempt(swap_vocab(i4q, f8q), "vocabulary matrices .* are e4m3 but the layer matrices are int4")
    attempt(swap_vocab(f8q, i4q), "vocabulary matrices .* are int4 but the layer matrices are e4m3")
    attempt(swap_vocab(bf, i4q), "layer matrices are bf16")
    attempt(swap_vocab(i4q, bf, ("lm_head",)), "lm_head' is bf16 but an earlier vocabulary matrix is not")
    attempt({k: v for k, v in i4q.items() if k != "lm_head.gscale"}, "lm_head.gscale")
    attempt({k: v for k, v in f8q.items() if k != "embed.f8"}, "embed.f8")
    short = dict(i4q)
    short["lm_head.i4"] = i4q["lm_head.i4"][:-16].contiguous()
    attempt(short, "lm_head.i4")
    short = dict(f8q)
    short["embed.scale"] = f8q["embed.scale"][:-1].contiguous()
    attempt(short, "embed.scale")

    # a failed finalize leaves the installed tables untouched (and the engine unfinalized, as for the layer matrices)
    eng = Engine(cfg, "cuda:0", max_streams=1, max_kv_tokens=256, max_step_tokens=32, max_vit_batch=1)
    try:
        eng.load_weights(i4q)
        assert eng.lib.vlo_vocab_format(eng._h) == FMT_I4
        with pytest.raises(VloError, match="more than one form"):
            eng.load_weights({k: v for k, v in f8q.items() if k.split(".")[0] in vocab})
        assert eng.lib.vlo_vocab_format(eng._h) == FMT_I4
        with pytest.raises(VloError, match="not loaded"):
            eng.embed_tokens(torch.tensor([3], dtype=torch.int64))
    finally:
        eng.close()


# ============================================================================================ FP8 and W8A8 engines
@pytest.mark.parametrize("fp8_act", [False, True])
def test_fp8_engines(lib, tiny, fp8_act):
    """hidden rows: those of the same form with the dequantized embedding table in bf16; logits: bf16(fl(P * s)) of the
    engine's own final-normed rows"""
    from videollm_online_b200 import weights as W
    cfg, llm = tiny
    eq = _model(cfg, llm, True, fp8=True, int4=False, fp8_act=fp8_act).engine
    ref_state = dict(llm)
    ref_state["model.embed_tokens.weight"] = _deq_vocab_state(llm, "fp8")["model.embed_tokens.weight"]
    eb = _model(cfg, ref_state, False, fp8=True, int4=False, fp8_act=fp8_act).engine
    assert eq.quantized_vocab and eq.lib.vlo_vocab_format(eq._h) == FMT_E4M3
    V, H = cfg.vocab_size, cfg.hidden_size
    f8, sc = eq.weights["lm_head.f8"], eq.weights["lm_head.scale"]
    up = f8.view(torch.float8_e4m3fn).bfloat16()
    for T in (1, 11, 128):
        hid = []
        for eng in (eq, eb):
            sid = eng.stream_open()
            eng.step([sid], [40], _emb(cfg, 40, 1), row_ids=_ids(cfg, 40, 1))
            lg, _ = eng.step([sid], [T], _emb(cfg, T, 2 + T), row_ids=_ids(cfg, T, 2 + T))
            hid.append((eng.last_step_hidden(T).clone(), FB._kv_all(eng, sid), lg.clone(), eng.last_step_logits(T).clone()))
            eng.stream_close(sid)
        assert torch.equal(hid[0][0], hid[1][0]), f"T={T}: final hidden rows"
        assert FB._same_kv(hid[0][1], hid[1][1]), f"T={T}: K/V"
        want = _e4m3_rule(lib, up, sc, V, hid[0][0], T, H)
        assert torch.equal(hid[0][3], want), f"T={T}: all-row logits"
        assert torch.equal(hid[0][2], want[-1:]), f"T={T}: step logits"
    eq.close()
    eb.close()


# ============================================================================================ LiveInfer
LIVE_FRAMES = 40
LIVE_SPEAK = {7, 22, 33}


def test_liveinfer_cli_quantized_vocab(tiny):
    """cli.main with LiveArguments(int4_weights=True, quantize_vocab=True), and with an int4 model on the dequantized
    vocabulary matrices in bf16: the same conversation, decision rows and final cache; the suspended state records the
    form"""
    from dataclasses import asdict
    import test_gpu_ordering as OR
    from videollm_online_b200 import cli, weights as W
    from videollm_online_b200.config import LiveArguments
    from videollm_online_b200.inference import LiveInfer
    from videollm_online_b200.modeling_live import build_model_and_tokenizer
    cfg, llm = tiny
    vis = W.synthetic_vision_state(cfg, seed=1)
    runs = []
    for qv, state in ((True, llm), (False, _deq_vocab_state(llm, "int4"))):
        args = LiveArguments(llm_pretrained="", frame_resolution=cfg.frame_resolution, int4_weights=True, quantize_vocab=qv)
        model, tok = build_model_and_tokenizer(is_training=False, set_vision_inside=True, config=cfg, llm_state=state,
                                               vision_state=vis, max_kv_tokens=2048, max_vit_batch=8, **asdict(args))
        assert model.engine.quantized_vocab == qv
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
        assert li.suspend().quantized_vocab is qv
        model.engine.close()
    (conv_q, raw_q, kv_q), (conv_b, raw_b, kv_b) = runs
    assert len(conv_q) >= 4
    assert conv_q == conv_b
    assert raw_q == raw_b
    assert FB._same_kv(kv_q, kv_b)
