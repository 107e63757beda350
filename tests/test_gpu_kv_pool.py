"""The KV cache as a shared pool of 64-token pages: the paged attention op, page reuse, over-subscription, page
accounting and the copy / fill hooks, each checked bit for bit against the same work on contiguous memory or on an
engine whose pool reserves max_streams x max_kv_tokens."""
import ctypes as C

import pytest
import torch

from attn_reference import DECODER, decoder_chain, reference

pytestmark = pytest.mark.gpu

PAGE = 64


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------------------------------------ op level
@pytest.mark.parametrize("kv_len,n_tok,G", [(kv, n, g) for kv in (1, 63, 64, 65, 12011, 66011) for n in (1, 11, 40)
                                             for g in (2, 4) if n <= kv] + [(66011, 272, 4)])
def test_paged_attention_op_matches_contiguous(lib, kv_len, n_tok, G):
    """scattered pages in an oversized pool whose unused pages hold NaN and whose last page has garbage past kv_len
    (+-Inf, NaN and values ~100): bit-identical to the contiguous op on the same logical K / V.  272 queries at G = 4 are 17 work items: with
    8 kv heads the plan gets one split per item, so one CTA walks all 1032 key blocks."""
    from videollm_online_b200._lib import check
    torch.manual_seed(kv_len * 7 + n_tok * 3 + G)
    Hk, D = 8, 128
    H = Hk * G
    nblk = (kv_len + PAGE - 1) // PAGE
    stride = nblk * PAGE
    q = torch.randn(n_tok, H, D, device="cuda").bfloat16()
    k = torch.randn(Hk, stride, D, device="cuda").bfloat16()
    v = torch.randn(Hk, stride, D, device="cuda").bfloat16()
    n_pages = nblk + 5
    perm = torch.randperm(n_pages, device="cuda")[:nblk]
    kp = torch.full((n_pages, Hk, PAGE, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    vp = torch.full_like(kp, float("nan"))
    kp[perm] = k.view(Hk, nblk, PAGE, D).transpose(0, 1)
    vp[perm] = v.view(Hk, nblk, PAGE, D).transpose(0, 1)
    tail = kv_len - (nblk - 1) * PAGE
    if tail < PAGE:   # rows past kv_len in the last page: not what the contiguous cache holds, some not finite
        for pool in (kp, vp):
            junk = torch.randn(Hk, PAGE - tail, D, device="cuda") * 100
            junk[:, 0::4, 0::3], junk[:, 1::4, 1::3], junk[:, 2::4] = float("inf"), float("-inf"), float("nan")
            pool[perm[-1], :, tail:] = junk.bfloat16()
    pt = perm.to(torch.int32).contiguous()
    ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, H, D, kv_len), device="cuda", dtype=torch.uint8)
    out_c = torch.empty(n_tok, H * D, device="cuda", dtype=torch.bfloat16)
    out_p = torch.empty_like(out_c)
    check(lib.vlo_op_attn_kvappend(_p(q), _p(k), _p(v), _p(out_c), _p(ws), n_tok, H, Hk, D, kv_len, stride, _st()), "attn")
    check(lib.vlo_op_attn_kvappend_paged(_p(q), _p(kp), _p(vp), _p(pt), n_pages, _p(out_p), _p(ws), n_tok, H, Hk, D, kv_len,
                                         _st()), "attn_paged")
    torch.cuda.synchronize()
    assert torch.equal(out_p, out_c)
    res = reference(q, k[:, :kv_len], v[:, :kv_len], torch.arange(kv_len - n_tok, kv_len), DECODER,
                    decoder_chain(kv_len, torch.cuda.get_device_properties(0).multi_processor_count))
    assert torch.isfinite(out_p.float()).all()
    assert res.excess(out_p.view(n_tok, H, D)) <= 0


# ------------------------------------------------------------------------------------------------ engine level
def _engine(tiny, max_streams, max_kv_tokens, kv_pool_tokens=None):
    from videollm_online_b200.modeling_live import build_live
    cfg, llm, _vis = tiny
    model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=max_streams,
                          max_kv_tokens=max_kv_tokens, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=kv_pool_tokens)
    return model.engine


def _emb(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, cfg.hidden_size, generator=g).to(torch.bfloat16).cuda()


def _step(eng, sids, lens, seed):
    """one step; returns (last-position logits, decisions, all-position logits), all cloned"""
    emb = _emb(eng.cfg, sum(lens), seed)
    logits, dec = eng.step(list(sids), list(lens), emb)
    out = (logits.clone(), dec.clone(), eng.last_step_logits(sum(lens)).clone())
    torch.cuda.synchronize()
    return out


def _kv_all(eng, sid):
    return [(eng.kv_read(sid, l, False).clone(), eng.kv_read(sid, l, True).clone()) for l in range(eng.cfg.num_hidden_layers)]


def _same_kv(a, b):
    return len(a) == len(b) and all(torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) for x, y in zip(a, b))


def _same_step(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b))


def _held(eng):
    info = eng.kv_pool_info()
    return info["total_pages"] - info["free_pages"]


def _want(eng, sids):
    return sum((eng.kv_len(s) + PAGE - 1) // PAGE for s in sids)


def test_page_reuse_after_close_matches_a_fresh_stream(tiny):
    """A, B, C grow interleaved so their pages interleave; B closes and D reuses B's dirty pages.  D computes exactly
    what stream 0 of a default engine computes on the same inputs."""
    eng = _engine(tiny, 4, 1024, kv_pool_tokens=4 * 1024)
    ref = _engine(tiny, 1, 1024)
    a, b, c = eng.stream_open(), eng.stream_open(), eng.stream_open()
    for r in range(4):
        for i, s in enumerate((a, b, c)):
            _step(eng, [s], [37 + 19 * i + r], seed=100 * r + i)
    eng.stream_close(b)
    d = eng.stream_open()
    r0 = ref.stream_open()
    for r, n in enumerate((70, 1, 11, 64, 11, 128, 3)):
        got, want = _step(eng, [d], [n], seed=1000 + r), _step(ref, [r0], [n], seed=1000 + r)
        assert _same_step(got, want), f"step {r}"
    assert eng.kv_len(d) == ref.kv_len(r0)
    assert _same_kv(_kv_all(eng, d), _kv_all(ref, r0))


def test_pool_exhaustion_fails_without_changing_any_stream(tiny):
    from videollm_online_b200._lib import VloError
    eng = _engine(tiny, 6, 1024, kv_pool_tokens=2048)
    ref = _engine(tiny, 6, 1024)
    assert eng.kv_pool_info() == {"page_tokens": PAGE, "total_pages": 32, "free_pages": 32}
    lens = (600, 500, 420, 300, 90)   # 10 + 8 + 7 + 5 + 2 = 32 pages: the pool is full
    sids = []
    for i, n in enumerate(lens):
        s, s_ref = eng.stream_open(), ref.stream_open()
        assert s == s_ref
        eng.kv_fill_synthetic(s, n, seed=40 + i)
        ref.kv_fill_synthetic(s_ref, n, seed=40 + i)
        sids.append(s)
    assert eng.kv_pool_info()["free_pages"] == 0
    before = {s: (eng.kv_len(s), _kv_all(eng, s)) for s in sids}
    batch, q = [sids[0], sids[4]], [40, 40]   # 600 -> 640 fits its last page, 90 -> 130 needs a third page
    rows = torch.ones(eng.cfg.num_key_value_heads, 130, eng.cfg.head_dim, dtype=torch.bfloat16, device="cuda")
    grows = {"step": lambda: eng.step(batch, q, _emb(eng.cfg, sum(q), 7)),
             "kv_write": lambda: eng.kv_write(sids[4], 0, False, rows),
             "kv_fill_synthetic": lambda: eng.kv_fill_synthetic(sids[4], 130, seed=8),
             "kv_copy_prefix": lambda: eng.kv_copy_prefix(sids[0], sids[4], 200)}
    for name, grow in grows.items():
        with pytest.raises(VloError, match="KV page pool exhausted"):
            grow()
        torch.cuda.synchronize()
        assert eng.kv_pool_info()["free_pages"] == 0, name
        for s in sids:
            assert eng.kv_len(s) == before[s][0], name
            assert _same_kv(_kv_all(eng, s), before[s][1]), name
    eng.stream_close(sids[3])
    ref.stream_close(sids[3])
    assert _same_step(_step(eng, batch, q, seed=7), _step(ref, batch, q, seed=7))
    for s in batch:
        assert _same_kv(_kv_all(eng, s), _kv_all(ref, s))


def test_page_accounting_follows_kv_len(tiny):
    eng = _engine(tiny, 3, 1024, kv_pool_tokens=3 * 1024)
    total = eng.kv_pool_info()["total_pages"]
    a, b = eng.stream_open(), eng.stream_open()
    open_ = [a, b]
    check = lambda: _held(eng) == _want(eng, open_)
    _step(eng, [a, b], [64, 65], seed=1)
    assert check() and _held(eng) == 3
    _step(eng, [a], [1], seed=2)
    assert check()
    _step(eng, [a, b], [127, 63], seed=3)
    assert check()
    for n in (150, 128, 127, 64, 63, 1, 0):
        eng.kv_truncate(a, n)
        assert eng.kv_len(a) == n and check(), n
    _step(eng, [a], [100], seed=4)
    assert check()
    eng.stream_reset(b)
    assert eng.kv_len(b) == 0 and check()
    eng.kv_write(b, 0, False, torch.zeros(eng.cfg.num_key_value_heads, 200, eng.cfg.head_dim, dtype=torch.bfloat16))
    assert eng.kv_len(b) == 200 and check()
    eng.kv_fill_synthetic(b, 70, seed=3)
    assert check()
    eng.stream_close(b)
    open_.remove(b)
    assert check()
    eng.stream_close(a)
    assert eng.kv_pool_info()["free_pages"] == total


def _fragment(eng, sids, rounds, seed):
    """grow the streams round-robin, so consecutive pages of one stream are far apart in the pool"""
    for r in range(rounds):
        for i, s in enumerate(sids):
            _step(eng, [s], [41 + 13 * i], seed=seed + 10 * r + i)


def test_copy_prefix_from_a_fragmented_stream(tiny):
    eng = _engine(tiny, 4, 1024, kv_pool_tokens=2 * 1024)
    src, other = eng.stream_open(), eng.stream_open()
    _fragment(eng, [src, other], 4, seed=50)
    dst = eng.stream_open()
    _step(eng, [dst], [90], seed=60)      # the destination's old pages are dropped
    n = 150
    assert eng.kv_len(src) > n and n % PAGE
    eng.kv_copy_prefix(src, dst, n)
    assert eng.kv_len(dst) == n
    assert _held(eng) == _want(eng, [src, other, dst])
    for (ks, vs), (kd, vd) in zip(_kv_all(eng, src), _kv_all(eng, dst)):
        assert torch.equal(kd, ks[:, :n]) and torch.equal(vd, vs[:, :n])
    eng.kv_truncate(src, n)
    for r, q in enumerate((11, 1, 40)):
        assert _same_step(_step(eng, [src], [q], seed=70 + r), _step(eng, [dst], [q], seed=70 + r))


def test_synthetic_fill_on_scattered_pages(tiny):
    eng = _engine(tiny, 3, 2048, kv_pool_tokens=3 * 2048)
    ref = _engine(tiny, 3, 2048)
    a, b, s = eng.stream_open(), eng.stream_open(), eng.stream_open()
    ra, rb, rs = ref.stream_open(), ref.stream_open(), ref.stream_open()
    assert (a, b, s) == (ra, rb, rs)
    _fragment(eng, [a, b], 3, seed=80)
    eng.stream_close(a)                   # s's pages: a's freed pages first, then fresh ones
    eng.kv_fill_synthetic(s, 1500, seed=9)
    ref.kv_fill_synthetic(rs, 1500, seed=9)
    assert _same_kv(_kv_all(eng, s), _kv_all(ref, rs))


def test_ragged_batch_of_fragmented_streams(tiny):
    """a ragged batch over interleaved pages equals the same batch over contiguous pages (the reference engine grows
    its streams one after another) bit for bit; so does each stream stepped alone, which agrees with its batch row"""
    eng = _engine(tiny, 4, 1024, kv_pool_tokens=4 * 1024)
    ref = _engine(tiny, 4, 1024)
    sids = [eng.stream_open() for _ in range(3)]
    assert sids == [ref.stream_open() for _ in range(3)]
    grow = lambda i, r: dict(lens=[29 + 31 * i], seed=200 + 10 * r + i)
    for r in range(3):      # pooled engine: round-robin growth, each stream's pages interleave with the others'
        for i, s in enumerate(sids):
            _step(eng, [s], **grow(i, r))
    for i, s in enumerate(sids):   # reference: one stream after another, so each stream's pages are consecutive
        for r in range(3):
            _step(ref, [s], **grow(i, r))
    q = [11, 1, 40]
    got, want = _step(eng, sids, q, seed=300), _step(ref, sids, q, seed=300)
    assert _same_step(got, want)
    for s in sids:
        assert _same_kv(_kv_all(eng, s), _kv_all(ref, s))
    # alone: a 1-sequence step has its own split-KV decomposition, so it matches the batch row within rounding only
    emb = _emb(eng.cfg, sum(q), 300)
    off = 0
    for i, s in enumerate(sids):
        eng.kv_truncate(s, eng.kv_len(s) - q[i])
        ref.kv_truncate(s, ref.kv_len(s) - q[i])
        rows = emb[off:off + q[i]].contiguous()
        alone = eng.step([s], [q[i]], rows)[0].clone()
        assert torch.equal(alone, ref.step([s], [q[i]], rows)[0])
        assert (alone[0].float() - got[0][i].float()).abs().max() < 0.5
        off += q[i]


def test_long_stream_in_a_wide_batch(tiny):
    """16 work items in one step (a 66k-token stream with 120 new tokens + 8 one-token streams) with 8 kv heads: the
    long stream has one split per item, over all of its 1034 key blocks.  Interleaved pages give the bits of contiguous ones."""
    from videollm_online_b200 import tiny_config, weights as W
    from videollm_online_b200.modeling_live import build_live
    cfg = tiny_config(hidden_size=4096, num_attention_heads=32, num_key_value_heads=8)   # Llama-3-8B attention shapes
    llm = W.synthetic_llm_state(cfg, seed=3)
    KV, CAP = 66011, 66011 + 256

    def engine(pool):
        model, _ = build_live(config=cfg, llm_state=llm, set_vision_inside=False, device="cuda:0", max_streams=9,
                              max_kv_tokens=CAP, max_step_tokens=128, max_vit_batch=1, kv_pool_tokens=pool)
        return model.engine
    eng, ref = engine(CAP + 8 * 256), engine(None)
    sids = [eng.stream_open() for _ in range(9)]
    assert sids == [ref.stream_open() for _ in range(9)]
    for part in range(1, 5):   # the long stream's pages interleave with another stream's in the pooled engine
        eng.kv_fill_synthetic(sids[0], KV * part // 4, seed=5)
        eng.kv_fill_synthetic(sids[1], 100 * part, seed=6)
    ref.kv_fill_synthetic(sids[0], KV, seed=5)
    ref.kv_fill_synthetic(sids[1], 400, seed=6)
    q = [120] + [1] * 8
    got, want = _step(eng, sids, q, seed=11), _step(ref, sids, q, seed=11)
    assert _same_step(got, want)
    assert torch.isfinite(got[0].float()).all()
    assert eng.kv_len(sids[0]) == KV + 120 and _held(eng) == _want(eng, sids)


def test_chunked_step_on_an_exhausted_pool_changes_nothing(tiny):
    """a step longer than max_step_tokens runs in pieces; when a later piece finds the pool exhausted the earlier
    pieces are undone, so the call can be retried whole"""
    from videollm_online_b200._lib import VloError
    eng = _engine(tiny, 2, 1024, kv_pool_tokens=256)
    a = eng.stream_open()
    with pytest.raises(VloError, match="KV page pool exhausted"):
        eng.step([a], [300], _emb(eng.cfg, 300, 3))
    assert eng.kv_len(a) == 0 and eng.kv_pool_info()["free_pages"] == 4
    eng.step([a], [250], _emb(eng.cfg, 250, 3))
    assert eng.kv_len(a) == 250 and eng.kv_pool_info()["free_pages"] == 0
