"""Masked rows: rows an attention kernel loads but must not see.  Their values may be anything, non-finite included.

The decoder attention (csrc/attn.cuh) loads whole 64-key blocks, so the block holding a sequence's key end also brings
the rows past it: on the engine's page pool those are stale rows of a page that another session (or this one, before a
truncate, evict or compact) wrote.  The ViT attention (vit_attn_kernel) reads frame f's last block from the first rows of
frame f + 1.  Masked rows get probability 0, but 0 x Inf and 0 x NaN are NaN, so both kernels zero those V rows.

A.  Decoder attention, kernel level: every case of test_gpu_attention_reference with its masked rows (rows >= kv_len on
    the last page, every row of the pages outside the table, rows kv_len .. stride of the contiguous cache) zero, then
    poisoned with +-Inf, two NaNs, +-bf16 max and random x 100 in K, V or both: the output must keep its bits.  A sweep
    over every kv_len mod 64 poisons the whole tail, only its first row and only the block's last row.
B.  ViT attention: a poisoned frame (all its rows, or only the rows its predecessor's last block loads) leaves every
    other frame's output bit-identical.
C.  Engine: a step fed an Inf embedding row leaves non-finite K / V at that position (the route is real), and a stream
    that takes pages such rows were written to, a stream rolled back before them, a swap image with NaN rows past its
    length, and a clean stream batched with a poisoned one all compute the bits of a run that never saw the poison.
"""
import ctypes as C
import pathlib
import sys

import pytest
import torch

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import test_gpu_attention_reference as AR  # noqa: E402  (the case list and its input builders)
from attn_reference import DECODER, decoder_chain, reference  # noqa: E402

pytestmark = pytest.mark.gpu

PAGE = 64
D = 128


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module", autouse=True)
def _scrub_poisoned_memory():
    """the caching allocator would hand the memory these tests filled with NaN and Inf to later tests: give it back to
    the driver zeroed, so that a later test's torch.empty buffers start clean.  Once, after this module,
    test_gpu_vit_kernels.py::test_tower_replay_bit_exact[11] did not repeat its bits; the record does not say whether
    vit_encode or the replay changed.  The replay's own stages read only what they wrote:
    test_gpu_ordering.py::test_tower_replay_reads_only_what_it_wrote runs it over NaN- and pattern-filled buffers with
    poisoned tails at every frame batch.  The engine's ViT workspaces inside vit_encode are not covered by that test."""
    yield
    torch.cuda.synchronize()
    free = torch.cuda.memory_reserved() - torch.cuda.memory_allocated()
    torch.cuda.empty_cache()
    if free > 0:
        torch.zeros(free, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    from videollm_online_b200._lib import check
    check(rc, what)


def _same(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# bf16 bit patterns of the poisons; "rand" is random x 100
BF16_POISON = {"+inf": 0x7F80, "-inf": 0xFF80, "nan_7fc1": 0x7FC1, "nan_ffc1": 0xFFC1, "+max": 0x7F7F, "-max": 0xFF7F,
               "rand": None}


def _poison_like(x, name, gen):
    """a tensor shaped like x (bf16) holding the poison"""
    bits = BF16_POISON[name]
    if bits is None:
        return (100.0 * torch.randn(x.shape, device="cuda", generator=gen)).bfloat16()
    b = bits - 0x10000 if bits >= 0x8000 else bits
    return torch.full(x.shape, b, dtype=torch.int16, device="cuda").view(torch.bfloat16)


# ============================================================================================ A: decoder attention
class _Decoder:
    """one attention case: q and the logical K / V [Hk, stride, D] (stride: whole pages, + one page for the contiguous
    cache), and the page layout of the paged entries (the table's pages scattered in a pool of 5 spare pages)"""

    def __init__(self, lib, path, segs, kv_len, Hq, Hk, q, k, v, seed):
        self.lib, self.path, self.segs, self.kv_len, self.Hq, self.Hk = lib, path, segs, kv_len, Hq, Hk
        self.q, self.k, self.v = q, k, v
        self.n_tok = sum(segs)
        self.nblk = (kv_len + PAGE - 1) // PAGE
        self.n_pages = self.nblk + 5
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.perm = torch.randperm(self.n_pages, device="cuda", generator=g)[:self.nblk]
        self.spare = torch.ones(self.n_pages, dtype=torch.bool, device="cuda")
        self.spare[self.perm] = False

    def run(self, k, v, spare_k=None, spare_v=None):
        """the output for logical K / V (rows past kv_len included) and the values of the spare pages (default 0)"""
        lib, n_tok, Hq, Hk = self.lib, self.n_tok, self.Hq, self.Hk
        out = torch.full((n_tok, Hq * D), float("nan"), device="cuda", dtype=torch.bfloat16)
        if self.path == "contig":
            ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, Hq, D, self.kv_len), device="cuda", dtype=torch.uint8)
            _check(lib.vlo_op_attn_kvappend(_p(self.q), _p(k), _p(v), _p(out), _p(ws), n_tok, Hq, Hk, D, self.kv_len,
                                            k.shape[1], _st()), "attn")
        else:
            pools = []
            for x, spare in ((k, spare_k), (v, spare_v)):
                pool = torch.zeros(self.n_pages, Hk, PAGE, D, device="cuda", dtype=torch.bfloat16)
                if spare is not None:
                    pool[self.spare] = spare
                pool[self.perm] = x[:, :self.nblk * PAGE].reshape(Hk, self.nblk, PAGE, D).transpose(0, 1)
                pools.append(pool)
            pt = self.perm.to(torch.int32).contiguous()
            if self.path == "paged":
                ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, Hq, D, self.kv_len), device="cuda", dtype=torch.uint8)
                _check(lib.vlo_op_attn_kvappend_paged(_p(self.q), _p(pools[0]), _p(pools[1]), _p(pt), self.n_pages,
                                                      _p(out), _p(ws), n_tok, Hq, Hk, D, self.kv_len, _st()),
                       "attn_paged")
            else:
                lens = (C.c_int32 * len(self.segs))(*self.segs)
                _check(lib.vlo_op_attn_kvappend_segments(_p(self.q), _p(pools[0]), _p(pools[1]), _p(pt), self.n_pages,
                                                         _p(out), len(self.segs), lens, Hq, Hk, D, self.kv_len, _st()),
                       "attn_segments")
        torch.cuda.synchronize()
        return out

    def poisoned(self, rows, name, target, gen):
        """run with the logical rows `rows` (a slice or index list past kv_len) and every spare page poisoned in
        target ("K", "V" or "KV")"""
        k, v = self.k.clone(), self.v.clone()
        spare = {"K": None, "V": None}
        for t, x in (("K", k), ("V", v)):
            if t in target:
                x[:, rows] = _poison_like(x[:, rows], name, gen)
                if self.path != "contig":
                    n_sp = int(self.spare.sum())
                    spare[t] = _poison_like(torch.empty(n_sp, self.Hk, PAGE, D), name, gen)
        return self.run(k, v, spare["K"], spare["V"])


def _decoder_case(lib, path, segs, kv_len, Hq, Hk, profile, seed):
    n_tok = sum(segs)
    items = AR._items(segs, kv_len, Hq, Hk)
    needles = AR._needle_keys(items, n_tok, kv_len)
    stride = (kv_len + PAGE - 1) // PAGE * PAGE + (PAGE if path == "contig" else 0)
    q, k, v = AR._decoder_inputs(n_tok, kv_len, Hq, Hk, needles, profile, stride, seed)
    k[:, kv_len:] = 0
    v[:, kv_len:] = 0
    return _Decoder(lib, path, segs, kv_len, Hq, Hk, q, k, v, seed)


def _assert_reaches(lib, path, segs, kv_len, Hq, Hk):
    counts = AR._plan_counts(lib, segs, Hq, Hk, kv_len)
    if path == "cluster":
        assert counts["clusters"] >= 1, counts
    if path == "packed":
        assert counts["packs"] >= 1, counts


@pytest.mark.parametrize("path,segs,kv_len,Hq,Hk,profile", AR.CASES, ids=[AR._id(c) for c in AR.CASES])
def test_decoder_attention_ignores_masked_rows(lib, path, segs, kv_len, Hq, Hk, profile):
    """zero masked rows: within the fp64 bound; every poison in K, V or both: the zero run's bits"""
    _assert_reaches(lib, path, segs, kv_len, Hq, Hk)
    seed = kv_len * 31 + sum(segs) * 7 + Hq + len(segs)
    case = _decoder_case(lib, path, segs, kv_len, Hq, Hk, profile, seed)
    clean = case.run(case.k, case.v)
    assert torch.isfinite(clean.float()).all()
    n_tok = case.n_tok
    res = reference(case.q, case.k[:, :kv_len], case.v[:, :kv_len], torch.arange(kv_len - n_tok, kv_len), DECODER,
                    decoder_chain(kv_len, AR._n_sm()))
    ex = res.excess(clean.view(n_tok, Hq, D))
    assert ex <= 0, f"attention leaves the fp64 bound by {ex}"
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    bad = []
    for name in BF16_POISON:
        for target in ("K", "V", "KV"):
            out = case.poisoned(slice(kv_len, None), name, target, gen)
            if not _same(out, clean):
                bad.append(f"{name} in {target} ({int(out.float().isnan().any(-1).sum())} NaN rows)")
    assert not bad, f"masked rows leak into the output: {bad}"


SWEEP = [(path, n_tok, Hq, Hk) for path in ("paged", "packed") for n_tok in (1, 11) for Hq, Hk in ((32, 8), (8, 2))
         if not (path == "packed" and n_tok == 1)] + [("packed", 2, 32, 8), ("packed", 2, 8, 2)]


@pytest.mark.parametrize("path,n_tok,Hq,Hk", SWEEP, ids=[f"{c[0]}-{c[1]}-{c[2]}x{c[3]}" for c in SWEEP])
def test_decoder_attention_masked_row_residues(lib, path, n_tok, Hq, Hk):
    """kv_len = 3 * 64 + r for every r: the whole tail, its first row and the block's last row poisoned (NaN and +Inf in
    K and V), each against the zero run"""
    segs = [n_tok] if path == "paged" else [1] * n_tok
    gen = torch.Generator(device="cuda").manual_seed(n_tok * 100 + Hq)
    bad = []
    for r in range(64):
        kv_len = 3 * PAGE + r
        _assert_reaches(lib, path, segs, kv_len, Hq, Hk)
        case = _decoder_case(lib, path, segs, kv_len, Hq, Hk, "flat", seed=kv_len + 7 * n_tok + Hq)
        clean = case.run(case.k, case.v)
        assert torch.isfinite(clean.float()).all(), f"kv_len {kv_len}: the zero run is not finite"
        end = case.nblk * PAGE
        modes = {"spare pages": []}
        if r:
            modes = {"tail": slice(kv_len, end), "first tail row": [kv_len], "last row of the block": [end - 1]}
        for mode, rows in modes.items():
            for name in ("nan_7fc1", "+inf"):
                out = case.poisoned(rows, name, "KV", gen)
                if not _same(out, clean):
                    bad.append(f"kv_len {kv_len} {mode} {name}")
    assert not bad, f"masked rows leak into the output: {bad[:12]} ({len(bad)} in all)"


# ============================================================================================ B: ViT attention
VIT_HD = 64


def _vit(lib, qkv, B, N, C_):
    out = torch.empty(B * N, C_, dtype=torch.float16, device="cuda")
    _check(lib.vlo_op_vit_attn(_p(qkv), _p(out), B, N, C_, _st()), "vit_attn")
    torch.cuda.synchronize()
    return out.view(B, N, C_)


@pytest.mark.parametrize("heads", [2, 16])
@pytest.mark.parametrize("N", [36, 257, 576, 577, 639])
def test_vit_attention_frames_ignore_a_poisoned_neighbour(lib, N, heads):
    """all q / k / v rows of frame f, or only its first 64 ceil(N / 64) - N rows (what frame f - 1's last block loads),
    set to +Inf or NaN: every other frame keeps the clean run's bits"""
    B = 3
    C_ = heads * VIT_HD
    qkv, _ = AR._vit_inputs(B, N, heads, seed=N * 10 + heads)
    clean = _vit(lib, qkv, B, N, C_)
    assert torch.isfinite(clean.float()).all()
    spill = (N + 63) // 64 * 64 - N
    bad = []
    for f in range(B):
        spans = {"frame": N}
        if spill:
            spans["spill rows"] = spill
        for what, n in spans.items():
            for bits in (0x7C00, 0x7E01):   # fp16 +Inf, NaN
                x = qkv.clone()
                x[f * N:f * N + n] = torch.full((n, 3 * C_), bits, dtype=torch.int16, device="cuda").view(torch.float16)
                out = _vit(lib, x, B, N, C_)
                for o in range(B):
                    if o != f and not _same(out[o], clean[o]):
                        bad.append(f"frame {f} {what} {bits:#x} -> frame {o}")
    assert not bad, f"a frame's non-finite rows reach another frame: {bad}"


# ============================================================================================ C: engine
FORMS = ["bf16", "fp8", "w8a8"]
IID = 11
POOL_PAGES = 5
FRAME = 11


class _Engines:
    """per weight form two tiny engines with the same weights and a 5-page pool: "clean" never sees a non-finite row,
    "work" is where they are written"""

    def __init__(self):
        self.cache = {}

    def get(self, form, which):
        if (form, which) not in self.cache:
            from videollm_online_b200 import tiny_config, weights as W
            from videollm_online_b200.engine import Engine
            cfg = tiny_config()
            eng = Engine(cfg, "cuda:0", max_streams=4, max_kv_tokens=POOL_PAGES * PAGE, max_step_tokens=64,
                         max_vit_batch=1, kv_pool_tokens=POOL_PAGES * PAGE, fp8_activations=form == "w8a8")
            eng.load_weights(W.synthetic_engine_weights(cfg, "cuda:0", POOL_PAGES * PAGE + 64, seed=5,
                                                        fp8_weights=form != "bf16"))
            self.cache[(form, which)] = eng
        eng = self.cache[(form, which)]
        assert eng.kv_pool_info()["free_pages"] == POOL_PAGES, "a test left pages taken"
        return eng

    def close(self):
        for eng in self.cache.values():
            eng.close()
        self.cache.clear()


@pytest.fixture(scope="module")
def engines():
    e = _Engines()
    yield e
    e.close()


def _embeds(eng, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, eng.cfg.hidden_size, device="cuda", generator=g).bfloat16()


def _run(eng, sids, plan, seed):
    """steps of `plan` on streams `sids`: each entry is (q_lens, segments or None); returns the clones of every step's
    logits and decision rows"""
    outs = []
    for i, (q_lens, segs) in enumerate(plan):
        emb = _embeds(eng, sum(q_lens), seed * 1000 + i)
        lg, dec = eng.step(sids, q_lens, emb, interval_id=IID, segments=segs)
        outs.append((lg.clone(), dec.clone()))
    torch.cuda.synchronize()
    return outs


def _kv(eng, sid):
    return [(eng.kv_read(sid, l, False), eng.kv_read(sid, l, True)) for l in range(eng.cfg.num_hidden_layers)]


def _assert_same_run(got, want, what):
    (g_out, g_kv), (w_out, w_kv) = got, want
    assert len(g_out) == len(w_out)
    for i, ((gl, gd), (wl, wd)) in enumerate(zip(g_out, w_out)):
        assert _same(gl, wl), f"{what}: step {i} logits differ ({int(gl.float().isnan().any(-1).sum())} NaN rows)"
        assert torch.equal(gd, wd), f"{what}: step {i} decision rows differ"
    for l, ((gk, gv), (wk, wv)) in enumerate(zip(g_kv, w_kv)):
        assert _same(gk, wk), f"{what}: layer {l} K differs"
        assert _same(gv, wv), f"{what}: layer {l} V differs"
    assert all(torch.isfinite(o[0].float()).all() for o in w_out)


# stream B of the page-reuse cases: a prompt, frame steps, a segmented backlog step, more frame steps; 250 positions on 4
# pages, so every kv_end mod 64 it crosses sees a different stale tail
B_PLAN = ([([40], None)] + [([FRAME], None)] * 12 + [([2 * FRAME + 1], [[FRAME, FRAME, 1]])] + [([FRAME], None)] * 5)


def _stream_b(eng, seed=7):
    sid = eng.stream_open()
    try:
        return _run(eng, [sid], B_PLAN, seed), _kv(eng, sid)
    finally:
        eng.stream_close(sid)


def _poison_rows(eng, sid, n, lo, hi, gen):
    """write positions [0, n) of every layer's K and V: random rows, NaN / +-Inf at [lo, hi)"""
    nkv, hd = eng.cfg.num_key_value_heads, eng.cfg.head_dim
    for l in range(eng.cfg.num_hidden_layers):
        for is_v in (False, True):
            rows = torch.randn(nkv, n, hd, device="cuda", generator=gen)
            rows[:, lo:hi:3], rows[:, lo + 1:hi:3], rows[:, lo + 2:hi:3] = float("nan"), float("inf"), float("-inf")
            eng.kv_write(sid, l, is_v, rows.bfloat16())
    torch.cuda.synchronize()


def test_inf_embedding_writes_non_finite_kv(engines):
    """the route the kernel guards against: one +Inf embedding row leaves non-finite K and V at its position in every
    layer, in every weight form (the rows before it attend to it through P = 0 from layer 1 on: not checked)"""
    for form in FORMS:
        eng = engines.get(form, "work")
        sid = eng.stream_open()
        try:
            emb = _embeds(eng, FRAME, 1)
            emb[3, 5] = float("inf")
            eng.step([sid], [FRAME], emb, interval_id=IID)
            for l, (k, v) in enumerate(_kv(eng, sid)):
                for name, x in (("K", k), ("V", v)):
                    if l == 0:
                        assert torch.isfinite(x[:, :3].float()).all(), f"{form} layer 0 {name}: rows before the Inf row"
                    assert bool((~torch.isfinite(x[:, 3].float())).any(-1).all()), \
                        f"{form} layer {l} {name}: the Inf row's position is finite"
        finally:
            eng.stream_close(sid)


A_CLEAN, A_LEN = 40, 170    # stream A: clean positions [0, 40), non-finite [40, 170): three pages, the last one to row 42


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("release", ["close", "truncate", "swap_out", "evict", "compact"])
def test_page_reuse_after_non_finite_rows(engines, form, release):
    """stream A's pages hold non-finite rows (also past its length after a truncate, evict or compact); stream B then
    takes every free page, A's among them, and must compute the bits of B on an engine that never saw them"""
    want = _stream_b(engines.get(form, "clean"))
    eng = engines.get(form, "work")
    gen = torch.Generator(device="cuda").manual_seed(3)
    opened = []
    try:
        if release in ("close", "swap_out"):
            opened.append(eng.stream_open())          # holds one page, so B needs all the pages A gives back
            eng.kv_fill_synthetic(opened[-1], 20, seed=9)
        a = eng.stream_open()
        opened.append(a)
        if release == "evict":
            _poison_rows(eng, a, A_LEN, 100, A_LEN, gen)
            eng.kv_truncate(a, 100)                   # positions 100 .. 127 of page 1 stay behind as its tail
            eng.kv_evict(a, 0, PAGE)                  # page 1 becomes A's only page: length 36, rows 36 .. 63 bad
            assert eng.kv_len(a) == 36
        else:
            _poison_rows(eng, a, A_LEN, A_CLEAN, A_LEN, gen)
            if release == "close":
                eng.stream_close(opened.pop())
            elif release == "truncate":
                eng.kv_truncate(a, 30)
            elif release == "swap_out":
                eng.kv_swap_out(a)
            else:
                eng.kv_compact(a, [(0, 20), (30, 10)])   # length 30; rows 40 .. 63 of page 0 stay behind as its tail
                assert eng.kv_len(a) == 30
        assert eng.kv_pool_info()["free_pages"] == 4
        b = eng.stream_open()
        opened.append(b)
        outs = _run(eng, [b], B_PLAN, 7)
        assert eng.kv_pool_info()["free_pages"] == 0, "B did not take every page A gave back"
        got = (outs, _kv(eng, b))
    finally:
        for s in opened:
            eng.stream_close(s)
    _assert_same_run(got, want, f"{form} after {release}")


ROLL_PLAN = [([40], None)] + [([FRAME], None)] * 3     # 73 positions
CONT_PLAN = [([FRAME], None)] * 3 + [([2 * FRAME + 1], [[FRAME, FRAME, 1]])] + [([FRAME], None)] * 2


@pytest.mark.parametrize("form", FORMS)
def test_rollback_past_non_finite_rows(engines, form):
    """a 30-token step of Inf embedding rows writes NaN K / V at positions 73 .. 102; kv_truncate(73) and the stream
    continues (its first step rewrites 73 .. 83 only) with the bits of a stream that never took that step"""
    clean = engines.get(form, "clean")
    s = clean.stream_open()
    try:
        want = (_run(clean, [s], ROLL_PLAN, 1) + _run(clean, [s], CONT_PLAN, 2), _kv(clean, s))
    finally:
        clean.stream_close(s)
    eng = engines.get(form, "work")
    s = eng.stream_open()
    try:
        outs = _run(eng, [s], ROLL_PLAN, 1)
        emb = _embeds(eng, 30, 99)
        emb[:, 0] = float("inf")
        eng.step([s], [30], emb, interval_id=IID)
        assert not bool(torch.isfinite(eng.kv_read(s, 0, True)[:, 73:].float()).any())
        eng.kv_truncate(s, 73)
        got = (outs + _run(eng, [s], CONT_PLAN, 2), _kv(eng, s))
    finally:
        eng.stream_close(s)
    _assert_same_run(got, want, f"{form} rollback")


@pytest.mark.parametrize("form", FORMS)
def test_swap_image_with_non_finite_rows_past_its_length(engines, form):
    """an image whose last page has NaN rows past n_tokens resumes with the bits of the untouched image"""
    from videollm_online_b200.engine import KvImage
    res = {}
    for which in ("clean", "work"):
        eng = engines.get(form, which)
        s = eng.stream_open()
        try:
            outs = _run(eng, [s], ROLL_PLAN, 1)
            img = eng.kv_swap_out(s).synchronize()
            n = img.n_tokens
            assert n % PAGE, "the image must end mid-page"
            if which == "work":
                L, nkv, hd, pt = img.layout
                data = img.data.clone().view(torch.int16).view(-1, L, 2, nkv, pt, hd)
                data[-1, :, :, :, n % PAGE:] = 0x7FC1       # bf16 NaN: the last page's rows past n_tokens, every plane
                img = KvImage(data.view(torch.uint8).reshape(-1).pin_memory(), n, img.layout)
            eng.kv_swap_in(s, img)
            res[which] = (outs + _run(eng, [s], CONT_PLAN, 2), _kv(eng, s))
        finally:
            eng.stream_close(s)
    _assert_same_run(res["work"], res["clean"], f"{form} swap image")


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("segmented", [False, True])
def test_batched_step_with_a_non_finite_stream(engines, form, segmented):
    """stream A with NaN K / V in its live rows and a clean stream B in one ragged (or segmented) step: B's logits,
    decision rows and K / V equal those of the same step with A clean"""
    res = {}
    for which in ("clean", "work"):
        eng = engines.get(form, which)
        a, b = eng.stream_open(), eng.stream_open()
        try:
            _run(eng, [a], [([30], None)], 5)
            _run(eng, [b], [([40], None)], 6)
            if which == "work":
                emb = _embeds(eng, FRAME, 98)
                emb[2, 1] = float("inf")
                eng.step([a], [FRAME], emb, interval_id=IID)
            else:
                _run(eng, [a], [([FRAME], None)], 8)
            plan = [([FRAME, 2 * FRAME + 1], [[FRAME], [FRAME, FRAME, 1]] if segmented else None)] * 3
            outs = _run(eng, [a, b], plan, 9)
            rows_b = slice(1, None)    # A has one logits / decision row per step, B the rest
            res[which] = ([(lg[rows_b], dec[rows_b]) for lg, dec in outs], _kv(eng, b))
        finally:
            eng.stream_close(a)
            eng.stream_close(b)
    _assert_same_run(res["work"], res["clean"], f"{form} batched segmented={segmented}")
