"""The decoder step's persistent bf16 GEMM against exact references at every token tile, and vlo_step replayed bit for
bit from the kernel-level entry points (which launch each kernel through the engine's own helper and default plan).

A.  gemm_ws_kernel in the forms the decoder runs: mode 0 (stream-K fp32 partial planes: q|k|v, o_proj, down_proj) and
    mode 1 (whole tiles, bf16 epilogue: lm_head), at T in every token tile (16 with its 6-stage ring, 32, 64, 96, 128),
    each with a full last tile and a one-row spill.  Every plane is checked on its own against the k-blocks of the one
    CTA that wrote it, restated from streamk.h; random operands are held to an accumulation bound per plane.
B.  One sequence's vlo_step chained from the entries in step_segments' order, in the three weight forms (bf16,
    fp8_weights, fp8_weights + fp8_activations): logits, decision rows, the final hidden rows and every layer's K and V
    must equal the engine's bit for bit.
"""
import ctypes as C
import pathlib
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = pathlib.Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests"))
import test_gpu_decoder_kernels as DK  # noqa: E402  (stream-K plane counts, SM count, bf16 sentinels)

U = 2.0 ** -24
FMT_BF16 = 1
ACT_NONE = 0
WS_TILE_FIT = 0
FIX_MAX_PLANES = 8                      # kFixMaxPlanes


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


def token_tile(T):
    """gemm.cu token_tile() for bf16 activations: the smallest instance covering T rows (16, 32, 64, 96, 128)"""
    for bn in (16, 32, 64, 96):
        if T <= bn:
            return bn
    return 128


# ============================================================================================ stream-K plan, restated
class SkPlan:
    """streamk.h for a mode-0 GEMM of N output features, K, over one token tile: units = (128-row tile, 64-wide
    k-block), CTA c of G = min(n_ctas or SM count, U) owns units [sk_lo(c), sk_lo(c + 1)); the planes of tile t are
    CTAs sk_first_cta(t) .. sk_owner(last unit of t), plane index = CTA - sk_first_cta(t)."""

    def __init__(self, N, K, n_ctas):
        self.tiles, self.kb = (N + 127) // 128, K // 64
        self.U = self.tiles * self.kb
        self.G = min(n_ctas if n_ctas > 0 else DK._n_sm(), self.U)
        self.ranges = []          # per tile: the k-block range [a, b) of each of its planes, in plane order
        for t in range(self.tiles):
            first, last = self.first_cta(t), self.owner((t + 1) * self.kb - 1)
            t0, t1 = t * self.kb, (t + 1) * self.kb
            rr = [(max(self.lo(c), t0) - t0, min(self.lo(c + 1), t1) - t0) for c in range(first, last + 1)]
            assert rr[0][0] == 0 and rr[-1][1] == self.kb and all(a < b for a, b in rr)
            assert all(rr[i][1] == rr[i + 1][0] for i in range(len(rr) - 1))
            self.ranges.append(rr)
        self.planes = max(len(r) for r in self.ranges)

    def lo(self, c):
        return (c * self.U) // self.G

    def owner(self, u):
        c = min((u * self.G) // self.U, self.G - 1)
        while self.lo(c + 1) <= u:
            c += 1
        while c > 0 and self.lo(c) > u:
            c -= 1
        return c

    def first_cta(self, t):
        return self.owner(t * self.kb)

    def column_ranges(self, N):
        """[planes, N] k-block bounds a, b of plane p at output feature n (a = b = 0 where tile n // 128 has no plane p)"""
        a = torch.zeros(self.planes, N, dtype=torch.long)
        b = torch.zeros(self.planes, N, dtype=torch.long)
        for t, rr in enumerate(self.ranges):
            n0, n1 = t * 128, min(N, t * 128 + 128)
            for p, (lo, hi) in enumerate(rr):
                a[p, n0:n1], b[p, n0:n1] = lo, hi
        return a.cuda(), b.cuda()


def _block_prefix(x, w, fn=lambda v: v):
    """prefix sums over 64-wide k-blocks: out[j][t, n] = sum over k < 64 j of fn(x[t, k]) fn(w[n, k]), [kb + 1, T, N],
    in the dtype of x"""
    T, K = x.shape
    N = w.shape[0]
    blocks = torch.einsum("tbk,nbk->btn", fn(x).view(T, K // 64, 64), fn(w).view(N, K // 64, 64))
    return torch.cat([torch.zeros(1, T, N, dtype=x.dtype, device=x.device), blocks.cumsum(0)], 0), blocks


def _plane_ref(prefix, a, b):
    """[planes, T, N]: prefix[b] - prefix[a] at every column, NaN where the tile has no such plane"""
    T = prefix.shape[1]
    ga = prefix.gather(0, a[:, None, :].expand(-1, T, -1))
    gb = prefix.gather(0, b[:, None, :].expand(-1, T, -1))
    return torch.where((b > a)[:, None, :], gb - ga, torch.full_like(ga, float("nan")))


def _run_planes(lib, w, x, N, K, n_ctas, plan_sk):
    """vlo_op_gemm_ws_tiled mode 0 into planes + 1 NaN-filled planes; returns them after checking the plan it reports"""
    T = x.shape[0]
    plan = (C.c_int32 * 3)()
    _check(lib.vlo_op_gemm_ws_tiled(FMT_BF16, 0, _p(w), N, _p(x), T, K, None, N, T * N, None, ACT_NONE, n_ctas, 0,
                                    WS_TILE_FIT, plan, _st()), "plan")
    assert list(plan) == [token_tile(T), 1, plan_sk.planes], f"plan {list(plan)} for T={T}"
    out = torch.full((plan_sk.planes + 1, T, N), float("nan"), device="cuda")
    _check(lib.vlo_op_gemm_ws_tiled(FMT_BF16, 0, _p(w), N, _p(x), T, K, _p(out), N, T * N, None, ACT_NONE, n_ctas, 0,
                                    WS_TILE_FIT, plan, _st()), "gemm_ws")
    torch.cuda.synchronize()
    return out


# ============================================================================================ A1: every plane, exactly
GEMM_T = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128]
LLAMA_SHAPES = [(6144, 4096), (4096, 4096), (28672, 4096), (4096, 14336)]  # q|k|v, o_proj, gate|up, down of Llama-3-8B
TINY_SHAPES = [(1024, 256), (256, 512)]                                     # tiny_config: q|k|v and gate|up, o and down
ODD_SHAPE = (1000, 1024)                                                    # N not a multiple of 128


@pytest.fixture(scope="module")
def int_operands():
    """per (N, K): w and 128 token rows with values in {-2 .. 2}: every partial sum is an integer of magnitude at most
    4 K <= 57344 < 2^24, so the fp32 accumulation is exact in any order, and so is the fp32 reference below"""
    cache = {}

    def get(N, K):
        if (N, K) not in cache:
            g = torch.Generator(device="cuda").manual_seed(N * 7 + K)
            w = torch.randint(-2, 3, (N, K), device="cuda", generator=g).bfloat16()
            x = torch.randint(-2, 3, (128, K), device="cuda", generator=g).bfloat16()
            cache[(N, K)] = (w, x)
        return cache[(N, K)]
    return get


def _planes_exact_case(lib, int_operands, N, K, T, n_ctas):
    w, x_all = int_operands(N, K)
    x = x_all[:T].contiguous()
    sk = SkPlan(N, K, n_ctas)
    out = _run_planes(lib, w, x, N, K, n_ctas, sk)
    prefix, _ = _block_prefix(x.float(), w.float())
    ref = _plane_ref(prefix, *sk.column_ranges(N))
    what = f"N={N} K={K} T={T} n_ctas={n_ctas} (G={sk.G}, {sk.planes} planes)"
    got = out[:sk.planes]
    ok = (got == ref) | (got.isnan() & ref.isnan())
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:4].tolist()
        raise AssertionError(f"{what}: {int((~ok).sum())} plane entries differ; at [plane, t, n] {bad} got "
                             f"{[got[tuple(i)].item() for i in bad]}, want {[ref[tuple(i)].item() for i in bad]}")
    assert out[sk.planes].isnan().all(), what + ": the plane past `planes` was written"
    return sk


@pytest.mark.parametrize("n_ctas", [0, 37, 7])
@pytest.mark.parametrize("T", GEMM_T)
@pytest.mark.parametrize("N,K", LLAMA_SHAPES + TINY_SHAPES + [ODD_SHAPE])
def test_gemm_ws_planes_exact(lib, int_operands, N, K, T, n_ctas):
    """mode 0: plane p of weight tile w equals, bit for bit, the sum over exactly the k-blocks of CTA
    sk_first_cta(w) + p; planes a tile does not use, and one plane past the plan's count, keep their NaN"""
    _planes_exact_case(lib, int_operands, N, K, T, n_ctas)


@pytest.mark.parametrize("T", [1, 16, 17, 97, 128])
@pytest.mark.parametrize("N,K", [(4096, 4096), (256, 512), ODD_SHAPE])
def test_gemm_ws_planes_exact_eight_planes(lib, int_operands, N, K, T):
    """the smallest CTA count whose plan gives some tile exactly kFixMaxPlanes planes"""
    n_ctas = DK._ctas_for_planes(N, K, FIX_MAX_PLANES)
    sk = _planes_exact_case(lib, int_operands, N, K, T, n_ctas)
    assert sk.planes == FIX_MAX_PLANES


# ============================================================================================ A2: accumulation bound
@pytest.mark.parametrize("T", [1, 16, 17, 33, 65, 97, 128])
@pytest.mark.parametrize("N,K", [(6144, 4096), (4096, 14336)])
def test_gemm_ws_planes_accumulation_bound(lib, N, K, T):
    """Random operands, whose sums are not exact: each plane against the fp64 sum of its own k-range within
    E_p = 4 K_p u S_p, S_p = sum over that range of |x w| (test_gpu_vit_kernels.py::test_gemm_accumulation_bound,
    per plane).  Self-check: the reference without any one 64-wide k-block leaves most elements outside E_p, so the
    bound sees a lost or doubled block."""
    g = torch.Generator(device="cuda").manual_seed(N + K + T)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).bfloat16()
    x = torch.randn(T, K, device="cuda", generator=g).bfloat16()
    sk = SkPlan(N, K, 0)
    out = _run_planes(lib, w, x, N, K, 0, sk)
    a, b = sk.column_ranges(N)
    prefix, blocks = _block_prefix(x.double(), w.double())
    exact = _plane_ref(prefix, a, b)
    del prefix
    aprefix, _ = _block_prefix(x.double(), w.double(), torch.abs)
    E = 4 * (b - a)[:, None, :].double() * 64 * U * _plane_ref(aprefix, a, b)
    del aprefix
    got = out[:sk.planes].double()
    live = (b > a)[:, None, :].expand_as(got)
    err = (got - exact).abs()
    assert bool((err[live] <= E[live]).all()), \
        f"N={N} K={K} T={T}: plane error {float((err[live] / E[live]).max()):.2f} x the derived bound"
    assert got[~live].isnan().all() and out[sk.planes].isnan().all(), "an unused plane was written"
    # plane of k-block j at column n: the p with a[p, n] <= j < b[p, n]
    j = torch.arange(sk.kb, device="cuda")[:, None, None]
    pidx = ((j >= a[None]) & (j < b[None])).double().argmax(1)               # [kb, N]
    Ej = E.gather(0, pidx[:, None, :].expand(-1, T, -1))                     # [kb, T, N]
    frac = (blocks.abs() > Ej).double().flatten(1).mean(1)
    assert bool((frac > 0.5).all()), f"k-block {int(frac.argmin())} hides inside the bound ({float(frac.min()):.2f})"


# ============================================================================================ A3: lm_head form
LM_T = [1, 8, 16, 17, 33, 97, 128]
SENTINEL16 = 0x7FC1


@pytest.fixture(scope="module")
def lm_operands():
    """per (V, K): w, 128 token rows and a bias, x and w = k 2^-6 with |k| <= 16 (exact in bf16): products are multiples
    of 2^-12 below 2^-4, so every partial sum over K = 4096 is a multiple of 2^-12 below 2^8 (20 bits) and exact in fp32
    in any order, also in the reference (whose TF32 mode, if on, holds these 5-bit inputs exactly)"""
    cache = {}

    def get(V, K):
        if (V, K) not in cache:
            g = torch.Generator(device="cuda").manual_seed(V + K)
            w = (torch.randint(-16, 17, (V, K), device="cuda", generator=g).float() / 64).bfloat16()
            x = (torch.randint(-16, 17, (128, K), device="cuda", generator=g).float() / 64).bfloat16()
            bias = (torch.randn(V, device="cuda", generator=g) * 2).bfloat16().float()
            cache[(V, K)] = (w, x, bias)
        return cache[(V, K)]
    return get


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("T", LM_T)
@pytest.mark.parametrize("V,K", [(128256, 4096), (1024, 256)])
def test_gemm_ws_lm_head_exact(lib, lm_operands, V, K, T, bias):
    """mode 1, bf16, no activation: out == bf16(acc) bit for bit (with a bias: bf16(fp32(acc + bias))), at the Llama-3
    vocabulary and at the tiny one (8 tiles, fewer than SMs); ld_out > V with sentinels past V and past T that must
    survive.  T <= 16 runs the decoder's 6-stage 16-token instance."""
    w, x_all, b = lm_operands(V, K)
    x = x_all[:T].contiguous()
    ld = V + 8
    out = torch.full((T + 2, ld), SENTINEL16, dtype=torch.int16, device="cuda").view(torch.bfloat16)
    plan = (C.c_int32 * 3)()
    _check(lib.vlo_op_gemm_ws_tiled(FMT_BF16, 1, _p(w), V, _p(x), T, K, _p(out), ld, 0, _p(b) if bias else None, ACT_NONE,
                                    0, 0, WS_TILE_FIT, plan, _st()), "gemm_ws lm_head")
    torch.cuda.synchronize()
    assert list(plan) == [token_tile(T), 1, 1], f"plan {list(plan)}"
    acc = x.float() @ w.float().t()
    if bias:
        acc = acc + b[None, :]                     # the kernel's one fp32 add: acc is exact, the sum rounds once
    want = acc.bfloat16()
    got = out[:T, :V]
    if not DK._same_bits(got, want):
        bad = (got.view(torch.int16) != want.view(torch.int16)).nonzero()[:4].tolist()
        raise AssertionError(f"V={V} T={T} bias={bias}: {len(bad)}+ logits differ; at {bad} got "
                             f"{[got[tuple(i)].item() for i in bad]}, want {[want[tuple(i)].item() for i in bad]}")
    assert bool((want.float() != acc).any()), "no logit needed rounding: the case cannot see a wrong rounding point"
    assert DK._same_bits(out[:T, V:], DK._sentinel(T, ld - V)), "columns past V were written"
    assert DK._same_bits(out[T:], DK._sentinel(2, ld)), "rows past T were written"


# ============================================================================================ B: vlo_step replayed
FORMS = ["bf16", "fp8", "w8a8"]
IID = 11                                   # the interval id every replayed step decides on
MAX_KV = 512
ROPE_ROWS = MAX_KV + 64                    # every replayed step ends well below the RoPE table's last row


class _Engines:
    """one engine per (width, weight form), built on first use and closed with the module"""

    def __init__(self):
        self.cache = {}

    def get(self, width, form):
        if (width, form) not in self.cache:
            from videollm_online_b200 import llama3_8b_siglip_l, tiny_config, weights as W
            from videollm_online_b200.engine import Engine
            if width == "tiny":
                cfg = tiny_config()
            else:
                cfg = llama3_8b_siglip_l()
                cfg.num_hidden_layers, cfg.vision_num_hidden_layers = 2, 1   # the vision tower is not under test
            eng = Engine(cfg, "cuda:0", max_streams=4 if width == "tiny" else 1, max_kv_tokens=MAX_KV,
                         max_step_tokens=128, max_vit_batch=1, fp8_activations=form == "w8a8")
            eng.load_weights(W.synthetic_engine_weights(cfg, "cuda:0", ROPE_ROWS, seed=5, fp8_weights=form != "bf16"))
            assert eng.fp8_weights == (form != "bf16") and eng.fp8_activations == (form == "w8a8")
            self.cache[(width, form)] = (cfg, eng)
        return self.cache[(width, form)]

    def close(self):
        for _, eng in self.cache.values():
            eng.close()
        self.cache.clear()


@pytest.fixture(scope="module")
def engines():
    e = _Engines()
    yield e
    e.close()


class _Kv:
    """one layer's K or V cache of the replayed sequence: contiguous [n_kv][cap][128] (vlo_op_attn_kvappend's layout) or
    64-token pages [cap / 64][n_kv][64][128] under an identity page table (vlo_op_attn_kvappend_segments').  Rows past
    the cached ones start at a NaN sentinel: the attention must not see the rows past kv_len it loads, and a row the
    replayed append fails to write stays NaN."""

    def __init__(self, rows, cap, paged):
        nkv, n, hd = rows.shape
        self.nkv, self.cap, self.paged = nkv, cap, paged
        c = torch.full((nkv, cap, hd), float("nan"), dtype=torch.bfloat16, device="cuda")
        c[:, :n] = rows
        self.buf = c.view(nkv, cap // 64, 64, hd).permute(1, 0, 2, 3).contiguous() if paged else c

    def row(self, pos):
        """the row of KV head 0 at position pos; head_stride() rows further per head"""
        return (pos // 64) * self.nkv * 64 + pos % 64 if self.paged else pos

    def head_stride(self):
        return 64 if self.paged else self.cap

    def contiguous(self, n):
        c = self.buf.permute(1, 0, 2, 3).reshape(self.nkv, self.cap, -1) if self.paged else self.buf
        return c[:, :n]


def _replay(lib, cfg, eng, form, P, embeds, row_ids, segs, kv0):
    """step_segments for one sequence of past length P, chained from the kernel-level entries in the engine's order with
    their default plans.  kv0[l] = (K, V) of layer l before the step (Engine.kv_read).  Returns (logits, decisions,
    hidden, [(K, V) after the step per layer])."""
    Wt = eng.weights
    st = _st()
    T, H = embeds.shape
    nh, nkv, hd, I, V = (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim, cfg.intermediate_size,
                         cfg.vocab_size)
    A, QKV, eps = nh * hd, (nh + 2 * nkv) * hd, cfg.rms_norm_eps
    a8, f8 = form == "w8a8", form != "bf16"
    bf = dict(dtype=torch.bfloat16, device="cuda")
    n_rows = len(segs)
    last_index = [-1] * T
    end = 0
    for s, n in enumerate(segs):
        end += n
        last_index[end - 1] = s
    li = torch.tensor(last_index, dtype=torch.int32, device="cuda")

    # residual stream: the packed embeddings, rows with an id >= 0 gathered from the embedding table
    h = embeds.clone()
    if row_ids is not None:
        take = row_ids >= 0
        h[take] = Wt["embed"][row_ids[take]]
    xn, xn_last = torch.empty(T, H, **bf), torch.empty(n_rows, H, **bf)
    xq = torch.empty(T, H, dtype=torch.uint8, device="cuda")
    xs = torch.empty(T, device="cuda")

    def norm(part, k, w, last):
        if a8 and not last:
            _check(lib.vlo_op_resid_rmsnorm_q8(_p(part), k, 0, _p(h), _p(w), _p(xn), None, None, _p(xq), _p(xs), T, H, eps,
                                               st), "resid_rmsnorm_q8")
        else:
            _check(lib.vlo_op_resid_rmsnorm(_p(part), k, 0, _p(h), _p(w), _p(xn), _p(xn_last) if last else None,
                                            _p(li) if last else None, T, H, eps, st), "resid_rmsnorm")

    def quant(x, K):
        q = torch.empty(T, K, dtype=torch.uint8, device="cuda")
        s = torch.empty(T, device="cuda")
        _check(lib.vlo_op_quant_rows_e4m3(_p(x), T, K, _p(q), _p(s), st), "quant_rows_e4m3")
        return q, s

    def planes(name, x, x_scale, N, K):
        """the partial planes of the step's dec_partial for this layer matrix"""
        n = C.c_int(0)
        for out in (None, "alloc"):
            if out == "alloc":
                out = torch.empty(n.value, T, N, device="cuda")
            if a8:
                _check(lib.vlo_op_gemm_ws_a8(_p(Wt[name + ".f8"]), _p(Wt[name + ".scale"]), N, _p(x), _p(x_scale), T, K,
                                             _p(out), T * N, 0, C.byref(n), st), "gemm_ws_a8")
            elif f8:
                _check(lib.vlo_op_gemm_ws_f8(_p(Wt[name + ".f8"]), _p(Wt[name + ".scale"]), N, _p(x), T, K, _p(out),
                                             T * N, 0, C.byref(n), st), "gemm_ws_f8")
            else:
                plan = (C.c_int32 * 3)()
                _check(lib.vlo_op_gemm_ws_tiled(FMT_BF16, 0, _p(Wt[name]), N, _p(x), T, K, _p(out), N, T * N, None,
                                                ACT_NONE, 0, 0, WS_TILE_FIT, plan, st), "gemm_ws")
                assert plan[0] == token_tile(T)
                n.value = plan[2]
        assert n.value <= FIX_MAX_PLANES
        return out

    def swiglu(name, x, x_scale):
        N = 2 * I
        buf = torch.empty(max(1, max(DK._sk_planes(N, H, 0)) - 1) * T * N, device="cuda")
        flags = torch.zeros(N // 128, dtype=torch.int32, device="cuda")
        act = torch.empty(T, I, **bf)
        tail = (_p(act), _p(buf), buf.numel(), _p(flags), flags.numel(), st)
        if a8:
            _check(lib.vlo_op_gemm_swiglu_a8(_p(Wt[name + ".f8"]), _p(Wt[name + ".scale"]), N, _p(x), _p(x_scale), T, H,
                                             *tail), "gemm_swiglu_a8")
        elif f8:
            _check(lib.vlo_op_gemm_swiglu_f8(_p(Wt[name + ".f8"]), _p(Wt[name + ".scale"]), N, _p(x), T, H, *tail),
                   "gemm_swiglu_f8")
        else:
            _check(lib.vlo_op_gemm_swiglu(_p(Wt[name]), N, _p(x), T, H, *tail), "gemm_swiglu")
        return act

    paged = n_rows > 1
    kv_len = P + T
    cap = (kv_len + 63) // 64 * 64
    kv = [(_Kv(k, cap, paged), _Kv(v, cap, paged)) for k, v in kv0]
    cos, sin = Wt["rope.cos"], Wt["rope.sin"]
    h_pos = (C.c_int32 * T)(*range(P, P + T))
    h_row = (C.c_int64 * T)(*[kv[0][0].row(P + j) for j in range(T)])
    q = torch.empty(T, nh, hd, **bf)
    attn = torch.empty(T, A, **bf)
    ws = torch.empty(int(lib.vlo_op_attn_ws_bytes(T, nh, hd, kv_len)) // 4 + 1, device="cuda")
    seg_arr = (C.c_int32 * n_rows)(*segs)
    pt = torch.arange(cap // 64, dtype=torch.int32, device="cuda")

    norm(None, 0, Wt["L0.in_norm"], False)
    for l in range(cfg.num_hidden_layers):
        L = f"L{l}."
        xin, xsc = (xq, xs) if a8 else (xn, None)
        part = planes(L + "qkv", xin, xsc, QKV, H)
        kc, vc = kv[l]
        _check(lib.vlo_op_qkv_rope_append(_p(part), H, 0, _p(cos), _p(sin), cos.shape[0], h_pos, h_row, kc.head_stride(),
                                          _p(q), _p(kc.buf), _p(vc.buf), T, nh, nkv, st), "qkv_rope_append")
        if paged:
            _check(lib.vlo_op_attn_kvappend_segments(_p(q), _p(kc.buf), _p(vc.buf), _p(pt), cap // 64, _p(attn), n_rows,
                                                     seg_arr, nh, nkv, hd, kv_len, st), "attn_kvappend_segments")
        else:
            _check(lib.vlo_op_attn_kvappend(_p(q), _p(kc.buf), _p(vc.buf), _p(attn), _p(ws), T, nh, nkv, hd, kv_len, cap,
                                            st), "attn_kvappend")
        aq, asc = quant(attn, A) if a8 else (attn, None)
        part = planes(L + "o", aq, asc, H, A)
        norm(part, A, Wt[L + "post_norm"], False)
        xin, xsc = (xq, xs) if a8 else (xn, None)
        act = swiglu(L + "gate_up", xin, xsc)
        actq, acts = quant(act, I) if a8 else (act, None)
        part = planes(L + "down", actq, acts, H, I)
        last = l == cfg.num_hidden_layers - 1
        norm(part, I, Wt["final_norm"] if last else Wt[f"L{l + 1}.in_norm"], last)
    logits = torch.empty(n_rows, V, **bf)
    plan = (C.c_int32 * 3)()
    _check(lib.vlo_op_gemm_ws_tiled(FMT_BF16, 1, _p(Wt["lm_head"]), V, _p(xn_last), n_rows, H, _p(logits), V, 0, None,
                                    ACT_NONE, 0, 0, WS_TILE_FIT, plan, st), "lm_head")
    assert plan[0] == token_tile(n_rows)
    dec = torch.full((n_rows, 8), -7, dtype=torch.int32, device="cuda")
    _check(lib.vlo_op_decision(_p(logits), n_rows, V, IID, _p(dec), st), "decision")
    torch.cuda.synchronize()
    return logits, dec, xn, [(k.contiguous(kv_len), v.contiguous(kv_len)) for k, v in kv]


def _step_case(lib, engines, width, form, P, T, segs=None, row_ids=None, fragment=False, seed=0):
    cfg, eng = engines.get(width, form)
    H = cfg.hidden_size
    others = []
    if fragment:
        # two streams grown in turns, then one closed: its pages 0 and 2 are handed out next, so the replayed stream's
        # cache rows are neither the identity nor contiguous across its page boundary
        others = [eng.stream_open(), eng.stream_open()]
        for n in (64, 128):
            for s in others:
                eng.kv_fill_synthetic(s, n, seed=n + s)
        eng.stream_close(others.pop(0))
    sid = eng.stream_open()
    try:
        if P:
            eng.kv_fill_synthetic(sid, P, seed=seed + 1)
        g = torch.Generator(device="cuda").manual_seed(seed)
        embeds = torch.randn(T, H, device="cuda", generator=g).bfloat16()
        ids = None
        if row_ids is not None:
            ids = torch.tensor(row_ids, dtype=torch.int64, device="cuda")
        kv0 = [(eng.kv_read(sid, l, False), eng.kv_read(sid, l, True)) for l in range(cfg.num_hidden_layers)]
        logits, dec = eng.step([sid], [T], embeds, row_ids=ids, interval_id=IID, segments=[segs] if segs else None)
        logits, dec = logits.clone(), dec.clone()
        hidden = eng.last_step_hidden(T)
        kv1 = [(eng.kv_read(sid, l, False), eng.kv_read(sid, l, True)) for l in range(cfg.num_hidden_layers)]
        torch.cuda.synchronize()
        r_logits, r_dec, r_hidden, r_kv = _replay(lib, cfg, eng, form, P, embeds, ids, segs or [T], kv0)
    finally:
        eng.stream_close(sid)
        for s in others:
            eng.stream_close(s)
    what = f"{width} {form} P={P} T={T} segs={segs} row_ids={'yes' if row_ids is not None else 'no'}"
    def rows_off(a, b):
        return (a.view(torch.int16) != b.view(torch.int16)).flatten(0, -2).any(-1).nonzero().flatten().tolist()[:8]

    for l, ((k, v), (rk, rv)) in enumerate(zip(kv1, r_kv)):
        assert DK._same_bits(k, rk), f"{what}: layer {l} K differs in (head, position) rows {rows_off(k, rk)}"
        assert DK._same_bits(v, rv), f"{what}: layer {l} V differs in (head, position) rows {rows_off(v, rv)}"
    assert DK._same_bits(hidden, r_hidden), f"{what}: last_step_hidden differs in rows {rows_off(hidden, r_hidden)}"
    assert DK._same_bits(logits, r_logits), f"{what}: logits differ in rows {rows_off(logits, r_logits)}"
    assert torch.equal(dec, r_dec), f"{what}: decision rows differ"
    assert not r_logits.isnan().any() and not r_hidden.isnan().any()


STEP_T = [1, 16, 17, 33, 64, 65, 97, 128]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("T", STEP_T)
def test_step_replay_token_tiles(lib, engines, form, T):
    """every decoder token tile, over 40 cached positions"""
    _step_case(lib, engines, "tiny", form, 40, T, seed=T)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("P,T", [(60, 17), (60, 70)])
def test_step_replay_page_boundaries(lib, engines, form, P, T):
    """new rows straddling one and two 64-token page boundaries, on a fragmented page pool"""
    _step_case(lib, engines, "tiny", form, P, T, fragment=True, seed=P + T)


@pytest.mark.parametrize("form", FORMS)
def test_step_replay_row_ids(lib, engines, form):
    """rows gathered from the embedding table by id (>= 0, including vocab - 1) mixed with packed embeddings (< 0)"""
    V = 1024
    ids = [(-1 if j % 3 == 1 else (j * 37) % V) for j in range(33)]
    ids[5], ids[32] = V - 1, V - 1
    _step_case(lib, engines, "tiny", form, 5, 33, row_ids=ids, seed=33)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("segs", [[1, 10, 1, 10], [1, 1, 1, 1], [7, 1, 24]])
def test_step_replay_segments(lib, engines, form, segs):
    """one lm_head row and one decision per segment, each read at its segment's last token"""
    _step_case(lib, engines, "tiny", form, 20, sum(segs), segs=segs, seed=len(segs) + sum(segs))


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("T", [1, 11, 128])
def test_step_replay_full_width(lib, engines, form, T):
    """two layers at Llama-3-8B width (4096 / 32 heads / 8 kv heads / 14336 / 128256): every GEMM has several planes"""
    _step_case(lib, engines, "full", form, 70, T, seed=100 + T)
