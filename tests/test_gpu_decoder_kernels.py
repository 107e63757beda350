"""The decoder step's fix-up, SwiGLU and decision kernels against plain references, through the kernel-level entry points
(which launch them with the step's own helpers).

References run in torch on the device: fp64 where a value is computed, explicit fp32 / bf16 rounding where a kernel
claims a rounding point.

Exactness rule.  An output must equal the bf16 rounding of its reference value bit for bit, except an element whose
fp64 pre-rounding value lies within a relative margin delta of a bf16 rounding boundary: that one may take either
neighbour (`_either`).  Each test derives its delta from the kernel's approximations, in units of u = 2^-24 (half an
fp32 ulp, the relative error of one fp32 rounding), with a factor 2 of headroom.  Every delta below is at most 2^-15;
the fraction of elements that are ambiguous is asserted small, so the rule cannot pass vacuously.
"""
import ctypes as C
import math
import pathlib
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = pathlib.Path(__file__).resolve().parents[1]
U = 2.0 ** -24
FIX_MAX_PLANES = 8                      # kFixMaxPlanes: planes the fix-up kernels unroll
SENTINEL16 = 0x7FC1                     # a NaN bit pattern: rows nobody may write keep it


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


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sk_planes(width, k, n_ctas):
    """planes of each 128-feature tile for the stream-K split of a GEMM with `width` outputs over one token tile
    (CTA c owns units [c U / G, (c + 1) U / G); a tile's planes = the CTAs that touch it)"""
    tiles, kb = (width + 127) // 128, k // 64
    U_ = tiles * kb
    G = min(n_ctas if n_ctas > 0 else _n_sm(), U_)
    lo = lambda c: (c * U_) // G
    def owner(u):
        c = min((u * G) // U_, G - 1)
        while lo(c + 1) <= u:
            c += 1
        while c > 0 and lo(c) > u:
            c -= 1
        return c
    return [owner((t + 1) * kb - 1) - owner(t * kb) + 1 for t in range(tiles)]


def _ctas_for_planes(width, k, want):
    """the smallest CTA count whose split gives some tile exactly `want` planes and none more"""
    U_ = ((width + 127) // 128) * (k // 64)
    for G in range(1, U_ + 1):
        if max(_sk_planes(width, k, G)) == want:
            return G
    raise AssertionError(f"no split of {width} x {k} has {want} planes")


def _poisoned_planes(T, width, ns, gen, scale=1.0):
    """random fp32 planes [kFixMaxPlanes, T, width]; every plane at or past ns(tile) is NaN"""
    part = torch.randn(FIX_MAX_PLANES, T, width, device="cuda", generator=gen) * scale
    ns_col = torch.tensor(ns, device="cuda").repeat_interleave(128)[:width]
    live = torch.arange(FIX_MAX_PLANES, device="cuda")[:, None] < ns_col[None, :]
    return part.masked_fill(~live[:, None, :], float("nan")), ns_col


def _fixup_sum(part, ns_col):
    """y = sum_{s < ns} part[s] in plane order in fp32, as the fix-up kernels add them"""
    y = part[0].clone()
    for s in range(1, part.shape[0]):
        y = torch.where(s < ns_col[None, :], y + part[s], y)
    return y


def _bf(x):
    """bf16 value of an fp64 tensor, as fp64.  Via fp32: the double rounding can only differ from a direct rounding
    within 2^-24 of a midpoint, which every delta here covers."""
    return x.float().bfloat16().double()


def _either(x64, delta):
    """the two bf16 values an fp64 pre-rounding value may take under the exactness rule (equal when unambiguous)"""
    d = delta if torch.is_tensor(delta) else torch.tensor(delta, dtype=torch.float64, device=x64.device)
    a, b = _bf(x64 * (1 - d)), _bf(x64 * (1 + d))
    return torch.minimum(a, b), torch.maximum(a, b)


def _assert_in(out, cands, what, max_ambiguous=0.02):
    """out (any float dtype) equals one of the candidate tensors elementwise; few elements have two candidates"""
    o = out.double()
    ok = torch.zeros_like(o, dtype=torch.bool)
    for c in cands:
        ok |= o == c
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:4]
        got = [o[tuple(i)].item() for i in bad]
        want = [[c[tuple(i)].item() for c in cands] for i in bad]
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements off; at {bad.tolist()} got {got}, "
                             f"allowed {want}")
    amb = (cands[0] != cands[-1]).double().mean().item()
    assert amb <= max_ambiguous, f"{what}: {amb:.3%} of the elements are ambiguous: the margin is too loose"


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _sentinel(*shape):
    return torch.full(shape, SENTINEL16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


# ============================================================================================ resid_rmsnorm
EPS = 1e-5


def _norm_delta(H):
    """Relative error bound of the kernel's pre-rounding value h * rstd.  blockDim = min(1024, max(32, H / 4)); a thread
    adds n_seq = 4 ceil(H / (4 blockDim)) squares in sequence, then 5 warp and 5 block shuffle levels follow: the sum
    of squares is within (n_seq + 11) u (squares rounded once each).  / H and + eps: 2 u; rsqrtf: 2 ulp = 4 u, and
    the square root halves the sum's error; the product with h: 1 u.  delta = 2 (0.5 (n_seq + 13) + 5) u, which is
    2^-19.4 at H = 8192."""
    bd = min(1024, max(32, H // 4))
    n_seq = 4 * math.ceil(H / (4 * bd))
    return 2 * (0.5 * (n_seq + 13) + 5) * U


def _run_resid(lib, part, k, n_ctas, h, w, n_last, last_index, eps=EPS):
    T, H = h.shape
    xn = _sentinel(T, H)
    xn_last = _sentinel(n_last, H) if n_last else None
    li = torch.tensor(last_index, dtype=torch.int32, device="cuda") if last_index is not None else None
    _check(lib.vlo_op_resid_rmsnorm(_p(part), k, n_ctas, _p(h), _p(w), _p(xn), _p(xn_last), _p(li), T, H, eps, _st()),
           "resid_rmsnorm")
    torch.cuda.synchronize()
    return xn, xn_last


def _check_norm(h_new, w, xn, xn_last, last_index, what):
    """xn under the exactness rule; xn_last rows = the xn rows last_index names, every other row untouched"""
    H = h_new.shape[1]
    hd = h_new.double()
    eps32 = float(torch.tensor(EPS, dtype=torch.float32))     # what the kernel receives
    rstd = 1.0 / torch.sqrt((hd * hd).mean(1, keepdim=True) + eps32)
    lo, hi = _either(hd * rstd, _norm_delta(H))
    wd = w.double()[None, :]
    _assert_in(xn, [_bf(wd * lo), _bf(wd * hi)], what + " xn")   # bf16 x bf16 products are exact: one rounding
    if xn_last is not None:
        exp = _sentinel(*xn_last.shape)
        for t, slot in enumerate(last_index):
            if slot >= 0:
                exp[slot] = xn[t]
        assert _same_bits(xn_last, exp), what + ": xn_last rows differ from the named xn rows or an unnamed row changed"


def _last_index(T, gen):
    """some rows named, to slots out of order; two slots are never named"""
    named = torch.randperm(T, generator=gen)[:max(1, T // 3)].tolist()
    n_last = len(named) + 2
    slots = torch.randperm(n_last, generator=gen)[:len(named)].tolist()
    li = [-1] * T
    for t, s in zip(named, slots):
        li[t] = s
    return li, n_last


def _resid_case(lib, H, T, n_ctas, k, scale, seed, part=None, ns=None):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    cgen = torch.Generator().manual_seed(seed)
    if part is None:
        ns = _sk_planes(H, k, n_ctas)
        part, ns_col = _poisoned_planes(T, H, ns, gen, scale)
    else:
        ns_col = torch.tensor(ns, device="cuda").repeat_interleave(128)[:H]
    h = (torch.randn(T, H, device="cuda", generator=gen) * scale).bfloat16()
    w = (1 + 0.25 * torch.randn(H, device="cuda", generator=gen)).bfloat16()
    h_ref = (h.float() + _fixup_sum(part, ns_col).bfloat16().float()).bfloat16()
    li, n_last = _last_index(T, cgen)
    xn, xn_last = _run_resid(lib, part, k, n_ctas, h, w, n_last, li)
    what = f"H={H} T={T} n_ctas={n_ctas} k={k} scale={scale}"
    assert _same_bits(h, h_ref), what + ": h != bf16(h + bf16(sum of the tile's planes))"
    _check_norm(h_ref, w, xn, xn_last, li, what)


def _resid_k(H):
    """k of the producing GEMM: a split over all SMs stays within 8 planes (2 and 3 tiles of 8 k-blocks: 8 planes)"""
    return 512 if H < 1024 else 1024


@pytest.mark.parametrize("H", [256, 384, 4096, 8192])
@pytest.mark.parametrize("T", [1, 11, 128])
@pytest.mark.parametrize("split", ["1", "3", "all", "8planes"])
def test_resid_rmsnorm_fixup(lib, H, T, split):
    """h' = bf16(h + bf16(sum_{s < ns} planes)) bit for bit, xn and xn_last under the exactness rule; planes past ns are
    NaN.  H = 384 runs 3 warps, H = 8192 the second sweep (re-planned plane count, weight not prefetched)."""
    k = _resid_k(H)
    if split == "8planes":
        n_ctas = _ctas_for_planes(H, k, FIX_MAX_PLANES)
        assert max(_sk_planes(H, k, n_ctas)) == FIX_MAX_PLANES
    else:
        n_ctas = {"1": 1, "3": 3, "all": 0}[split]
    _resid_case(lib, H, T, n_ctas, k, 1.0, H * 131 + T)


@pytest.mark.parametrize("scale", [1e-3, 1e4])
@pytest.mark.parametrize("H", [384, 8192])
def test_resid_rmsnorm_magnitudes(lib, H, scale):
    """rows of magnitude 1e-3 (eps matters) and 1e4"""
    _resid_case(lib, H, 11, 0, _resid_k(H), scale, 7)


@pytest.mark.parametrize("H", [256, 384, 4096, 8192])
def test_resid_rmsnorm_no_partials(lib, H):
    """part == NULL: h untouched, plain RMSNorm (the first layer's input norm)"""
    gen = torch.Generator(device="cuda").manual_seed(H)
    T = 11
    h = torch.randn(T, H, device="cuda", generator=gen).bfloat16()
    h0 = h.clone()
    w = (1 + 0.25 * torch.randn(H, device="cuda", generator=gen)).bfloat16()
    li, n_last = _last_index(T, torch.Generator().manual_seed(H))
    xn, xn_last = _run_resid(lib, None, 0, 0, h, w, n_last, li)
    assert _same_bits(h, h0)
    _check_norm(h0, w, xn, xn_last, li, f"H={H} no partials")


@pytest.mark.parametrize("H,T,k,n_ctas", [(4096, 11, 4096, 0), (8192, 128, 1024, 37), (384, 1, 14336, 5)])
def test_resid_rmsnorm_fed_by_gemm_ws(lib, H, T, k, n_ctas):
    """planes written by the real producer (vlo_op_gemm_ws mode 0, same k / n_ctas): the two plans must agree, so the
    planes the producer leaves unwritten (NaN) are never read"""
    gen = torch.Generator(device="cuda").manual_seed(k + T)
    wg = (torch.randn(H, k, device="cuda", generator=gen) * 0.05).bfloat16()
    x = torch.randn(T, k, device="cuda", generator=gen).bfloat16()
    part = torch.full((FIX_MAX_PLANES, T, H), float("nan"), device="cuda")
    planes = C.c_int(0)
    _check(lib.vlo_op_gemm_ws(1, 0, _p(wg), H, _p(x), T, k, _p(part), H, T * H, None, 0, n_ctas, 0, C.byref(planes),
                              _st()), "gemm_ws")
    ns = _sk_planes(H, k, n_ctas)
    assert planes.value == max(ns) <= FIX_MAX_PLANES
    _resid_case(lib, H, T, n_ctas, k, 1.0, 3, part=part, ns=ns)


def test_fixup_entries_reject_what_the_kernels_cannot_do(lib):
    """more than one token tile, or a plan of more planes than the kernels unroll, fails before any launch"""
    from videollm_online_b200._lib import VloError
    H, k = 256, 1024
    h = torch.zeros(129, H, device="cuda").bfloat16()
    w = torch.ones(H, device="cuda").bfloat16()
    part = torch.zeros(FIX_MAX_PLANES, 129, H, device="cuda")
    with pytest.raises(VloError, match="token rows"):
        _check(lib.vlo_op_resid_rmsnorm(_p(part), k, 0, _p(h), _p(w), None, None, None, 129, H, EPS, _st()), "r")
    g9 = _ctas_for_planes(H, k, FIX_MAX_PLANES + 1)
    with pytest.raises(VloError, match="partial planes"):
        _check(lib.vlo_op_resid_rmsnorm(_p(part), k, g9, _p(h), _p(w), None, None, None, 11, H, EPS, _st()), "r")
    pos = (C.c_int32 * 1)(5)
    row = (C.c_int64 * 1)(0)
    with pytest.raises(VloError, match="RoPE tables"):
        _check(lib.vlo_op_qkv_rope_append(_p(part), k, 1, _p(w), _p(w), 5, pos, row, 64, _p(h), _p(h), _p(h), 1, 1, 1,
                                          _st()), "q")


# ============================================================================================ qkv_rope_append
ROPE_POS = 66048
LISTED_POS = [0, 63, 64, 8191, 8192, 12000, 66010]


@pytest.fixture(scope="module")
def rope():
    from videollm_online_b200 import tiny_config, weights as W
    return W.rope_tables(tiny_config(), ROPE_POS, "cuda")


def _rotate_half(x):
    return torch.cat((-x[..., 64:], x[..., :64]), -1)


def _tokens(T, gen):
    """(stream, position) pairs, all distinct: the listed positions spread over three streams, then random ones"""
    toks = [(i % 3, p) for i, p in enumerate(LISTED_POS)][:T]
    seen = set(toks)
    while len(toks) < T:
        tk = (int(torch.randint(0, 3, (1,), generator=gen)), int(torch.randint(0, ROPE_POS - 38, (1,), generator=gen)))
        if tk not in seen:
            seen.add(tk)
            toks.append(tk)
    return toks


@pytest.mark.parametrize("nh,nkv", [(32, 8), (4, 2), (8, 8), (8, 1)])
@pytest.mark.parametrize("T", [1, 7, 128])
@pytest.mark.parametrize("layout", ["paged", "contiguous"])
def test_qkv_rope_append(lib, rope, nh, nkv, T, layout):
    """q and the K / V rows bit for bit against HF's apply_rotary_pos_emb in bf16 over the same tables (V unrotated);
    planes past ns are NaN; every cache row the step does not own keeps its sentinel"""
    cos, sin = rope
    k = 4096
    width = (nh + 2 * nkv) * 128
    # all SMs where that split fits the fix-up kernels (the 8B model's 6144-wide q|k|v: 4 planes), else 8 or 2 planes
    n_ctas = {(4, 2): _ctas_for_planes(width, k, FIX_MAX_PLANES), (8, 8): 5, (8, 1): 5}.get((nh, nkv), 0)
    gen = torch.Generator(device="cuda").manual_seed(nh * 100 + nkv + T)
    cgen = torch.Generator().manual_seed(T + nkv)
    ns = _sk_planes(width, k, n_ctas)
    part, ns_col = _poisoned_planes(T, width, ns, gen)
    toks = _tokens(T, cgen)
    pos = [p for _, p in toks]
    if layout == "paged":
        # every (stream, 64-token page) the tokens touch gets its own page of a pool, scattered and out of order
        pages = sorted({(s, p // 64) for s, p in toks})
        n_pages = len(pages) + 5
        phys = torch.randperm(n_pages, generator=cgen)[:len(pages)].tolist()
        table = dict(zip(pages, phys))
        stride = 64
        rows = [(table[(s, p // 64)] * nkv) * 64 + p % 64 for s, p in toks]
        pool_rows = n_pages * nkv * 64
    else:
        ld = ROPE_POS        # [stream][kv head][ld][128]
        stride = ld
        rows = [s * nkv * ld + p for s, p in toks]
        pool_rows = 3 * nkv * ld
    kc, vc = _sentinel(pool_rows, 128), _sentinel(pool_rows, 128)
    q = _sentinel(T, nh, 128)
    h_pos = (C.c_int32 * T)(*pos)
    h_row = (C.c_int64 * T)(*rows)
    _check(lib.vlo_op_qkv_rope_append(_p(part), k, n_ctas, _p(cos), _p(sin), ROPE_POS, h_pos, h_row, stride, _p(q), _p(kc),
                                      _p(vc), T, nh, nkv, _st()), "qkv_rope_append")
    torch.cuda.synchronize()
    y = _fixup_sum(part, ns_col).bfloat16().view(T, nh + 2 * nkv, 128)
    pt = torch.tensor(pos, device="cuda")
    c = torch.cat([cos[pt], cos[pt]], -1)[:, None, :]
    s = torch.cat([sin[pt], sin[pt]], -1)[:, None, :]
    qk = y[:, :nh + nkv]
    rot = qk * c + _rotate_half(qk) * s          # bf16 ops: each product and the sum round once
    assert _same_bits(q, rot[:, :nh]), f"q differs (nh={nh} nkv={nkv} T={T})"
    kv_rows = (torch.tensor(rows, device="cuda")[:, None] + torch.arange(nkv, device="cuda")[None, :] * stride).reshape(-1)
    k_exp, v_exp = _sentinel(pool_rows, 128), _sentinel(pool_rows, 128)
    k_exp[kv_rows] = rot[:, nh:].reshape(-1, 128)
    v_exp[kv_rows] = y[:, nh + nkv:].reshape(-1, 128)
    assert _same_bits(kc, k_exp), f"K cache differs (nh={nh} nkv={nkv} T={T} {layout})"
    assert _same_bits(vc, v_exp), f"V cache differs (nh={nh} nkv={nkv} T={T} {layout})"


# ============================================================================================ gemm_swiglu
SWIGLU_T = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128]
SWIGLU_SHAPES = [(512, 256), (320, 1024), (14336, 4096)]
FLT_MAX = 3.4028234663852886e38


@pytest.fixture(scope="module")
def swiglu_operands():
    """per (I, K): interleaved gate|up weights (a quarter of the gate rows scaled so that gates reach +-100 and silu
    saturates both ways) and 128 token rows"""
    from videollm_online_b200 import weights as W
    ops = {}
    for I, K in SWIGLU_SHAPES:
        gen = torch.Generator(device="cuda").manual_seed(I + K)
        gs = torch.where(torch.arange(I, device="cuda") % 4 == 0, 40.0, 1.0)[:, None]
        gate = (torch.randn(I, K, device="cuda", generator=gen) * gs / math.sqrt(K)).bfloat16()
        up = (torch.randn(I, K, device="cuda", generator=gen) / math.sqrt(K)).bfloat16()
        x = torch.randn(128, K, device="cuda", generator=gen).bfloat16()
        ops[(I, K)] = (W.interleave_gate_up(gate, up), x)
    return ops


def _silu_delta():
    """silu = g / (1 + expf(-g)) in fp32: expf is within 2 ulp (4 u), 1 + e and the division round once each:
    delta = 2 (4 + 1 + 1) u = 2^-20.4"""
    return 12 * U


@pytest.mark.parametrize("T", SWIGLU_T)
@pytest.mark.parametrize("I,K", SWIGLU_SHAPES)
def test_gemm_swiglu(lib, swiglu_operands, I, K, T):
    """act = bf16(bf16(silu(g)) * u) where g | u are the bf16 plane sums of vlo_op_gemm_ws mode 0 on the same operands
    (same planner, token tile and mainloop: the same partials), under the exactness rule; then against an fp64 matmul
    within the accumulation bound.  Twice in a row: identical outputs, arrival counters back at zero after each."""
    wgu, x_all = swiglu_operands[(I, K)]
    x = x_all[:T].contiguous()
    N = 2 * I
    ns = _sk_planes(N, K, 0)
    planes_buf = torch.full((max(1, max(ns) - 1) * T * N,), float("nan"), device="cuda")
    flags = torch.zeros(N // 128 + 3, dtype=torch.int32, device="cuda")
    outs = []
    for _ in range(2):
        act = _sentinel(T + 3, I)
        _check(lib.vlo_op_gemm_swiglu(_p(wgu), N, _p(x), T, K, _p(act), _p(planes_buf), planes_buf.numel(), _p(flags),
                                      flags.numel(), _st()), "gemm_swiglu")
        torch.cuda.synchronize()
        assert int(flags.abs().sum()) == 0, "the finisher left arrival counters set"
        assert _same_bits(act[T:], _sentinel(3, I)), "rows past rows_x were written"
        outs.append(act[:T])
    assert _same_bits(outs[0], outs[1]), "two launches on the same operands differ"
    act = outs[0]

    # bit-exact reference from the unfused producer's planes
    planes = C.c_int(0)
    _check(lib.vlo_op_gemm_ws(1, 0, _p(wgu), N, _p(x), T, K, None, N, T * N, None, 0, 0, 0, C.byref(planes), _st()), "plan")
    assert planes.value == max(ns)
    ws = torch.zeros(planes.value, T, N, device="cuda")
    _check(lib.vlo_op_gemm_ws(1, 0, _p(wgu), N, _p(x), T, K, _p(ws), N, T * N, None, 0, 0, 0, C.byref(planes), _st()),
           "gemm_ws")
    torch.cuda.synchronize()
    y = _fixup_sum(ws, torch.tensor(ns, device="cuda").repeat_interleave(128)).bfloat16().double()
    y = y.view(T, I // 64, 2, 64)
    g, u = y[:, :, 0].reshape(T, I), y[:, :, 1].reshape(T, I)
    e = torch.exp(-g)
    silu = torch.where(e > FLT_MAX, -0.0 * g.abs(), g / (1 + e))   # expf overflows to inf there: silu = -0, as in fp32
    lo, hi = _either(silu, _silu_delta())
    _assert_in(act, [_bf(lo * u), _bf(hi * u)], f"SwiGLU I={I} K={K} T={T}")
    assert bool((g.abs() > 88.8).any()) or T * I < 2048, "no saturated gate in the case"

    # independent: fp64 matmul.  The fp32 accumulation of K products (wgmma, stream-K planes, their sum) is within
    # (K + 8) 2^-23 sum|x w| (one ulp per addition, truncation allowed); the bf16 roundings of g, u, silu and the product
    # add 2^-8 relative each (rounding to nearest gives 2^-9).
    ref = x.double() @ wgu.double().t()
    acc = (K + 8) * 2.0 ** -23 * (x.double().abs() @ wgu.double().abs().t())
    ref, acc = ref.view(T, I // 64, 2, 64), acc.view(T, I // 64, 2, 64)
    g64, u64 = ref[:, :, 0].reshape(T, I), ref[:, :, 1].reshape(T, I)
    eg = acc[:, :, 0].reshape(T, I) + 2.0 ** -8 * g64.abs() * 1.01
    eu = acc[:, :, 1].reshape(T, I) + 2.0 ** -8 * u64.abs() * 1.01
    s64 = g64 * torch.sigmoid(g64)
    bound = 1.1 * eg * u64.abs() + (s64.abs() + 1.1 * eg) * eu + 2 * 2.0 ** -8 * (s64.abs() + 1.1 * eg) * (u64.abs() + eu)
    err = (act.double() - s64 * u64).abs()
    assert bool((err <= bound + 1e-30).all()), f"fp64 reference: worst excess {(err - bound).max().item()}"


# ============================================================================================ decision
VOCABS = [128256, 1024, 8, 8200]


def _n_seq(V):
    """logits one thread takes in sweep A in sequence: 8 per 16-byte vector, vectors strided by the 1024 threads"""
    return 8 * math.ceil(V / 8 / 1024)


def _p_delta(V, dx):
    """Relative error bound of the kernel's pre-rounding probability __expf(x - max) / sum, dx = |x - max|.
    x - max: up to 1 u of rounding, relative to z = x - max, so |z| u.  __expf(z) = ex2.approx(z log2 e): 2 ulp (4 u)
    plus the rounding of the scaled argument, |z| u.  The sum: n_seq sequential additions per thread, 10 shuffle merges;
    each term and each rescale __expf(m_old - m_new) contributes relatively |z| e^-|z| u <= 0.37 u on top of its 4 u,
    so the sum is within (n_seq + 10 + 5) u.  The division: 1 u.
    delta = 2 (n_seq + 15 + 4 + 2 dx + 1) u, 2^-15.8 for the top of a 128 256-entry row."""
    return 2 * (_n_seq(V) + 20 + 2 * dx) * U


def _ref(row, iid):
    x = row.double()
    V = x.numel()
    m1 = x.max()
    top = (x == m1).nonzero().flatten()
    i1 = int(top[0])
    m2 = m1 if top.numel() > 1 else x[x < m1].max() if V > 1 else torch.tensor(float("-inf"))
    z = x - m1
    se = torch.exp(z).sum()
    lse = float(m1 + torch.log(se))
    p = torch.exp(z) / se
    lo, hi = _either(p, _p_delta(V, z.abs()))
    ftz = z < -87.33                       # __expf flushes results below 2^-126 to zero
    lo = torch.where(ftz, torch.zeros_like(lo), lo)
    return dict(x=x, m1=float(m1), m2=float(m2), i1=i1, lse=lse, lo=lo, hi=hi, V=V, iid=iid, se_err=(_n_seq(V) + 15) * U)


def _first_argmax_ok(idx, lo, hi, x, zeroed=None):
    """can `idx` be the first index of the max of values v_i in {lo_i, hi_i}?  The kernel's probability is a monotone
    function of the logit, so equal logits give equal probabilities exactly"""
    if idx < 0 or idx >= x.numel():
        return False
    for m in {float(lo[idx]), float(hi[idx])}:
        if bool((lo > m).any()) or bool((lo[:idx] >= m).any()):
            continue
        same = x[:idx] == x[idx]
        if zeroed is not None and zeroed < idx:
            same[zeroed] = False
        if idx != zeroed and bool(same.any()):
            continue
        return True
    return False


def _check_decision(d, r, what):
    V, iid = r["V"], r["iid"]
    assert d["argmax_id"] == r["i1"], what + ": argmax_id"
    assert d["max_logit"] == r["m1"], what + ": max_logit"
    assert d["top2_margin"] == float(torch.tensor(r["m1"] - r["m2"], dtype=torch.float32)), what + ": top2_margin"
    tol = 2 * r["se_err"] + 4 * U * (abs(r["lse"]) + abs(r["m1"]))
    assert abs(d["lse"] - r["lse"]) <= tol, what + f": lse {d['lse']} vs {r['lse']}"
    if 0 <= iid < V:
        lo, hi = float(r["lo"][iid]), float(r["hi"][iid])
        assert d["p_interval"] in (lo, hi), what + f": p_interval {d['p_interval']} not in {{{lo}, {hi}}}"
    else:
        assert d["p_interval"] == 0.0
    assert _first_argmax_ok(d["argmax_prob_id"], r["lo"], r["hi"], r["x"]), \
        what + f": argmax_prob_id {d['argmax_prob_id']}"
    lo, hi = r["lo"].clone(), r["hi"].clone()
    if 0 <= iid < V:
        lo[iid] = hi[iid] = 0.0
    assert _first_argmax_ok(d["argmax_excl_id"], lo, hi, r["x"], zeroed=iid if 0 <= iid < V else None), \
        what + f": argmax_excl_id {d['argmax_excl_id']}"


def _run_decision(lib, rows, iid):
    from videollm_online_b200.engine import Decision
    n, V = rows.shape
    out = torch.full((n, 8), -7, dtype=torch.int32, device="cuda")
    _check(lib.vlo_op_decision(_p(rows), n, V, iid, _p(out), _st()), "decision")
    torch.cuda.synchronize()
    oi, of = out.cpu(), out.cpu().view(torch.float32)
    res = []
    for i in range(n):
        dec = Decision(oi[i], of[i])
        res.append((dec, {s: getattr(dec, s) for s in Decision.__slots__}))
    return res


def _bfv(v):
    return float(torch.tensor(v).bfloat16())


def _prob_tie_row(V, gen):
    """the max logit at a higher index than a slightly smaller logit whose bf16 probability is the same: the probability
    argmax is the smaller logit's index.  Three more logits c move the normalisation until the fp64 row has the
    property unambiguously."""
    x = torch.full((V,), -30.0, dtype=torch.float64)
    a, b, c = (7, 1, [2, 3, 4]) if V <= 8 else (V - 3, 1, [5, 6, 7])
    x[a], x[b] = 0.5, 0.5 - 2.0 ** -8
    for cv in torch.arange(0.4375, -4.0, -1.0 / 64):
        x[c] = _bfv(float(cv))
        row = x.bfloat16().cuda()
        r = _ref(row, -1)
        if bool((r["lo"] == r["hi"]).all()) and r["lo"][a] == r["lo"][b] and bool((r["lo"] <= r["lo"][a]).all()):
            assert r["i1"] == a and _first_argmax_ok(b, r["lo"], r["hi"], r["x"]) and b != r["i1"]
            return row
    raise AssertionError("no probability tie found")


def _p_interval_row(V, target, iid):
    """a row whose bf16 softmax at iid is `target`, away from a rounding boundary: the interval logit 0, a competitor at
    a searched bf16 logit, everything else far below"""
    x = torch.full((V,), -40.0, dtype=torch.float64)
    x[iid] = 0.0
    comp = (iid + 3) % V
    best = None
    for dv in torch.arange(-1.25, -0.75, 1.0 / 256):
        x[comp] = _bfv(float(dv))
        r = _ref(x.bfloat16().cuda(), iid)
        pz = float(torch.exp(r["x"][iid] - r["lse"]))
        if float(r["lo"][iid]) == float(r["hi"][iid]) == target:
            margin = abs(pz - target)
            if best is None or margin < best[0]:
                best = (margin, float(x[comp]))
    assert best is not None, f"no row with p_interval {target}"
    x[comp] = best[1]
    return x.bfloat16().cuda()


def _decision_rows(V, gen):
    """named rows of one vocab: (name, row, interval id)"""
    cases = []
    iid = (V // 3 + 1) if V > 8 else 3
    for sig in (1.0, 10.0, 30.0):
        cases.append((f"random sigma {sig}", (torch.randn(V, generator=gen) * sig).bfloat16(), iid))
    def tied(idxs, name, iid_=iid):
        r = torch.randn(V, generator=gen).bfloat16()
        for i in idxs:
            r[i] = 6.0
        cases.append((name, r, iid_))
    tied([min(V - 1, 8 * 2 + 2), min(V - 1, 8 * 2 + 5)] if V > 8 else [2, 5], "max tied in one 8-vector")
    if V >= 1024:
        tied([8 * 3 + 1, 8 * 17 + 6], "max tied across threads of a warp")
    if V >= 8200:
        tied([8 * 40 + 7, 8 * 1000 + 0], "max tied across warps")
        tied([8 * 1024 + 3, 8 * 5 + 3], "max tied in the vector past the threads and thread 5")
    tied([0, V - 1], "max tied at 0 and vocab-1")
    r = torch.randn(V, generator=gen).bfloat16(); r[iid] = 7.0
    cases.append(("interval id the unique max", r, iid))
    lo_i, hi_i = max(0, iid - 2), min(V - 1, iid + 2)
    r = torch.randn(V, generator=gen).bfloat16(); r[iid] = 7.0; r[lo_i] = 7.0
    cases.append(("interval id tied with the max at a lower index", r, iid))
    r = torch.randn(V, generator=gen).bfloat16(); r[iid] = 7.0; r[hi_i] = 7.0
    cases.append(("interval id tied with the max at a higher index", r, iid))
    cases.append(("bf16 probability tie without a logit tie", _prob_tie_row(V, gen).cpu(), iid))
    for at in (V // 2, 0):
        r = torch.randn(V, generator=gen).bfloat16(); r[at] = 200.0
        cases.append((f"dominant logit at {at}, interval id 0", r, 0))
        cases.append((f"dominant logit at {at}", r, iid))
    cases.append(("uniform", torch.zeros(V).bfloat16(), iid))
    return cases


@pytest.mark.parametrize("V", VOCABS)
def test_decision_rows(lib, V):
    """every field against fp64 (argmax_id, max_logit, top2_margin exact; p_interval under the exactness rule; the
    probability argmaxes among the ambiguous set only; lse within the sum's bound).  V = 8: one vector, every other
    thread empty; V = 8200: one vector more than threads."""
    gen = torch.Generator().manual_seed(V)
    for name, row, iid in _decision_rows(V, gen):
        rr = row.cuda()[None].contiguous()
        (_, d), = _run_decision(lib, rr, iid)
        _check_decision(d, _ref(rr[0], iid), f"V={V} {name}")
    # the probability-tie case is not vacuous: the probability argmax differs from the logit argmax
    row = _prob_tie_row(V, gen)
    (_, d), = _run_decision(lib, row[None].contiguous(), -1)
    assert d["argmax_prob_id"] != d["argmax_id"]


@pytest.mark.parametrize("V", [128256, 1024])
def test_decision_eight_rows_in_one_launch(lib, V):
    gen = torch.Generator().manual_seed(V + 8)
    rows = (torch.randn(8, V, generator=gen) * torch.tensor([0.5, 1, 2, 3, 5, 10, 20, 30])[:, None]).bfloat16()
    rows[3, 17] = rows[3].max()      # a tie in one of them
    iid = 11
    got = _run_decision(lib, rows.cuda(), iid)
    for i, (_, d) in enumerate(got):
        _check_decision(d, _ref(rows[i].cuda(), iid), f"V={V} row {i} of 8")


THRESHOLDS = [0.0, 0.3, 0.5, 0.725, 0.9, 1.0]


@pytest.mark.parametrize("V", [128256, 1024, 8])
def test_decision_threshold_rule_matches_reference(lib, V):
    """p_interval of bf16(0.725) = 0.7265625 and one bf16 ulp to either side, and random rows: Decision.next_id(thr)
    equals the reference's rule (bf16 softmax in torch on the GPU, then vlo_oracle.decide)"""
    sys.path.insert(0, str(ROOT / "oracle"))
    import vlo_oracle as O
    iid = min(V - 1, 5)
    ulp = 2.0 ** -8
    targets = [0.7265625 - ulp, 0.7265625, 0.7265625 + ulp]
    assert _bfv(0.725) == 0.7265625
    rows = [_p_interval_row(V, t, iid) for t in targets]
    gen = torch.Generator().manual_seed(V)
    rows += [(torch.randn(V, generator=gen) * s).bfloat16().cuda() for s in (1.0, 3.0)]
    n_checked = 0
    for j, row in enumerate(rows):
        (dec, d), = _run_decision(lib, row[None].contiguous(), iid)
        r = _ref(row, iid)
        if j < 3:
            assert d["p_interval"] == targets[j]
        _check_decision(d, r, f"V={V} threshold row {j}")
        if j >= 3 and not bool((r["lo"] == r["hi"]).all()):
            continue                       # an ambiguous probability may round either way in torch's softmax too
        for thr in THRESHOLDS:
            assert dec.next_id(iid, thr) == O.decide(row.clone(), iid, thr), f"V={V} row {j} thr={thr}"
        n_checked += 1
    assert n_checked >= 3
