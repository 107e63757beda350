"""The vision tower kernel by kernel against plain references, through the kernel-level entry points (which launch the
kernels with vlo_vit_encode's own helpers), and vlo_vit_encode replayed bit for bit from those entry points at every
frame-batch tiling the engine runs.

References run in torch on the device: fp64 where a value is computed, explicit fp32 / fp16 rounding where a kernel
claims a rounding point.

Exactness rule (fp16).  An output must equal the fp16 rounding of its reference value, except an element whose fp64
pre-rounding value lies within an absolute margin E of an fp16 rounding boundary: it may take either neighbour
(`_either16`).  Each test derives E from the kernel's approximations, in units of u = 2^-24 (half an fp32 ulp), with a
factor 2 of headroom, and asserts that few elements are ambiguous, so the rule cannot pass vacuously.

Operands are chosen so that the sums a kernel forms are exact in fp32 in any order wherever the kernel's summation
order is not part of its contract (GEMM accumulators, LayerNorm means): dyadic values of few significant bits.
"""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
FIX_MAX_PLANES = 8                      # kFixMaxPlanes
NAN16 = {torch.float16: 0x7E01, torch.bfloat16: 0x7FC1}   # NaN bit patterns: elements nobody may write keep them
EPS = 1e-6                              # SigLIP's layer_norm_eps
ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF_PY = 0, 1, 2
EPI_STORE16, EPI_PATCH32 = 1, 3
FMT_F16, FMT_BF16 = 0, 1
ERFF_ULP = 2                            # CUDA C Programming Guide: erff, maximum ulp error


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


def _nan16(*shape, dtype=torch.float16):
    return torch.full(shape, NAN16[dtype], dtype=torch.int16, device="cuda").view(dtype)


def _nan32(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    it = torch.int16 if a.element_size() == 2 else torch.int32
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(it), b.view(it))


def _r16(x, dtype=torch.float16):
    """16-bit value of an fp32 tensor, as fp32 (one rounding)"""
    return x.float().to(dtype).float()


def _either16(x64, E, dtype=torch.float16):
    """the 16-bit values an fp64 pre-rounding value within an absolute error E may round to (lo, hi).  Via fp32: the
    double rounding can only differ from a direct rounding within 2^-24 relative of a midpoint, inside every E here."""
    a = (x64 - E).float().to(dtype).double()
    b = (x64 + E).float().to(dtype).double()
    return a, b


def _assert_between(out, lo, hi, what, max_ambiguous=0.03):
    """lo <= out <= hi elementwise, and lo, hi are at most one 16-bit step apart for all but few elements"""
    o = out.double()
    ok = (o >= lo) & (o <= hi)
    if not bool(ok.all()):
        bad = (~ok).nonzero()[:4]
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.numel()} elements outside the bound; at {bad.tolist()} "
                             f"got {[o[tuple(i)].item() for i in bad]}, allowed "
                             f"{[(lo[tuple(i)].item(), hi[tuple(i)].item()) for i in bad]}")
    amb = (lo != hi).double().mean().item()
    assert amb <= max_ambiguous, f"{what}: {amb:.3%} of the elements are ambiguous: the margin is too loose"


def _dyadic(shape, lim, scale_log2, gen, offset=0.0):
    """offset + k 2^-scale_log2, k uniform in [-lim, lim]: few significant bits, so sums stay exact in fp32"""
    k = torch.randint(-lim, lim + 1, shape, device="cuda", generator=gen).double()
    return k * 2.0 ** -scale_log2 + offset


# ============================================================================================ patchify
def _patch_table():
    """fp16((x / 255 - 0.5) / 0.5) of every byte value, computed in fp64 and rounded once (numpy rounds fp64 -> fp16
    directly)"""
    import numpy as np
    x = np.arange(256, dtype=np.float64)
    return torch.from_numpy(((x / 255.0 - 0.5) / 0.5).astype(np.float16)).cuda()


def _patchify_ref(frames, ps):
    B, _, S, _ = frames.shape
    g = S // ps
    t = frames.view(B, 3, g, ps, g, ps).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, 3 * ps * ps)
    return _patch_table()[t.long()]


def _run_patchify(lib, frames, ps, extra_rows=3):
    B, _, S, _ = frames.shape
    rows = B * (S // ps) ** 2
    out = _nan16(rows + extra_rows, 3 * ps * ps)
    _check(lib.vlo_op_patchify(_p(frames), B, S, ps, _p(out), _st()), "patchify")
    torch.cuda.synchronize()
    return out, rows


def test_patchify_every_byte_value(lib):
    """every byte value in every lane of the 8-pixel vector load (frame b holds (i + b) % 256 at pixel i, so value x
    sits in lane (x - b) % 8): bit for bit against the fp64 formula"""
    S = ps = 16
    frames = ((torch.arange(3 * S * S, device="cuda")[None, :] + torch.arange(8, device="cuda")[:, None]) % 256)
    frames = frames.to(torch.uint8).view(8, 3, S, S).contiguous()
    out, rows = _run_patchify(lib, frames, ps)
    assert _same_bits(out[:rows], _patchify_ref(frames, ps))
    assert _same_bits(out[rows:], _nan16(*out[rows:].shape)), "rows past B * P were written"


@pytest.mark.parametrize("S", [96, 384])
@pytest.mark.parametrize("B", [1, 3, 5])
def test_patchify_im2col_order(lib, S, B):
    """random frames: row b P + py g + px, column (c ps + iy) ps + ix; nothing past B * P rows written"""
    gen = torch.Generator(device="cuda").manual_seed(S + B)
    frames = torch.randint(0, 256, (B, 3, S, S), device="cuda", generator=gen, dtype=torch.int32).to(torch.uint8)
    out, rows = _run_patchify(lib, frames, 16)
    assert _same_bits(out[:rows], _patchify_ref(frames, 16))
    assert _same_bits(out[rows:], _nan16(*out[rows:].shape)), "rows past B * P were written"


# ============================================================================================ 16-bit GEMM epilogues
def _gemm_operands(M, N, K, gen, dtype=torch.float16):
    """x, w = k 2^-6 with |k| <= 16: products are multiples of 2^-12 below 2^-4, so every partial sum over K <= 4096 is
    a multiple of 2^-12 below 2^8 (20 bits) and exact in fp32 in any order; the sums are not 16-bit values, so the
    epilogue's rounding points show.  Bias: any 16-bit value, as pack_*_for_engine holds it."""
    x = _dyadic((M, K), 16, 6, gen).to(dtype)
    w = _dyadic((N, K), 16, 6, gen).to(dtype)
    bias = (torch.randn(N, device="cuda", generator=gen) * 0.5).to(dtype).float()
    acc = x.double() @ w.double().t()            # exact
    return x, w, bias, acc


def _tanh_approx(lib, x):
    """tanh.approx.f32 of an fp32 tensor, by the instruction the GELU-tanh epilogue runs"""
    x = x.contiguous()
    y = _nan32(*x.shape)
    _check(lib.vlo_op_tanh_approx(_p(x), _p(y), x.numel(), _st()), "tanh_approx")
    return y


def _gelu_tanh_candidates(lib, v, dtype):
    """The 16-bit values the GELU-tanh epilogue may give for its 16-bit input v (an fp32 tensor), emulated in fp32 in the
    kernel's order: inner = k0 (v + ((k1 v) v) v), the last product and the add either rounded one by one or contracted
    into one FMA (two candidates); th = tanh.approx.f32(inner) from the same instruction; out = r16(fl(0.5 v) fl(1 + th))
    with one fp32 rounding of the product.  A wrong constant, or an erf form in place of the tanh form, changes inner or
    th, and with it the rounded output of a large share of the elements."""
    k0 = torch.tensor(0.7978845608028654, dtype=torch.float32)
    k1 = torch.tensor(0.044715, dtype=torch.float32)
    t = (k1 * v) * v
    separate = v + t * v
    # t v is exact in fp64 (24 + 24 bits); the fp64 add can double-round only within 2^-29 of an fp32 midpoint
    fused = (t.double() * v.double() + v.double()).float()
    outs = []
    for s_ in (separate, fused):
        th = _tanh_approx(lib, k0 * s_)
        outs.append(_r16((0.5 * v) * (1.0 + th), dtype))
    return outs


def _epilogue_check(lib, out, acc, bias, act, what, dtype=torch.float16):
    """out == act(r16(acc + bias)) under the rounding points the epilogue claims"""
    v = _r16(acc.float() + bias[None, :], dtype)     # the fp32 add (acc exact in fp32), then one 16-bit rounding
    if act == ACT_NONE:
        assert _same_bits(out, v.to(dtype)), what + ": out != r16(acc + bias)"
        return
    if act == ACT_GELU_TANH:
        c0, c1 = (c.double() for c in _gelu_tanh_candidates(lib, v, dtype))
        ok = (out.double() == c0) | (out.double() == c1)
        if not bool(ok.all()):
            bad = (~ok).nonzero()[:4]
            raise AssertionError(f"{what} gelu_tanh: {int((~ok).sum())} of {ok.numel()} elements off; at {bad.tolist()} "
                                 f"v {[v[tuple(i)].item() for i in bad]} got {[out[tuple(i)].item() for i in bad]}, allowed "
                                 f"{[(c0[tuple(i)].item(), c1[tuple(i)].item()) for i in bad]}")
        amb = (c0 != c1).double().mean().item()
        assert amb <= 0.02, f"{what} gelu_tanh: {amb:.3%} of the elements have two candidates"
        return
    # GELU python form: five 16-bit roundings; erff within ERFF_ULP fp32 ulp (relative 2 ERFF_ULP u), doubled
    t1 = _r16(v * 0.5, dtype)
    t2 = _r16(v / torch.tensor(1.4142135623730951, dtype=torch.float32), dtype)
    e64 = torch.erf(t2.double())
    outs = []
    for s in (-1, 1):
        t3 = _r16((e64 * (1 + s * 2 * 2 * ERFF_ULP * U)).float(), dtype)
        t4 = _r16(1.0 + t3, dtype)
        outs.append(_r16(t1 * t4, dtype).double())
    lo, hi = torch.minimum(*outs), torch.maximum(*outs)
    _assert_between(out, lo, hi, what + " gelu_erf_py")


@pytest.mark.parametrize("M", [576, 1152])
@pytest.mark.parametrize("N", [3072, 1027])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF_PY])
def test_gemm_vit_epilogue_exact(lib, M, N, act):
    """gemm_vit_kernel: r16(acc + bias) then the activation; odd N ends on an unpaired column of the __half2 store;
    columns past N and rows past M keep their NaN sentinels"""
    gen = torch.Generator(device="cuda").manual_seed(M + N + act)
    K = 1024
    x, w, bias, acc = _gemm_operands(M, N, K, gen)
    ld = N + 5 if N % 2 else N + 8
    out = _nan16(M + 3, ld)
    _check(lib.vlo_op_gemm_vit(_p(w), N, _p(x), M, K, _p(out), ld, _p(bias), act, 0, _st()), "gemm_vit")
    torch.cuda.synchronize()
    _epilogue_check(lib, out[:M, :N], acc, bias, act, f"gemm_vit M={M} N={N}")
    assert _same_bits(out[:M, N:], _nan16(M, ld - N)) and _same_bits(out[M:], _nan16(3, ld)), "sentinel overwritten"


@pytest.mark.parametrize("fmt,bn", [(FMT_F16, 16), (FMT_F16, 32), (FMT_F16, 64), (FMT_F16, 96), (FMT_F16, 128),
                                    (FMT_F16, 192), (FMT_BF16, 32), (FMT_BF16, 64), (FMT_BF16, 96), (FMT_BF16, 128)])
@pytest.mark.parametrize("act", [ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF_PY])
def test_gemm_ws_store16_epilogue_exact(lib, fmt, bn, act):
    """gemm_ws mode 1 (whole tiles, 16-bit epilogue) at every fp16 and bf16 token tile: rows end part-way through the
    last token tile, N = 1000 is a multiple of neither 128 nor 16, ld_out > N with sentinels"""
    dtype = torch.float16 if fmt == FMT_F16 else torch.bfloat16
    gen = torch.Generator(device="cuda").manual_seed(bn * 7 + fmt + act)
    M, N, K = 3 * bn - 5, 1000, 512
    x, w, bias, acc = _gemm_operands(M, N, K, gen, dtype)
    ld = 1016
    out = _nan16(M + 2, ld, dtype=dtype)
    _check(lib.vlo_op_gemm_ws(fmt, 1, _p(w), N, _p(x), M, K, _p(out), ld, 0, _p(bias), act, 0, bn, None, _st()), "gemm_ws")
    torch.cuda.synchronize()
    _epilogue_check(lib, out[:M, :N], acc, bias, act, f"gemm_ws fmt={fmt} bn={bn}", dtype)
    assert _same_bits(out[:M, N:], _nan16(M, ld - N, dtype=dtype)) and _same_bits(out[M:], _nan16(2, ld, dtype=dtype))


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("epi,act", [(EPI_STORE16, ACT_NONE), (EPI_STORE16, ACT_GELU_TANH), (EPI_PATCH32, ACT_NONE)])
def test_gemm_tn_epilogue_exact(lib, bn, epi, act):
    """gemm_tn_kernel (patch embed, MAP-head K/V): STORE16 as above; PATCH32 = r16(acc + bias) + pos[row % pos_rows]
    in fp32, bit for bit.  1100 rows over a 576-row position table; N = 1000; ld_out > N with sentinels."""
    gen = torch.Generator(device="cuda").manual_seed(bn + epi * 10 + act)
    M, N, K, P, ld = 1100, 1000, 768, 576, 1016
    x, w, bias, acc = _gemm_operands(M, N, K, gen)
    pos = torch.randn(P, ld, device="cuda", generator=gen)
    out = _nan16(M + 2, ld) if epi == EPI_STORE16 else _nan32(M + 2, ld)
    _check(lib.vlo_op_gemm(epi, act, _p(x), M, _p(w), N, K, _p(out), ld, _p(bias), _p(pos), P, bn, _st()), "gemm")
    torch.cuda.synchronize()
    if epi == EPI_STORE16:
        _epilogue_check(lib, out[:M, :N], acc, bias, act, f"gemm_tn bn={bn}")
        assert _same_bits(out[:M, N:], _nan16(M, ld - N)) and _same_bits(out[M:], _nan16(2, ld))
    else:
        v = _r16(acc.float() + bias[None, :])
        rows = torch.arange(M, device="cuda") % P
        assert _same_bits(out[:M, :N], v + pos[rows, :N]), "PATCH32 != r16(acc + bias) + pos[row % pos_rows]"
        assert out[:M, N:].isnan().all() and out[M:].isnan().all(), "sentinel overwritten"


@pytest.mark.parametrize("kernel", ["ws_f16", "ws_bf16", "gemm_vit", "gemm_tn"])
def test_gemm_accumulation_bound(lib, kernel):
    """Random operands, whose sums are not exact: the fp32 accumulator against the fp64 product.  A product of two
    16-bit values is exact in fp32; each of the K additions errs by at most one fp32 ulp (2 u relative, which also
    covers an accumulator that truncates) of a running sum no larger than S = sum_k |x w|, so |acc - exact| <= 2 K u S;
    doubled, E = 4 K u S.  The stream-K kernels are read through fp32 planes (whole tiles per CTA: one plane), the
    16-bit kernels through r16(acc) in [r16(exact - E - 2 u |exact|), r16(exact + E + 2 u |exact|)].
    Self-check: the reference without any one 64-wide k-block leaves E on most elements, so the bound sees a lost block."""
    gen = torch.Generator(device="cuda").manual_seed(len(kernel))
    M, N, K = (128, 1024, 1024) if kernel.startswith("ws") else (576, 1027, 1024)
    dtype = torch.bfloat16 if kernel == "ws_bf16" else torch.float16
    x = torch.randn(M, K, device="cuda", generator=gen).to(dtype)
    w = (torch.randn(N, K, device="cuda", generator=gen) * 0.05).to(dtype)
    blocks = torch.einsum("mbk,nbk->bmn", x.double().view(M, K // 64, 64), w.double().view(N, K // 64, 64))
    exact = blocks.sum(0)
    E = 4 * K * U * (x.double().abs() @ w.double().abs().t())
    for j in range(K // 64):
        assert float(((blocks[j]).abs() > E).double().mean()) > 0.5, f"k-block {j} hides inside the bound"
    if kernel.startswith("ws"):
        fmt = FMT_BF16 if kernel == "ws_bf16" else FMT_F16
        part = _nan32(2, M, N)
        planes = C.c_int(0)
        _check(lib.vlo_op_gemm_ws(fmt, 0, _p(w), N, _p(x), M, K, _p(part), N, M * N, None, 0, (N + 127) // 128, 0,
                                  C.byref(planes), _st()), "gemm_ws")
        torch.cuda.synchronize()
        assert planes.value == 1 and part[1].isnan().all()
        err = (part[0].double() - exact).abs()
        assert bool((err <= E).all()), f"{kernel}: accumulator error {float((err / E).max()):.2f} x the derived bound"
        return
    ld = N + 5
    out = _nan16(M, ld)
    if kernel == "gemm_vit":
        _check(lib.vlo_op_gemm_vit(_p(w), N, _p(x), M, K, _p(out), ld, None, ACT_NONE, 0, _st()), "gemm_vit")
    else:
        _check(lib.vlo_op_gemm(EPI_STORE16, ACT_NONE, _p(x), M, _p(w), N, K, _p(out), ld, None, None, 0, 128, _st()), "gemm")
    torch.cuda.synchronize()
    Et = E + 2 * U * exact.abs()
    lo, hi = _either16(exact, Et)
    # E spans several fp16 steps at these sizes: the interval, not an exactness rule, is what is asserted here
    _assert_between(out[:, :N], lo, hi, kernel, max_ambiguous=1.0)


# ============================================================================================ LayerNorm
def _ln_eps(C, fix_ln=False):
    """Relative bound of the kernel's LayerNorm against fp64, for rows whose sum is exact in fp32 (dyadic rows, C a
    power of two: the mean is exact, and so is every x - mean).  A thread adds n_seq squares in sequence: ceil(C / 256)
    in layernorm_kernel (one channel per sweep), 4 ceil(C / 1024) in vit_fix_ln_kernel (4 channels per sweep); 5 warp
    shuffle levels and 8 warp partials follow: the sum of squares is within (n_seq + 14) u (each square rounded once).
    / C exact, + eps 1 u more, rsqrtf 2 ulp = 4 u, halved by the square root except rsqrtf's own; then
    (x - mean) rstd, * w and + b: 3 u of |(x - mean) rstd w| + |b|.  Doubled."""
    n_seq = 4 * math.ceil(C / 1024) if fix_ln else math.ceil(C / 256)
    return 2 * (0.5 * (n_seq + 16) + 4 + 3) * U


def _ln_check(x64, w, b, out16, out32, what, fix_ln=False):
    C = x64.shape[1]
    eps32 = float(torch.tensor(EPS, dtype=torch.float32))
    mean = x64.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x64 - mean) ** 2).mean(1, keepdim=True) + eps32)
    a = (x64 - mean) * rstd * w.double()[None, :]
    y = a + b.double()[None, :]
    E = _ln_eps(C, fix_ln) * (a.abs() + b.double().abs()[None, :])
    if out16 is not None:
        lo, hi = _either16(y, E)
        _assert_between(out16, lo, hi, what + " out16")
    if out32 is not None:
        err = (out32.double() - y).abs()
        assert bool((err <= E).all()), f"{what} out32: error {float((err / E).max()):.2f} x the derived bound"


def _ln_rows(rows, C, gen, offsets, lim=512, scale_log2=8):
    """dyadic rows k 2^-8 (|k| <= 512) around a per-row offset: rows with |mean| >> std make a one-pass variance
    (E[x^2] - mean^2) lose log2(mean^2 / var) bits"""
    off = torch.tensor(offsets, dtype=torch.float64, device="cuda").repeat(rows // len(offsets) + 1)[:rows, None]
    return _dyadic((rows, C), lim, scale_log2, gen) + off


@pytest.mark.parametrize("C", [128, 1024])
@pytest.mark.parametrize("in_f16", [0, 1])
def test_vit_layernorm(lib, C, in_f16):
    """both instances: fp32 input (the first layer_norm1) and fp16 input (the MAP head's layernorm); out16 under the
    exactness rule, out32 within the derived bound; rows of offsets 0, +-16 (fp32) or +-2 (fp16-exact values)"""
    gen = torch.Generator(device="cuda").manual_seed(C + in_f16)
    rows = 45
    x64 = _ln_rows(rows, C, gen, [0.0, 2.0, -2.0] if in_f16 else [0.0, 16.0, -16.0])
    x = x64.half() if in_f16 else x64.float()
    assert torch.equal(x.double(), x64)
    w = 1 + 0.1 * torch.randn(C, device="cuda", generator=gen)
    b = 0.02 * torch.randn(C, device="cuda", generator=gen)
    out16, out32 = _nan16(rows + 1, C), _nan32(rows + 1, C)
    _check(lib.vlo_op_vit_layernorm(_p(x), in_f16, rows, C, _p(w), _p(b), _p(out16), _p(out32), EPS, _st()), "layernorm")
    torch.cuda.synchronize()
    _ln_check(x64, w, b, out16[:rows], out32[:rows], f"layernorm C={C} f16={in_f16}")
    assert _same_bits(out16[rows:], _nan16(1, C)) and out32[rows:].isnan().all()


# ============================================================================================ vit_fix_ln
def _sk_planes(tiles, kb, G):
    """planes of each output tile for the stream-K split of tiles x kb units over G CTAs (CTA c owns units
    [c U / G, (c + 1) U / G); a tile's planes = the CTAs that touch it)"""
    U_ = tiles * kb
    G = min(G if G > 0 else _n_sm(), U_)
    owner = lambda u: ((u + 1) * G - 1) // U_
    return [owner((t + 1) * kb - 1) - owner(t * kb) + 1 for t in range(tiles)]


def _ctas_for_planes(tiles, kb, want):
    for G in range(1, tiles * kb + 1):
        if max(_sk_planes(tiles, kb, G)) == want:
            return G
    raise AssertionError(f"no split of {tiles} tiles x {kb} k-blocks has {want} planes")


def _plane_count_map(rows, C, bn, ns):
    """ns of the tile (feature / 128, token / bn) of every element [rows, C]: tile = w_tile x_tiles + x_tile"""
    x_tiles = (rows + bn - 1) // bn
    ns_t = torch.tensor(ns, device="cuda").view(-1, x_tiles)                    # [w_tiles, x_tiles]
    wt = torch.arange(C, device="cuda") // 128
    xt = torch.arange(rows, device="cuda") // bn
    return ns_t[wt[None, :], xt[:, None]]


def _fix_ln_case(lib, rows, C, k, bn, n_ctas, seed, part=None):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x_tiles = (rows + bn - 1) // bn
    ns = _sk_planes((C // 128) * x_tiles, k // 64, n_ctas)
    nsm = _plane_count_map(rows, C, bn, ns)
    if part is None:
        # dyadic planes: their sums stay dyadic, so h' keeps an exact fp32 row sum (the bound of _ln_eps applies)
        part = _dyadic((FIX_MAX_PLANES, rows, C), 256, 8, gen).float()
        live = torch.arange(FIX_MAX_PLANES, device="cuda")[:, None, None] < nsm[None]
        part = part.masked_fill(~live, float("nan"))
    bias = _dyadic((C,), 1024, 8, gen).float()
    h = _ln_rows(rows, C, gen, [0.0, 16.0, -16.0]).float()
    ln_w = 1 + 0.1 * torch.randn(C, device="cuda", generator=gen)
    ln_b = 0.02 * torch.randn(C, device="cuda", generator=gen)
    y = part[0].clone()
    for s in range(1, FIX_MAX_PLANES):
        y = torch.where(s < nsm, y + part[s], y)
    h_ref = h + _r16(y + bias[None, :])
    out16, out32 = _nan16(rows + 1, C), _nan32(rows + 1, C)
    _check(lib.vlo_op_vit_fix_ln(_p(part), rows, C, k, bn, n_ctas, _p(bias), _p(h), _p(ln_w), _p(ln_b), _p(out16),
                                 _p(out32), EPS, _st()), "vit_fix_ln")
    torch.cuda.synchronize()
    what = f"vit_fix_ln rows={rows} C={C} k={k} bn={bn} n_ctas={n_ctas} planes={max(ns)}"
    assert _same_bits(h, h_ref), what + ": h != h + fp16(sum of the tile's planes + bias)"
    _ln_check(h_ref.double(), ln_w, ln_b, out16[:rows], out32[:rows], what, fix_ln=True)
    assert _same_bits(out16[rows:], _nan16(1, C)) and out32[rows:].isnan().all(), what + ": row past rows written"
    return ns


# (rows, C, k): full width at the frame batches of the tiling table, and tiny rows ending part-way through a token tile
FIX_SHAPES = [(576, 1024, 1024), (576 * 3, 1024, 4096), (576 * 5, 1024, 1024), (576 * 11, 1024, 1024),
              (100, 128, 256), (250, 128, 256)]


@pytest.mark.parametrize("bn", [64, 96, 128, 192])
@pytest.mark.parametrize("shape", FIX_SHAPES)
@pytest.mark.parametrize("want", [1, 2, 3, 8])
def test_vit_fix_ln(lib, bn, shape, want):
    """h' = h + fp16(sum_{s < ns(tile)} planes + bias) bit for bit with tile = (feature / 128) x_tiles + row / bn, planes
    past each tile's ns NaN; out16 / out32 as LayerNorm; n_ctas chosen to give 1, 2, 3 and 8 planes"""
    rows, C, k = shape
    tiles = (C // 128) * ((rows + bn - 1) // bn)
    try:
        n_ctas = _ctas_for_planes(tiles, k // 64, want)
    except AssertionError:
        pytest.skip(f"no split of {tiles} tiles x {k // 64} k-blocks has exactly {want} planes")
    ns = _fix_ln_case(lib, rows, C, k, bn, n_ctas, rows + bn + want)
    assert max(ns) == want


@pytest.mark.parametrize("rows,bn,k,n_ctas", [(576, 64, 1024, 0), (576 * 3, 192, 4096, 0), (576 * 6, 192, 1024, 0),
                                              (576 * 5, 96, 1024, 0), (576 * 2, 128, 1024, 200), (250, 96, 4096, 37)])
def test_vit_fix_ln_fed_by_gemm_ws(lib, rows, bn, k, n_ctas):
    """planes written by the real producer (vlo_op_gemm_ws mode 0, fp16, same bn / k / n_ctas): the producer's tile
    w_tile x_tiles + x_tile and the fold's (feature / 128) x_tiles + row / bn must agree, so the planes the producer
    leaves unwritten (NaN) are never read"""
    Cw = 1024
    gen = torch.Generator(device="cuda").manual_seed(rows + k)
    # k 2^-4 with |k| <= 2: the planes are multiples of 2^-8 like the synthetic ones, so h' keeps an exact row sum
    w = _dyadic((Cw, k), 2, 4, gen).half()
    x = _dyadic((rows, k), 2, 4, gen).half()
    part = _nan32(FIX_MAX_PLANES, rows, Cw)
    mp = C.c_int(0)
    _check(lib.vlo_op_gemm_ws(FMT_F16, 0, _p(w), Cw, _p(x), rows, k, _p(part), Cw, rows * Cw, None, 0, n_ctas, bn,
                              C.byref(mp), _st()), "gemm_ws")
    ns = _fix_ln_case(lib, rows, Cw, k, bn, n_ctas, 5, part=part)
    assert mp.value == max(ns) <= FIX_MAX_PLANES


# ============================================================================================ pool, cls_residual
def _pool_ref(x, B, g, ph, pw):
    """fp32 in the kernel's order: y outer, x inner, sequential adds from 0, one division"""
    xv = x.view(B, g, g, -1)
    cells = []
    for i in range(ph):
        y0, y1 = (i * g) // ph, -(-((i + 1) * g) // ph)
        for j in range(pw):
            x0, x1 = (j * g) // pw, -(-((j + 1) * g) // pw)
            s = torch.zeros_like(xv[:, 0, 0])
            for yy in range(y0, y1):
                for xx in range(x0, x1):
                    s = s + xv[:, yy, xx]
            # a tensor divisor: torch divides by a Python scalar through its reciprocal, the kernel divides once
            cells.append(s / torch.full_like(s, float((y1 - y0) * (x1 - x0))))
    return torch.stack(cells, 1)


@pytest.mark.parametrize("g,ph,pw", [(24, 3, 3), (6, 3, 3), (24, 5, 5), (24, 7, 4), (24, 24, 24)])
@pytest.mark.parametrize("tok_off", [0, 1])
def test_vit_pool(lib, g, ph, pw, tok_off):
    """adaptive average pool bit for bit (24 -> 3x3 shipped, 6 -> 3x3 tiny, overlapping 24 -> 5x5 and 7x4, identity);
    the CLS slot, a spare slot per frame and the rows of frames past B keep their sentinels"""
    gen = torch.Generator(device="cuda").manual_seed(g * 100 + ph * 10 + pw)
    B, Cc = 3, 136
    x = torch.randn(B, g * g, Cc, device="cuda", generator=gen)
    n_tok = tok_off + ph * pw + 1
    tokens = _nan32(B + 1, n_tok, Cc)
    _check(lib.vlo_op_vit_pool(_p(x), B, g, Cc, ph, pw, n_tok, tok_off, _p(tokens), _st()), "vit_pool")
    torch.cuda.synchronize()
    assert _same_bits(tokens[:B, tok_off:tok_off + ph * pw], _pool_ref(x, B, g, ph, pw))
    assert tokens[:B, :tok_off].isnan().all() and tokens[:B, tok_off + ph * pw:].isnan().all() and tokens[B:].isnan().all()


def test_cls_residual(lib):
    """tokens[b n_tok] = fp16(resid + mlp) bit for bit; every other token slot keeps its sentinel"""
    gen = torch.Generator(device="cuda").manual_seed(3)
    B, Cc, n_tok = 5, 1024, 12
    resid = torch.randn(B, Cc, device="cuda", generator=gen).half()
    mlp = (torch.randn(B, Cc, device="cuda", generator=gen) * 3).half()
    tokens = _nan32(B + 1, n_tok, Cc)
    _check(lib.vlo_op_cls_residual(_p(resid), _p(mlp), _p(tokens), B, Cc, n_tok, _st()), "cls_residual")
    torch.cuda.synchronize()
    assert _same_bits(tokens[:B, 0], _r16(resid.float() + mlp.float()))
    assert tokens[:B, 1:].isnan().all() and tokens[B:].isnan().all()


def test_vit_entries_reject_bad_arguments(lib):
    """bad sizes and null pointers fail before any launch"""
    from videollm_online_b200._lib import VloError
    f = torch.zeros(FIX_MAX_PLANES, 64, 1024, device="cuda")
    h16 = torch.zeros(64, 1024, device="cuda").half()
    u8 = torch.zeros(1, 3, 32, 32, device="cuda", dtype=torch.uint8)
    cases = [
        lambda: lib.vlo_op_patchify(None, 1, 32, 16, _p(h16), _st()),
        lambda: lib.vlo_op_patchify(_p(u8), 1, 32, 12, _p(h16), _st()),       # ps not a multiple of 8
        lambda: lib.vlo_op_patchify(_p(u8), 1, 40, 16, _p(h16), _st()),       # S not a multiple of ps
        lambda: lib.vlo_op_patchify(_p(u8), 0, 32, 16, _p(h16), _st()),
        lambda: lib.vlo_op_vit_layernorm(_p(f), 0, 64, 1024, None, _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_layernorm(_p(f), 0, 64, 1024, _p(f), _p(f), None, None, EPS, _st()),
        lambda: lib.vlo_op_vit_layernorm(_p(f), 0, 0, 1024, _p(f), _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_layernorm(_p(f), 0, 1, 12289, _p(f), _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_fix_ln(_p(f), 64, 1022, 1024, 64, 0, _p(f), _p(f), _p(f), _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_fix_ln(_p(f), 1, 12292, 1024, 64, 0, _p(f), _p(f), _p(f), _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_fix_ln(_p(f), 64, 1024, 1024, 64, _ctas_for_planes(8, 16, 9), _p(f), _p(f), _p(f), _p(f),
                                      _p(h16), None, EPS, _st()),                     # 9 planes
        lambda: lib.vlo_op_vit_fix_ln(_p(f), 64, 1024, 1000, 64, 0, _p(f), _p(f), _p(f), _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_fix_ln(_p(f), 64, 1024, 1024, 0, 0, _p(f), _p(f), _p(f), _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_fix_ln(None, 64, 1024, 1024, 64, 0, _p(f), _p(f), _p(f), _p(f), _p(h16), None, EPS, _st()),
        lambda: lib.vlo_op_vit_fix_ln(_p(f[0, 0, 1:]), 64, 1024, 1024, 64, 0, _p(f), _p(f), _p(f), _p(f), _p(h16), None, EPS,
                                      _st()),                                          # part not 16-byte aligned
        lambda: lib.vlo_op_vit_fix_ln(_p(f), 64, 1024, 1024, 64, 0, _p(f), _p(f), _p(f), _p(f), _p(h16[0, 2:]), None, EPS,
                                      _st()),                                          # out16 not 8-byte aligned
        lambda: lib.vlo_op_tanh_approx(None, _p(f), 4, _st()),
        lambda: lib.vlo_op_vit_pool(_p(f), 1, 24, 8, 25, 3, 100, 0, _p(f), _st()),     # ph > grid
        lambda: lib.vlo_op_vit_pool(_p(f), 1, 24, 8, 3, 3, 9, 1, _p(f), _st()),        # cells past n_tok
        lambda: lib.vlo_op_vit_pool(_p(f), 1, 24, 8, 3, 3, 10, -1, _p(f), _st()),
        lambda: lib.vlo_op_vit_pool(None, 1, 24, 8, 3, 3, 10, 1, _p(f), _st()),
        lambda: lib.vlo_op_cls_residual(_p(h16), None, _p(f), 1, 8, 10, _st()),
        lambda: lib.vlo_op_cls_residual(_p(h16), _p(h16), _p(f), 0, 8, 10, _st()),
        lambda: lib.vlo_op_vit_tiling(0, 576, 1024, 4096, (C.c_int32 * 11)()),
        lambda: lib.vlo_op_vit_tiling(1, 576, 1024, 4096, None),
        lambda: lib.vlo_op_gemm_ws_tiled(0, 1, _p(h16), 64, _p(h16), 64, 1024, _p(h16), 64, 0, None, 0, 0, 0, 7, None, _st()),
    ]
    n0 = lib.vlo_launch_count()
    for i, call in enumerate(cases):
        with pytest.raises(VloError):
            _check(call(), f"case {i}")
    assert lib.vlo_launch_count() == n0, "a rejected call launched a kernel"


# ============================================================================================ the tower, replayed
TOWER_BATCHES = [1, 2, 3, 4, 5, 6, 7, 8, 11]
MAX_VIT_BATCH = 11


def _tower_config():
    from videollm_online_b200 import llama3_8b_siglip_l
    cfg = llama3_8b_siglip_l()
    cfg.num_hidden_layers, cfg.vocab_size, cfg.intermediate_size = 1, 1024, 1024     # the decoder is not under test
    cfg.vision_num_hidden_layers = 2            # the ln1-of-the-next-layer fold and the post_layernorm fold both run
    cfg.frame_token_pooled, cfg.frame_num_tokens = [24, 24], 577        # identity pool: every patch token is an output
    return cfg


def _tower_engine(cfg):
    from videollm_online_b200 import weights as W
    from videollm_online_b200.modeling_live import build_live
    llm = W.synthetic_llm_state(cfg, seed=2)
    vis = W.synthetic_vision_state(cfg, seed=1)
    model, _ = build_live(config=cfg, llm_state=llm, vision_state=vis, set_vision_inside=True, device="cuda:0",
                          max_streams=1, max_kv_tokens=256, max_step_tokens=32, max_vit_batch=MAX_VIT_BATCH)
    return model.engine


@pytest.fixture(scope="module")
def tower():
    cfg = _tower_config()
    return cfg, _tower_engine(cfg)


def _tiling(lib, B, cfg):
    t = (C.c_int32 * 11)()
    _check(lib.vlo_op_vit_tiling(B, cfg.num_patches, cfg.vision_hidden_size, cfg.vision_intermediate_size, t), "vit_tiling")
    return list(t)


def _tiling_combos(t):
    """the (GEMM, kernel, token tile, planes) combinations one frame batch runs"""
    return {("qkv", t[0], t[1]), ("fc1", t[0], t[2]), ("out_proj", t[3], t[4], t[5]), ("fc2", t[3], t[6], t[7]),
            ("patch", t[8]), ("head_kv", t[9]), ("head", t[10])}


def _replay(lib, eng, cfg, frames, t):
    """vlo_vit_encode chained from the kernel-level entry points in the engine's order, with the queried tiling"""
    Wt = eng.weights
    B = frames.shape[0]
    Cc, M, P, ps = cfg.vision_hidden_size, cfg.vision_intermediate_size, cfg.num_patches, cfg.vision_patch_size
    rows, K0, S, eps, st = B * P, 3 * ps * ps, cfg.frame_resolution, cfg.vision_layer_norm_eps, _st()
    f16 = dict(dtype=torch.float16, device="cuda")
    patches = torch.empty(rows, K0, **f16)
    _check(lib.vlo_op_patchify(_p(frames), B, S, ps, _p(patches), st), "patchify")
    h = torch.empty(rows, Cc, device="cuda")
    _check(lib.vlo_op_gemm(EPI_PATCH32, 0, _p(patches), rows, _p(Wt["vit.patch.w"]), Cc, K0, _p(h), Cc,
                           _p(Wt["vit.patch.b"]), _p(Wt["vit.pos"]), P, t[8], st), "patch embed")
    xn = torch.empty(rows, Cc, **f16)
    _check(lib.vlo_op_vit_layernorm(_p(h), 0, rows, Cc, _p(Wt["vit.L0.ln1.w"]), _p(Wt["vit.L0.ln1.b"]), _p(xn), None, eps, st),
           "ln1")

    def tiles(x, w, b, n_out, k, bn, act):
        out = torch.empty(rows, n_out, **f16)
        if t[0] == 0:
            _check(lib.vlo_op_gemm_vit(_p(w), n_out, _p(x), rows, k, _p(out), n_out, _p(b), act, 0, st), "gemm_vit")
        else:
            plan = (C.c_int32 * 3)()
            _check(lib.vlo_op_gemm_ws_tiled(FMT_F16, 1, _p(w), n_out, _p(x), rows, k, _p(out), n_out, 0, _p(b), act, 0, 0,
                                            t[0], plan, st), "gemm_ws tiles")
            assert plan[0] == bn
        return out

    def partial_fix(x, w, k, bn, planes, bias, lw, lb, out32):
        part = torch.empty(planes, rows, Cc, device="cuda")
        plan = (C.c_int32 * 3)()
        _check(lib.vlo_op_gemm_ws_tiled(FMT_F16, 0, _p(w), Cc, _p(x), rows, k, _p(part), Cc, rows * Cc, None, 0, 0, 0, t[3],
                                        plan, st), "gemm_ws partial")
        assert (plan[0], plan[2]) == (bn, planes)
        _check(lib.vlo_op_vit_fix_ln(_p(part), rows, Cc, k, bn, 0, _p(bias), _p(h), _p(lw), _p(lb), _p(xn), _p(out32), eps,
                                     st), "vit_fix_ln")

    L = cfg.vision_num_hidden_layers
    ln32 = torch.empty(rows, Cc, device="cuda")
    for l in range(L):
        q = f"vit.L{l}."
        qkv = tiles(xn, Wt[q + "qkv.w"], Wt[q + "qkv.b"], 3 * Cc, Cc, t[1], ACT_NONE)
        attn = torch.empty(rows, Cc, **f16)
        _check(lib.vlo_op_vit_attn(_p(qkv), _p(attn), B, P, Cc, st), "vit_attn")
        partial_fix(attn, Wt[q + "out.w"], Cc, t[4], t[5], Wt[q + "out.b"], Wt[q + "ln2.w"], Wt[q + "ln2.b"], None)
        mlp = tiles(xn, Wt[q + "fc1.w"], Wt[q + "fc1.b"], M, Cc, t[2], ACT_GELU_TANH)
        last = l == L - 1
        nq = "vit.post_ln." if last else f"vit.L{l + 1}.ln1."
        partial_fix(mlp, Wt[q + "fc2.w"], M, t[6], t[7], Wt[q + "fc2.b"], Wt[nq + "w"], Wt[nq + "b"], ln32 if last else None)
    NT = cfg.frame_num_tokens
    g = S // ps
    tokens = _nan32(B, NT, Cc)
    _check(lib.vlo_op_vit_pool(_p(ln32), B, g, Cc, g, g, NT, 1, _p(tokens), st), "pool")
    kv = torch.empty(rows, 2 * Cc, **f16)
    _check(lib.vlo_op_gemm(EPI_STORE16, 0, _p(xn), rows, _p(Wt["vit.head.kv.w"]), 2 * Cc, Cc, _p(kv), 2 * Cc,
                           _p(Wt["vit.head.kv.b"]), None, 0, t[9], st), "head kv")
    pa = torch.empty(B, Cc, **f16)
    _check(lib.vlo_op_probe_attn(_p(kv), _p(Wt["vit.head.q"]), _p(pa), B, P, Cc, st), "probe_attn")

    def head_gemm(x, w, b, n_out, k, act):
        out = torch.empty(B, n_out, **f16)
        plan = (C.c_int32 * 3)()
        _check(lib.vlo_op_gemm_ws_tiled(FMT_F16, 1, _p(w), n_out, _p(x), B, k, _p(out), n_out, 0, _p(b), act, 0, 0, 0, plan,
                                        st), "head gemm")
        assert plan[0] == t[10]
        return out

    resid = head_gemm(pa, Wt["vit.head.out.w"], Wt["vit.head.out.b"], Cc, Cc, ACT_NONE)
    lnh = torch.empty(B, Cc, **f16)
    _check(lib.vlo_op_vit_layernorm(_p(resid), 1, B, Cc, _p(Wt["vit.head.ln.w"]), _p(Wt["vit.head.ln.b"]), _p(lnh), None,
                                    eps, st), "head ln")
    m1 = head_gemm(lnh, Wt["vit.head.fc1.w"], Wt["vit.head.fc1.b"], M, Cc, ACT_GELU_TANH)
    m2 = head_gemm(m1, Wt["vit.head.fc2.w"], Wt["vit.head.fc2.b"], Cc, M, ACT_NONE)
    _check(lib.vlo_op_cls_residual(_p(resid), _p(m2), _p(tokens), B, Cc, NT, st), "cls_residual")
    torch.cuda.synchronize()
    return tokens


def _frames(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (B, 3, S, S), dtype=torch.uint8, generator=g).cuda()


def test_tower_batches_cover_every_tiling(lib, tower):
    """the replayed frame batches reach every (GEMM, kernel, token tile, planes) combination the engine runs up to
    max_vit_batch, so the replay's coverage is checked, not assumed"""
    cfg, _ = tower
    every = set().union(*(_tiling_combos(_tiling(lib, B, cfg)) for B in range(1, MAX_VIT_BATCH + 1)))
    tested = set().union(*(_tiling_combos(_tiling(lib, B, cfg)) for B in TOWER_BATCHES))
    assert every == tested, f"untested tilings: {sorted(map(str, every - tested))}"


@pytest.mark.parametrize("B", TOWER_BATCHES)
def test_tower_replay_bit_exact(lib, tower, B):
    """every fp32 token of vlo_vit_encode (577 per frame: CLS + the identity-pooled post-LN patch tokens) equals the
    kernel-level chain bit for bit, and its bf16 embeds equal the connector of bf16(tokens) bit for bit"""
    cfg, eng = tower
    frames = _frames(B, cfg.frame_resolution, B)
    emb, tok = eng.vit_encode(frames, return_vit_tokens=True)
    ref = _replay(lib, eng, cfg, frames, _tiling(lib, B, cfg))
    assert not ref.isnan().any(), "the replay left a token slot unwritten"
    if not _same_bits(tok, ref):
        frames_off = (tok != ref).flatten(1).any(1).nonzero().flatten().tolist()
        _, tok2 = eng.vit_encode(frames, return_vit_tokens=True)
        ref2 = _replay(lib, eng, cfg, frames, _tiling(lib, B, cfg))
        raise AssertionError(f"B={B}: {int((tok != ref).sum())} tokens of frames {frames_off} differ from the replay; "
                             f"encode repeats its bits: {_same_bits(tok, tok2)}, replay repeats: {_same_bits(ref, ref2)}")
    assert _same_bits(emb, eng.connector(ref.bfloat16()))


@pytest.mark.parametrize("B", TOWER_BATCHES[1:])
def test_tower_frame_isolation(tower, B):
    """a frame's 577 tokens and embeds do not depend on the other frames of its batch (token tiles straddle frames
    at odd B)"""
    cfg, eng = tower
    S, NT, j = cfg.frame_resolution, cfg.frame_num_tokens, B // 2
    a = _frames(B, S, 100 + B)
    b = _frames(B, S, 200 + B)
    b[j] = a[j]
    ea, ta = eng.vit_encode(a, return_vit_tokens=True)
    ea, ta = ea.clone(), ta.clone()
    eb, tb = eng.vit_encode(b, return_vit_tokens=True)
    assert _same_bits(ta[j], tb[j]) and _same_bits(ea[j * NT:(j + 1) * NT], eb[j * NT:(j + 1) * NT])


def test_tower_no_stale_state(tower):
    """B = max_vit_batch unrelated frames first, then B = b: the same bits as B = b on a fresh engine"""
    cfg, eng = tower
    S = cfg.frame_resolution
    fresh = _tower_engine(cfg)
    try:
        for b in (1, 3, 5):
            frames = _frames(b, S, 300 + b)
            e0, t0 = fresh.vit_encode(frames, return_vit_tokens=True)
            e0, t0 = e0.clone(), t0.clone()
            fresh.vit_encode(_frames(MAX_VIT_BATCH, S, 400 + b))
            eng.vit_encode(_frames(MAX_VIT_BATCH, S, 500 + b))
            e1, t1 = eng.vit_encode(frames, return_vit_tokens=True)
            assert _same_bits(t0, t1) and _same_bits(e0, e1), f"b={b}"
    finally:
        fresh.close()
