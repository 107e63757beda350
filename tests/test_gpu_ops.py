"""GPU parity of the kernel-level C-ABI entry points against plain torch fp32 references."""
import ctypes as C
import math

import pytest
import torch

from attn_reference import DECODER, decoder_chain, reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _gemm(lib, epi, act, x, w, out, ld, bias=None, pos=None, pos_rows=0, bn=0):
    from videollm_online_b200._lib import check
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    check(lib.vlo_op_gemm(epi, act, p(x), x.shape[0], p(w), w.shape[0], x.shape[1], p(out), ld, p(bias), p(pos), pos_rows, bn,
                          C.c_void_p(torch.cuda.current_stream().cuda_stream)), "gemm")
    torch.cuda.synchronize()


@pytest.mark.parametrize("M,N,K,bn", [(576, 1024, 1024, 128), (300, 200, 768, 64), (1152, 4096, 1024, 128)])
def test_gemm_tn_epilogues(lib, M, N, K, bn):
    """one-tile fp16 GEMM of the ViT patch embed / MAP-head K/V projection: bias + GELU-tanh fp16 store, and the fp32
    patch-embed store with the position embedding added"""
    torch.manual_seed(M)
    a = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    bias = torch.randn(N, device="cuda")
    ld = (N + 7) // 8 * 8
    lin = (a.float() @ w.float().t() + bias).half().float()
    out = torch.zeros(M, ld, device="cuda", dtype=torch.float16)
    _gemm(lib, 1, 1, a, w, out, ld, bias=bias, bn=bn)
    ref = torch.nn.functional.gelu(lin, approximate="tanh")
    assert (out[:, :N].float() - ref).abs().max() <= 1e-2 * ref.abs().max()
    pos = torch.randn(36, ld, device="cuda")
    o32 = torch.zeros(M, ld, device="cuda")
    _gemm(lib, 3, 0, a, w, o32, ld, bias=bias, pos=pos, pos_rows=36, bn=bn)
    ref = lin + pos[torch.arange(M, device="cuda") % 36][:, :N]
    assert (o32[:, :N] - ref).abs().max() <= 1e-2 * ref.abs().max()


@pytest.mark.parametrize("n_tok,H,Hk,kv_len,stride", [
    (1, 32, 8, 1, 64), (11, 32, 8, 28, 64), (11, 32, 8, 1000, 1024), (1, 32, 8, 777, 1024), (40, 32, 8, 40, 128),
    (37, 8, 4, 300, 320), (3, 4, 2, 130, 192), (11, 32, 8, 13211, 13312), (17, 32, 8, 5000, 5056)])
def test_attn_kvappend_vs_torch(lib, n_tok, H, Hk, kv_len, stride):
    """empty-ish (kv=1), ragged, multi-chunk (q>16) and BASELINE-size (13.2k) contexts, within the fp64 bound of
    attn_reference.py"""
    from videollm_online_b200._lib import check
    torch.manual_seed(kv_len)
    D = 128
    q = torch.randn(n_tok, H, D, device="cuda").bfloat16()
    k = torch.randn(Hk, stride, D, device="cuda").bfloat16()
    v = torch.randn(Hk, stride, D, device="cuda").bfloat16()
    ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, H, D, kv_len), device="cuda", dtype=torch.uint8)
    out = torch.empty(n_tok, H * D, device="cuda", dtype=torch.bfloat16)
    p = lambda t: C.c_void_p(t.data_ptr())
    check(lib.vlo_op_attn_kvappend(p(q), p(k), p(v), p(out), p(ws), n_tok, H, Hk, D, kv_len, stride,
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)), "attn")
    torch.cuda.synchronize()
    res = reference(q, k[:, :kv_len], v[:, :kv_len], torch.arange(kv_len - n_tok, kv_len), DECODER,
                    decoder_chain(kv_len, torch.cuda.get_device_properties(0).multi_processor_count))
    assert torch.isfinite(out.float()).all()
    assert res.excess(out.view(n_tok, H, D)) <= 0


def test_attention_is_a_convex_combination_at_full_size(lib):
    """size-independent property at BASELINE size: with V == const the output is that constant;
    with one huge key the output equals that key's value row."""
    from videollm_online_b200._lib import check
    n_tok, H, Hk, D, kv_len = 11, 32, 8, 128, 13211
    stride = 13248
    torch.manual_seed(1)
    q = torch.randn(n_tok, H, D, device="cuda").bfloat16()
    k = torch.randn(Hk, stride, D, device="cuda").bfloat16()
    v = torch.full((Hk, stride, D), 0.5, device="cuda").bfloat16()
    ws = torch.empty(lib.vlo_op_attn_ws_bytes(n_tok, H, D, kv_len), device="cuda", dtype=torch.uint8)
    out = torch.empty(n_tok, H * D, device="cuda", dtype=torch.bfloat16)
    p = lambda t: C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.vlo_op_attn_kvappend(p(q), p(k), p(v), p(out), p(ws), n_tok, H, Hk, D, kv_len, stride, st), "attn")
    torch.cuda.synchronize()
    assert (out.float() - 0.5).abs().max() < 4e-3


def _py_sk_planes(rows_w, k, G):
    tiles, kb = (rows_w + 127) // 128, k // 64
    U = tiles * kb
    lo = lambda c: (c * U) // G
    def owner(u):
        c = min((u * G) // U, G - 1)
        while lo(c + 1) <= u:
            c += 1
        while c > 0 and lo(c) > u:
            c -= 1
        return c
    return [owner((t + 1) * kb - 1) - owner(t * kb) + 1 for t in range(tiles)]


@pytest.mark.parametrize("T,N,K,G", [(11, 6144, 4096, 0), (11, 4096, 14336, 0), (11, 28672, 4096, 0), (1, 512, 256, 0),
                                     (33, 1000, 1024, 7), (128, 640, 4096, 148), (11, 256, 128, 148), (88, 4096, 4096, 0), (90, 1024, 512, 37),
                                     (11, 512, 1024, 4), (11, 4096, 14336, 7), (40, 640, 4096, 3)])
def test_gemm_ws_streamk_partials(lib, T, N, K, G):
    """persistent stream-K weight-streaming GEMM: planes sum to X W^T; decomposition covers every unit once"""
    from videollm_online_b200._lib import check
    torch.manual_seed(N + T)
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    x = torch.randn(T, K, device="cuda").bfloat16()
    planes = C.c_int(0)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.vlo_op_gemm_ws(1, 0, p(w), N, p(x), T, K, None, N, T * N, None, 0, G, 0, C.byref(planes), st), "plan")
    ws = torch.zeros(planes.value, T, N, device="cuda")
    check(lib.vlo_op_gemm_ws(1, 0, p(w), N, p(x), T, K, p(ws), N, T * N, None, 0, G, 0, C.byref(planes), st), "gemm_ws")
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t()
    assert (ws.sum(0) - ref).abs().max() <= 2e-3 * ref.abs().max()
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    Gs = min(G if G > 0 else n_sm, ((N + 127) // 128) * (K // 64))
    assert max(_py_sk_planes(N, K, Gs)) == planes.value


@pytest.mark.parametrize("T,N,K,act", [(8, 128256, 4096, 0), (40, 4096, 1024, 2), (128, 1000, 512, 0), (3, 256, 64, 1),
                                       (1, 128, 64, 0), (11, 256, 128, 0), (33, 1000, 1024, 0), (88, 4096, 4096, 0), (130, 512, 256, 0),
                                       (20, 512, 256, 2)])
def test_gemm_ws_tiles_store16(lib, T, N, K, act):
    """whole-tile bf16 epilogue: bias, then GELU (erf, python form: act 2; tanh: act 1)"""
    from videollm_online_b200._lib import check
    torch.manual_seed(T)
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    x = torch.randn(T, K, device="cuda").bfloat16()
    bias = torch.randn(N, device="cuda")
    out = torch.zeros(T, N, device="cuda", dtype=torch.bfloat16)
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    bn = 128 if T > 128 else 0  # more than 128 rows: two 128-token tiles
    check(lib.vlo_op_gemm_ws(1, 1, p(w), N, p(x), T, K, p(out), N, 0, p(bias), act, 0, bn, None, st), "gemm_ws")
    torch.cuda.synchronize()
    y = (x.float() @ w.float().t() + bias).bfloat16()
    if act == 2:
        y = y * 0.5 * (1.0 + torch.erf(y / math.sqrt(2.0)))
    elif act == 1:
        y = torch.nn.functional.gelu(y.float(), approximate="tanh").bfloat16()
    assert (out.float() - y.float()).abs().max() <= 1e-2 * y.float().abs().max()


@pytest.mark.parametrize("M,N,K,bn,mode", [(576, 3072, 1024, 96, 1), (576, 4096, 1024, 64, 1), (576, 1024, 4096, 192, 0),
                                           (576, 1024, 1024, 192, 0), (1152, 4096, 1024, 192, 1), (300, 200, 256, 128, 1),
                                           (36, 384, 128, 64, 0)])
def test_gemm_ws_vit_shapes_fp16(lib, M, N, K, bn, mode):
    """ViT trunk on the persistent kernel: token rows tiled along MMA-N (bn = 64/96/128/192), fp16"""
    from videollm_online_b200._lib import check
    torch.manual_seed(M + N)
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    x = torch.randn(M, K, device="cuda").half()
    bias = torch.randn(N, device="cuda")
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    lin = x.float() @ w.float().t()
    if mode == 1:
        out = torch.zeros(M, N, device="cuda", dtype=torch.float16)
        check(lib.vlo_op_gemm_ws(0, 1, p(w), N, p(x), M, K, p(out), N, 0, p(bias), 1, 0, bn, None, st), "gemm_ws")
        torch.cuda.synchronize()
        ref = torch.nn.functional.gelu((lin + bias).half().float(), approximate="tanh")
        assert (out.float() - ref).abs().max() <= 1e-2 * ref.abs().max()
    else:
        planes = C.c_int(0)
        check(lib.vlo_op_gemm_ws(0, 0, p(w), N, p(x), M, K, None, N, M * N, None, 0, 0, bn, C.byref(planes), st), "plan")
        ws = torch.zeros(planes.value, M, N, device="cuda")
        check(lib.vlo_op_gemm_ws(0, 0, p(w), N, p(x), M, K, p(ws), N, M * N, None, 0, 0, bn, C.byref(planes), st), "gemm_ws")
        torch.cuda.synchronize()
        assert (ws.sum(0) - lin).abs().max() <= 2e-3 * lin.abs().max()
