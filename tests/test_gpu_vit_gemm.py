"""GPU parity of the ViT trunk GEMM (vlo_op_gemm_vit, 128-token x 128-feature tiles) at the QKV and fc1 shapes of
one and two frames (576 rows end in a half-full token tile): against an fp32 matmul, and bit for bit against the
64-token swap-AB tiles of the persistent GEMM that ran these layers before it."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(3072, 1024), (4096, 1024), (1024, 1024), (1024, 4096)]  # (N, K): QKV, fc1, and the out_proj / fc2 sizes


@pytest.fixture(scope="module")
def lib():
    from videollm_online_b200 import _lib
    return _lib.load()


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _run(lib, M, N, K, act, ld=None):
    from videollm_online_b200._lib import check
    torch.manual_seed(M + N + K + act)
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") * 0.05).half()
    bias = torch.randn(N, device="cuda")
    ld = ld or N
    out = torch.full((M + 8, ld), 7.0, device="cuda", dtype=torch.float16)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.vlo_op_gemm_vit(_ptr(w), N, _ptr(x), M, K, _ptr(out), ld, _ptr(bias), act, 0, st), "gemm_vit")
    torch.cuda.synchronize()
    return x, w, bias, out


@pytest.mark.parametrize("M", [576, 1152])
@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("act", [0, 1])
def test_gemm_vit_matches_fp32_matmul(lib, M, N, K, act):
    """bias, fp16 rounding, GELU-tanh (act 1), fp16 rounding; rows past M and columns past N untouched"""
    x, w, bias, out = _run(lib, M, N, K, act, ld=N + 8)
    ref = (x.float() @ w.float().t() + bias).half().float()
    if act == 1:
        ref = torch.nn.functional.gelu(ref, approximate="tanh").half().float()
    assert (out[:M, :N].float() - ref).abs().max() <= 1e-2 * ref.abs().max()
    assert (out[M:] == 7.0).all() and (out[:, N:] == 7.0).all()


@pytest.mark.parametrize("M", [576, 1152])
@pytest.mark.parametrize("N,K", SHAPES)
def test_gemm_vit_bits_equal_swap_ab_kernel(lib, M, N, K):
    """tokens on MMA-M accumulate every output over all of K in the same k order as the swap-AB kernel with 64-token
    tiles, so a frame's embeddings do not depend on which of the two ran QKV / fc1"""
    from videollm_online_b200._lib import check
    x, w, bias, out = _run(lib, M, N, K, 1)
    ref = torch.zeros(M, N, device="cuda", dtype=torch.float16)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.vlo_op_gemm_ws(0, 1, _ptr(w), N, _ptr(x), M, K, _ptr(ref), N, 0, _ptr(bias), 1, 0, 64, None, st), "gemm_ws")
    torch.cuda.synchronize()
    assert torch.equal(out[:M], ref)
