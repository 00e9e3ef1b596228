"""The bf16 variant of the TMA + tensor-core GEMM building block (bf16 operands, fp32 accumulation; BASELINE config 3's
arithmetic) against a plain PyTorch reference of the same op.  bf16 x bf16 products are exact in fp32, so with fp32
outputs only the summation order differs (tolerance 1e-5 of sum |a||b|); bf16 outputs add one rounding (2^-8 relative)."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_BIAS, EPI_RELU, EPI_ADD_AUX, EPI_MASK_AUX, EPI_ATOMIC, EPI_DROPOUT, EPI_COLSUM = 1, 2, 4, 8, 16, 32, 64


@pytest.fixture(scope="module")
def gemm():
    from allrank_b200 import _lib
    c_p, c_i, c_f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float
    _lib.register("arb_gemm_bf16", c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_f, c_i, c_i, c_p, c_p])

    def call(A, B, C, aux, bias, M, N, K, a_mn, b_mn, block_n, flags, alpha=1.0, split_k=1, colsum=None):
        rc = _lib.lib().arb_gemm_bf16(_lib.ptr(A), _lib.ptr(B), _lib.ptr(C), _lib.ptr(aux), _lib.ptr(bias), M, N, K,
                                      a_mn, b_mn, block_n, flags, alpha, split_k, 1 if C.dtype == torch.bfloat16 else 0,
                                      _lib.ptr(colsum), _lib.stream_ptr())
        _lib.check(rc, "arb_gemm_bf16")
        torch.cuda.synchronize()
    return call


def operands(M, N, K, a_mn, b_mn, seed):
    torch.manual_seed(seed)
    A = torch.randn(M, K, device="cuda").bfloat16()
    B = torch.randn(N, K, device="cuda").bfloat16()
    return A, B, (A.t().contiguous() if a_mn else A), (B.t().contiguous() if b_mn else B)


@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (240, 96, 136), (304, 200, 40), (64, 64, 512), (256, 1024, 256)])   # bf16 rows need 16-byte pitches: multiples of 8
@pytest.mark.parametrize("out16", [False, True])
def test_bf16_gemm_all_majors(gemm, block_n, a_mn, b_mn, M, N, K, out16):
    A, B, As, Bs = operands(M, N, K, a_mn, b_mn, M * 7 + N * 3 + K + a_mn * 2 + b_mn)
    C = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16 if out16 else torch.float32)
    gemm(As, Bs, C, None, None, M, N, K, a_mn, b_mn, block_n, 0)
    ref = A.double() @ B.double().t()
    bound = (1e-5 + (2.0 ** -8 if out16 else 0.0)) * (A.double().abs() @ B.double().abs().t()) + 1e-6
    assert torch.isfinite(C).all()
    assert ((C.double() - ref).abs() <= bound).all(), float(((C.double() - ref).abs() / bound).max())


@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("M,N,K", [(128, 128, 4096), (256, 136, 983), (512, 256, 2048), (96, 72, 640)])
def test_bf16_weight_gradient_split_k(gemm, block_n, M, N, K):
    """dW[M,N] += dY[K,M]^T X[K,N]: both operands MN-major, split-K with fp32 red.add (K must keep 16-byte rows)."""
    K = K // 8 * 8
    A, B, As, Bs = operands(M, N, K, 1, 1, 5 + M + K)
    C = torch.randn(M, N, device="cuda")
    start = C.clone()
    gemm(As, Bs, C, None, None, M, N, K, 1, 1, block_n, EPI_ATOMIC, split_k=7)
    ref = start.double() + A.double() @ B.double().t()
    bound = 1e-5 * (A.double().abs() @ B.double().abs().t()) + 1e-5
    assert ((C.double() - ref).abs() <= bound).all(), float(((C.double() - ref).abs() / bound).max())


def test_bf16_epilogues(gemm):
    M, N, K = 384, 256, 128
    A, B, As, Bs = operands(M, N, K, 0, 0, 11)
    bias = torch.randn(N, device="cuda")
    base = A.double() @ B.double().t()
    # bias + ReLU into a bf16 output (first FFN linear)
    C = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    gemm(A, B, C, None, bias, M, N, K, 0, 0, 128, EPI_BIAS | EPI_RELU)
    want = torch.relu(base + bias.double())
    assert ((C.double() - want).abs() <= 2.0 ** -8 * want.abs() + 1e-3).all()
    # bias + fp32 residual into an fp32 output (second FFN linear / attention output projection)
    res = torch.randn(M, N, device="cuda")
    C32 = torch.empty(M, N, device="cuda")
    gemm(A, B, C32, res, bias, M, N, K, 0, 0, 128, EPI_BIAS | EPI_ADD_AUX)
    assert torch.allclose(C32.double(), base + bias.double() + res.double(), rtol=1e-5, atol=1e-4)
    # input gradient through ReLU: bf16 mask tile (the stored hidden activation), in place, scaled, + column sums
    _, _, _, Bt = operands(M, N, K, 0, 1, 11)            # B stored [K, N] for the MN-major form
    hid = torch.relu(torch.randn(M, N, device="cuda")).bfloat16()
    out = hid.clone()
    colsum = torch.zeros(N, device="cuda")
    gemm(A, Bt, out, out, None, M, N, K, 0, 1, 128, EPI_MASK_AUX | EPI_COLSUM, alpha=1.25, colsum=colsum)
    want = torch.where(hid.double() > 0, 1.25 * base, torch.zeros_like(base))
    assert ((out.double() - want).abs() <= 2.0 ** -8 * want.abs() + 1e-3).all()
    assert torch.allclose(colsum.double(), out.double().sum(0), rtol=1e-4, atol=1e-2)
