"""fp32 products whose operands are both MN-major -- the split-K weight gradients dW = dY^T X, reduced over the rows of
the batch -- on warpgroup MMA: each ring stage is rewritten K-major on chip, rounded to nearest tf32 on the way (or left
for the tensor core to truncate with rounding off).  Ragged row counts, N = 136 (a ragged last column tile), two output
row tiles and more, one split and many."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_ATOMIC = 16


@pytest.fixture(scope="module")
def gemm():
    from allrank_b200 import _lib
    c_p, c_i, c_f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float
    _lib.register("arb_gemm_tf32", c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, ctypes.c_int64,
                                         ctypes.c_int64, ctypes.c_int64, c_i, c_i, c_f, c_i, c_p])
    _lib.register("arb_set_tf32_round_on_load", None, [ctypes.c_int32])

    def call(A, B, C, M, N, K, a_mn, b_mn, block_n, flags=0, split_k=1):
        rc = _lib.lib().arb_gemm_tf32(_lib.ptr(A), _lib.ptr(B), _lib.ptr(C), None, None, M, N, K, a_mn, b_mn, 1, 0, 0,
                                      0, block_n, flags, 1.0, split_k, _lib.stream_ptr())
        _lib.check(rc, "arb_gemm_tf32")
        torch.cuda.synchronize()
    return call


def _tf32(x, nearest):
    """fp32 -> tf32 on the host: round to nearest even, or truncate."""
    b = x.view(torch.int32)
    if nearest:
        b = b + 0xFFF + ((b >> 13) & 1)
    return (b & ~0x1FFF).view(torch.float32)


@pytest.mark.parametrize("split_k", [1, 37])
@pytest.mark.parametrize("M", [384, 512])
@pytest.mark.parametrize("block_n", [32, 64, 128])
def test_split_k_weight_gradient_rounding_modes(gemm, block_n, M, split_k):
    """dW[M, N] = dY^T X over 4013 rows (the last 32-row k-block holds 13): with rounding on, the product of the
    nearest-rounded operands, with it off the one of the truncated operands (each within fp32 accumulation error,
    far below the gap between the two)."""
    from allrank_b200 import _lib
    torch.manual_seed(block_n + M + split_k)
    rows, N = 4013, 136
    dY = torch.randn(rows, M, device="cuda")
    X = torch.randn(rows, N, device="cuda")
    out = {}
    try:
        for nearest in (1, 0):
            _lib.lib().arb_set_tf32_round_on_load(nearest)
            dW = torch.zeros(M, N, device="cuda")
            gemm(dY, X, dW, M, N, rows, 1, 1, block_n, EPI_ATOMIC, split_k)
            out[nearest] = dW
    finally:
        _lib.lib().arb_set_tf32_round_on_load(1)
    scale = dY.abs().double().t() @ X.abs().double()
    for nearest, dW in out.items():
        ref = _tf32(dY, nearest).double().t() @ _tf32(X, nearest).double()
        other = _tf32(dY, 1 - nearest).double().t() @ _tf32(X, 1 - nearest).double()
        err = ((dW.double() - ref).abs() / scale).max().item()
        gap = ((other - ref).abs() / scale).max().item()
        assert err < 1e-5 and gap > 10 * err, (nearest, err, gap)


@pytest.mark.parametrize("block_n", [32, 64, 128])
def test_mn_major_product_equals_the_k_major_one_bit_for_bit(gemm, block_n):
    """The same product from MN-major operands (rewritten K-major on chip) and from their K-major copies: same
    instruction shapes, same k8 order, same rounding -> the same bits."""
    torch.manual_seed(block_n)
    M, N, K = 300, 136, 1000
    A = torch.randn(K, M, device="cuda")          # MN-major: [K, M]
    B = torch.randn(K, N, device="cuda")          # MN-major: [K, N]
    C_mn = torch.full((M, N), float("nan"), device="cuda")
    C_k = torch.full((M, N), float("nan"), device="cuda")
    gemm(A, B, C_mn, M, N, K, 1, 1, block_n)
    gemm(A.t().contiguous(), B.t().contiguous(), C_k, M, N, K, 0, 0, block_n)
    assert torch.equal(C_mn, C_k)
