"""The TMA + tensor-core TF32 GEMM building block against an fp64 reference of the same op.

The kernels round each fp32 operand to tf32 (nearest even) and accumulate in fp32, one rounding per k8 step of the
tensor core.  The reference is therefore the fp64 product of the operands rounded the same way on the host, and the
bound is the accumulation depth's: TAU * (ceil(K / 8) + 1) * 2^-24 * sum_k |a~||b~| (+1: the epilogue's rounding);
truncated operands, or operands rounded another way, miss it by orders of magnitude.  The epilogue and the exact
bits of the rounding are pinned by tests/test_gpu_gemm_epilogues.py."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_BIAS, EPI_RELU, EPI_ADD_AUX, EPI_MASK_AUX, EPI_ATOMIC = 1, 2, 4, 8, 16


@pytest.fixture(scope="module")
def gemm():
    from allrank_b200 import _lib
    c_p, c_i, c_f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float
    _lib.register("arb_gemm_tf32", c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, ctypes.c_int64,
                                         ctypes.c_int64, ctypes.c_int64, c_i, c_i, c_f, c_i, c_p])

    def call(A, B, C, aux, bias, M, N, K, a_mn, b_mn, batch, sa, sb, sc, block_n, flags, alpha, split_k=1):
        rc = _lib.lib().arb_gemm_tf32(_lib.ptr(A), _lib.ptr(B), _lib.ptr(C), _lib.ptr(aux), _lib.ptr(bias), M, N, K,
                                      a_mn, b_mn, batch, sa, sb, sc, block_n, flags, alpha, split_k,
                                      _lib.stream_ptr())
        _lib.check(rc, "arb_gemm_tf32")
        torch.cuda.synchronize()
    return call


TAU = 2.0      # as tests/test_gpu_gemm_epilogues.py


def tf32(x):
    """fp32 -> tf32, round to nearest even (what the kernels do to their operands)"""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    b = (b + 0xFFF + ((b >> 13) & 1)) & 0xFFFFE000
    return torch.where(b >= 2 ** 31, b - 2 ** 32, b).to(torch.int32).view(torch.float32)


def ref_and_bound(A, B, steps=0):
    """A [.., M,K], B [.., N,K] logical; returns the fp64 product of the tf32-rounded operands and the depth bound
    (steps: further fp32 roundings of the result, e.g. the split-K slot sums)."""
    Ar, Br = tf32(A).double(), tf32(B).double()
    ref = Ar @ Br.transpose(-1, -2)
    depth = math.ceil(A.shape[-1] / 8) + 1 + steps
    bound = TAU * depth * 2.0 ** -24 * (Ar.abs() @ Br.abs().transpose(-1, -2)) + 1e-30
    return ref, bound


def epi_bound(bound, want):
    """the product's bound, plus one fp32 rounding of each epilogue addition"""
    return bound + 2.0 ** -23 * want.abs()


@pytest.mark.parametrize("block_n", [32, 64, 128])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 128), (240, 96, 136), (300, 200, 40), (64, 32, 512)])
def test_plain_gemm_all_majors(gemm, block_n, a_mn, b_mn, M, N, K):
    if (M % 4 or N % 4 or K % 4):
        pytest.skip("TMA needs 16-byte row pitch")
    torch.manual_seed(M * 7 + N * 3 + K + a_mn * 2 + b_mn)
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(N, K, device="cuda")
    C = torch.full((M, N), float("nan"), device="cuda")
    As = A.t().contiguous() if a_mn else A
    Bs = B.t().contiguous() if b_mn else B
    gemm(As, Bs, C, None, None, M, N, K, a_mn, b_mn, 1, 0, 0, 0, block_n, 0, 1.0)
    ref, bound = ref_and_bound(A, B)
    assert torch.isfinite(C).all()
    assert ((C.double() - ref).abs() <= bound).all(), float(((C.double() - ref).abs() / bound).max())


def test_epilogues(gemm):
    torch.manual_seed(0)
    M, N, K = 256, 128, 128
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") / K ** 0.5
    bias = torch.randn(N, device="cuda")
    X = torch.randn(M, N, device="cuda")
    base, bound = ref_and_bound(A, W)
    # bias + relu
    C = torch.empty(M, N, device="cuda")
    gemm(A, W, C, None, bias, M, N, K, 0, 0, 1, 0, 0, 0, 64, EPI_BIAS | EPI_RELU, 1.0)
    want = torch.relu(base + bias.double())
    assert ((C.double() - want).abs() <= epi_bound(bound, want)).all()
    # bias + residual, in place (C aliases aux)
    Xc = X.clone()
    gemm(A, W, Xc, Xc, bias, M, N, K, 0, 0, 1, 0, 0, 0, 128, EPI_BIAS | EPI_ADD_AUX, 1.0)
    want = base + bias.double() + X.double()
    assert ((Xc.double() - want).abs() <= epi_bound(2 * bound, want)).all()
    # relu-backward mask with a scale
    C = torch.empty(M, N, device="cuda")
    gemm(A, W, C, X, None, M, N, K, 0, 0, 1, 0, 0, 0, 32, EPI_MASK_AUX, 0.5)
    assert ((C.double() - 0.5 * base * (X > 0).double()).abs() <= 0.5 * bound).all()


def test_batched_and_broadcast(gemm):
    torch.manual_seed(1)
    nb, M, N, K = 6, 240, 240, 32
    Q = torch.randn(nb, M, K, device="cuda")
    Kt = torch.randn(nb, N, K, device="cuda")
    C = torch.full((nb, M, N), float("nan"), device="cuda")
    gemm(Q, Kt, C, None, None, M, N, K, 0, 0, nb, M * K, N * K, M * N, 64, 0, 0.25)
    ref, bound = ref_and_bound(Q, Kt)
    assert ((C.double() - 0.25 * ref).abs() <= bound).all()
    # P @ V: A = P [M, keys] K-major, B = V [keys, 32] stored row-major = MN-major operand
    P = torch.softmax(C, dim=-1)
    V = torch.randn(nb, N, 32, device="cuda")
    O = torch.full((nb, M, 32), float("nan"), device="cuda")
    gemm(P, V, O, None, None, M, 32, N, 0, 1, nb, M * N, N * 32, M * 32, 32, 0, 1.0)
    ref, bound = ref_and_bound(P, V.transpose(-1, -2))
    assert ((O.double() - ref).abs() <= bound).all()
    # weights shared across the batch (stride 0)
    W = torch.randn(48, K, device="cuda")
    Y = torch.full((nb, M, 48), float("nan"), device="cuda")
    gemm(Q, W, Y, None, None, M, 48, K, 0, 0, nb, M * K, 0, M * 48, 64, 0, 1.0)
    ref, bound = ref_and_bound(Q, W.expand(nb, 48, K))
    assert ((Y.double() - ref).abs() <= bound).all()


def test_split_k_weight_gradient(gemm):
    """dW[out,in] = dY^T X with the reduction over all rows split across CTAs (both operands MN-major)."""
    torch.manual_seed(2)
    rows, out_f, in_f = 15360, 128, 136
    dY = torch.randn(rows, out_f, device="cuda")
    X = torch.randn(rows, in_f, device="cuda")
    dW = torch.zeros(out_f, in_f, device="cuda")
    gemm(dY, X, dW, None, None, out_f, in_f, rows, 1, 1, 1, 0, 0, 0, 64, EPI_ATOMIC, 1.0, split_k=37)
    ref, bound = ref_and_bound(dY.t(), X.t(), steps=37)
    assert ((dW.double() - ref).abs() <= bound).all()


def test_linearity_property(gemm):
    """Size-independent check at a large shape: GEMM(A, B1 + B2) == GEMM(A, B1) + GEMM(A, B2) up to TF32
    rounding, and the result is invariant to the tile width."""
    torch.manual_seed(3)
    M, N, K = 4096, 512, 128
    A = torch.randn(M, K, device="cuda")
    B1 = torch.randn(N, K, device="cuda")
    outs = []
    for bn in (32, 64, 128):
        C = torch.empty(M, N, device="cuda")
        gemm(A, B1, C, None, None, M, N, K, 0, 0, 1, 0, 0, 0, bn, 0, 1.0)
        outs.append(C)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    ref, bound = ref_and_bound(A, B1)
    assert ((outs[0].double() - ref).abs() <= bound).all()


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("K", [128, 512])
@pytest.mark.parametrize("block_n", [64, 128])
def test_persistent_modes_are_bit_identical_to_the_tile_kernel(gemm, mode, K, block_n):
    """Every CTA of the persistent kernel walks several tiles (M x N = 400 x 2 tiles of 128 x 128 on 148 SMs), with
    and without a residual / ReLU-mask tile, ragged last tiles included; same MMA order per tile -> same bits as the
    one-tile-per-CTA kernel."""
    from allrank_b200 import _lib
    _lib.register("arb_set_gemm_persistent", None, [ctypes.c_int32])
    torch.manual_seed(K + block_n)
    M, N = 128 * 400 - 40, 256 - 8
    A = torch.randn(M, K, device="cuda")
    W = torch.randn(N, K, device="cuda") / K ** 0.5
    bias = torch.randn(N, device="cuda")
    X = torch.randn(M, N, device="cuda")

    def run():
        outs = []
        C = torch.empty(M, N, device="cuda")
        gemm(A, W, C, None, bias, M, N, K, 0, 0, 1, 0, 0, 0, block_n, EPI_BIAS | EPI_RELU, 1.0)
        outs.append(C)
        Xc = X.clone()
        gemm(A, W, Xc, Xc, bias, M, N, K, 0, 0, 1, 0, 0, 0, block_n, EPI_BIAS | EPI_ADD_AUX, 1.0)
        outs.append(Xc)
        C = torch.empty(M, N, device="cuda")
        gemm(A, W, C, X, None, M, N, K, 0, 0, 1, 0, 0, 0, block_n, EPI_MASK_AUX, 0.5)
        outs.append(C)
        # no specialised epilogue for this combination: both kernels run their generic per-element path
        Xc = X.clone()
        gemm(A, W, Xc, Xc, None, M, N, K, 0, 0, 1, 0, 0, 0, block_n, EPI_RELU | EPI_ADD_AUX, 0.5)
        outs.append(Xc)
        return outs

    try:
        _lib.lib().arb_set_gemm_persistent(0)
        want = run()
        _lib.lib().arb_set_gemm_persistent(mode)
        got = run()
    finally:
        import os
        _lib.lib().arb_set_gemm_persistent(int(os.environ.get("ARB_GEMM_PERSISTENT", 2)))
    base, bound = ref_and_bound(A, W)
    ref = base + bias.double() + X.double()
    assert ((want[1].double() - ref).abs() <= epi_bound(2 * bound, ref)).all()
    for w, g in zip(want, got):
        assert torch.equal(w, g)
