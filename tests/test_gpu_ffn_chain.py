"""The chained feed-forward kernels (arb_ffn_forward / arb_ffn_backward_input, csrc/ffn_chain.cu) against the two
GEMMs they replace, bit for bit.

The reference composes arb_gemm_tf32 products on the same tf32-rounded weights: H = relu(x W1^T + b1) and
Y = H W2^T + b2 + res forward; dH = (dY W2) masked by H > 0 (the mask-tile epilogue) and dX = dH W1 backward.  Y, H,
the bit words (equal to H > 0), dH and dX must be equal (torch.equal).  The b1 gradient must equal the EPI_COLSUM
epilogue's order, restated on the host in float32: per 128-row tile and column four 32-row segments summed in row order
from 0.f, (s0 + s1) + (s2 + s3), the tile slots reduced by det_reduce_kernel's grouping and added to the incoming
gradient.  Outputs are NaN-prefilled: with a device-side row count, the tiles past it stay untouched.

At the scorer level the chained build must give the scores and every parameter gradient of the two-GEMM path
(arb_set_relu_bits(0)) bit for bit -- except the b1 gradient: that path's mask-tile epilogue runs in the one-tile GEMM,
whose EPI_COLSUM sums each tile's 128 rows in one sequence, so it differs in the association of the column sums only."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_gpu_attn_bwd_order import det_reduce

pytestmark = pytest.mark.gpu

EPI_BIAS, EPI_RELU, EPI_ADD_AUX, EPI_MASK_AUX = 1, 2, 4, 8
F32 = np.float32


@pytest.fixture(scope="module")
def lib():
    from allrank_b200 import _lib
    i, p, f = ctypes.c_int32, ctypes.c_void_p, ctypes.c_float
    q = ctypes.c_int64
    _lib.register("arb_gemm_tf32", i, [p, p, p, p, p, i, i, i, i, i, i, q, q, q, i, i, f, i, p])
    _lib.register("arb_ffn_forward", i, [p, p, p, p, p, p, i, i, i, p, p, p, p, p])
    _lib.register("arb_ffn_backward_input", i, [p, p, p, p, i, i, i, p, p, p, p, p])
    _lib.register("arb_set_tf32_round_on_load", None, [i])
    return _lib


def pick_block_n(n):
    return 32 if n <= 32 else (64 if n < 128 else 128)


def gemm(lib, A, B, M, N, K, flags, bias=None, aux=None):
    C = torch.full((M, N), float("nan"), device="cuda")
    rc = lib.lib().arb_gemm_tf32(lib.ptr(A), lib.ptr(B), lib.ptr(C), lib.ptr(aux), lib.ptr(bias), M, N, K, 0, 0, 1, 0, 0,
                                 0, pick_block_n(N), flags, 1.0, 1, lib.stream_ptr())
    lib.check(rc, "arb_gemm_tf32")
    return C


def tf32(t):
    """round to nearest even tf32, as the scorer's weight copy does"""
    b = t.contiguous().view(torch.int32).long()
    b = (b + 0xFFF + ((b >> 13) & 1)) & ~0x1FFF
    return ((b + 2 ** 31) % 2 ** 32 - 2 ** 31).int().view(torch.float32)


def pack_bits(h):
    rows, f = h.shape
    w = ((h > 0).view(rows, f // 32, 32).long() << torch.arange(32, device=h.device)).sum(-1)
    return ((w + 2 ** 31) % 2 ** 32 - 2 ** 31).int()


def make(rows, d, f, seed, rnd=True):
    g = torch.Generator().manual_seed(seed)
    w = lambda *s, sc=1.0: (sc * torch.randn(*s, generator=g)).cuda()   # noqa: E731
    x, res, dy = w(rows, d), w(rows, d), w(rows, d)
    w1, w2 = w(f, d, sc=d ** -0.5), w(d, f, sc=f ** -0.5)
    if rnd:
        w1, w2 = tf32(w1), tf32(w2)
    b1, b2, gb1 = w(f, sc=0.3), w(d, sc=0.3), w(f)
    return x, res, dy, w1, w2, b1, b2, gb1


def chain_fwd(lib, x, w1, b1, w2, b2, res, rows, d, f, rows_dev=None):
    y = torch.full((rows, d), float("nan"), device="cuda")
    h = torch.full((rows, f), float("nan"), device="cuda")
    bits = torch.full((rows, f // 32), -1, dtype=torch.int32, device="cuda")
    rc = lib.lib().arb_ffn_forward(lib.ptr(x), lib.ptr(w1), lib.ptr(b1), lib.ptr(w2), lib.ptr(b2), lib.ptr(res), rows, d,
                                   f, lib.ptr(y), lib.ptr(h), lib.ptr(bits), lib.ptr(rows_dev), lib.stream_ptr())
    lib.check(rc, "arb_ffn_forward")
    return y, h, bits


def chain_bwd(lib, dy, w2, w1, bits, gb1, rows, d, f, rows_dev=None):
    dx = torch.full((rows, d), float("nan"), device="cuda")
    dh = torch.full((rows, f), float("nan"), device="cuda")
    gb = gb1.clone()
    w2t, w1t = w2.t().contiguous(), w1.t().contiguous()
    rc = lib.lib().arb_ffn_backward_input(lib.ptr(dy), lib.ptr(w2t), lib.ptr(w1t),
                                          lib.ptr(bits), rows, d, f, lib.ptr(dx), lib.ptr(dh), lib.ptr(gb),
                                          lib.ptr(rows_dev), lib.stream_ptr())
    lib.check(rc, "arb_ffn_backward_input")
    return dx, dh, gb


def emulate_b1(dh, n_tiles, gb1):
    """the EPI_COLSUM order over the chain's own dH (rows past it: exact zeros), then the slot reduction"""
    f = dh.shape[1]
    a = np.zeros((n_tiles * 128, f), F32)
    a[:dh.shape[0]] = dh.cpu().numpy()
    a = a.reshape(n_tiles, 4, 32, f)
    s = np.zeros((n_tiles, 4, f), F32)
    for r in range(32):
        s = s + a[:, :, r]
    slots = (s[:, 0] + s[:, 1]) + (s[:, 2] + s[:, 3])
    return gb1.cpu().numpy() + det_reduce(slots)


def assert_bits_equal(got, want, what):
    g, w = got.cpu().numpy().view(np.int32), np.asarray(want, F32).view(np.int32)
    diff = np.nonzero(g != w)[0]
    assert diff.size == 0, f"{what}: {diff.size} columns differ, first {diff[:4].tolist()}"


def check(lib, rows, d, f, seed, rnd=True):
    x, res, dy, w1, w2, b1, b2, gb1 = make(rows, d, f, seed, rnd)
    h_ref = gemm(lib, x, w1, rows, f, d, EPI_BIAS | EPI_RELU, bias=b1)
    y_ref = gemm(lib, h_ref, w2, rows, d, f, EPI_BIAS | EPI_ADD_AUX, bias=b2, aux=res)
    y, h, bits = chain_fwd(lib, x, w1, b1, w2, b2, res, rows, d, f)
    assert torch.equal(h, h_ref)
    assert torch.equal(y, y_ref)
    assert torch.equal(bits, pack_bits(h_ref))
    dh_ref = gemm(lib, dy, w2.t().contiguous(), rows, f, d, EPI_MASK_AUX, aux=h_ref)
    dx_ref = gemm(lib, dh_ref, w1.t().contiguous(), rows, d, f, 0)
    dx, dh, gb = chain_bwd(lib, dy, w2, w1, bits, gb1, rows, d, f)
    assert torch.equal(dh, dh_ref)
    assert torch.equal(dx, dx_ref)
    assert_bits_equal(gb, emulate_b1(dh, (rows + 127) // 128, gb1), "b1 gradient")


DS = [32, 64, 96, 128, 256]
FS = [64, 128, 512, 1024]


@pytest.mark.parametrize("f", FS)
@pytest.mark.parametrize("d", DS)
def test_chain_equals_the_two_gemms(lib, d, f):
    check(lib, 4013, d, f, seed=d + f)


@pytest.mark.parametrize("rows,d,f", [(1, 128, 512), (127, 128, 512), (128, 128, 512), (129, 96, 128),
                                      (2 ** 17 + 37, 128, 512), (2 ** 17 + 37, 256, 1024)])
def test_chain_row_counts(lib, rows, d, f):
    check(lib, rows, d, f, seed=rows % 1000)


@pytest.mark.parametrize("d,f", [(128, 512), (96, 64)])
def test_chain_truncation(lib, d, f):
    """arb_set_tf32_round_on_load(0): the tensor core truncates both products' operands"""
    lib.lib().arb_set_tf32_round_on_load(0)
    try:
        check(lib, 1000, d, f, seed=5, rnd=False)
    finally:
        lib.lib().arb_set_tf32_round_on_load(1)


@pytest.mark.parametrize("d,f", [(128, 512), (256, 1024)])
def test_chain_device_row_count(lib, d, f):
    rows, live = 4013, 1500
    done = (live + 127) // 128 * 128                        # the last live tile is written whole
    x, res, dy, w1, w2, b1, b2, gb1 = make(rows, d, f, seed=11)
    rd = torch.tensor([live], dtype=torch.int32, device="cuda")
    h_ref = gemm(lib, x, w1, rows, f, d, EPI_BIAS | EPI_RELU, bias=b1)
    y_ref = gemm(lib, h_ref, w2, rows, d, f, EPI_BIAS | EPI_ADD_AUX, bias=b2, aux=res)
    y, h, bits = chain_fwd(lib, x, w1, b1, w2, b2, res, rows, d, f, rows_dev=rd)
    assert torch.equal(h[:done], h_ref[:done]) and torch.equal(y[:done], y_ref[:done])
    assert torch.equal(bits[:done], pack_bits(h_ref[:done]))
    assert torch.isnan(h[done:]).all() and torch.isnan(y[done:]).all() and (bits[done:] == -1).all()
    dh_ref = gemm(lib, dy, w2.t().contiguous(), rows, f, d, EPI_MASK_AUX, aux=h_ref)
    dx_ref = gemm(lib, dh_ref, w1.t().contiguous(), rows, d, f, 0)
    bits = torch.where(torch.arange(rows, device="cuda")[:, None] < done, bits, pack_bits(h_ref))
    dx, dh, gb = chain_bwd(lib, dy, w2, w1, bits, gb1, rows, d, f, rows_dev=rd)
    assert torch.equal(dh[:done], dh_ref[:done]) and torch.equal(dx[:done], dx_ref[:done])
    assert torch.isnan(dh[done:]).all() and torch.isnan(dx[done:]).all()
    assert_bits_equal(gb, emulate_b1(dh[:done], (rows + 127) // 128, gb1), "b1 gradient")


@pytest.mark.parametrize("pack", [1, 0], ids=["packed", "dense"])
def test_scorer_chain_equals_the_two_gemm_path(lib, pack):
    """a cfg2-shaped model (d 128, d_ff 512, S 240): the chained FFN against arb_set_relu_bits(0)'s two GEMMs.  The
    scorer chains the linears from four 128-row tiles per SM on: the batch is just above that."""
    from tests.test_gpu_pack_rows import _model, _run, _slates
    model = _model(N=2, d=128, h=4, dff=512)
    S = 240
    B = 4 * 128 * torch.cuda.get_device_properties(0).multi_processor_count // S + 8
    x, y = _slates(B, S)
    x, y = x.cuda(), y.cuda()
    w = torch.randn(B, S, generator=torch.Generator().manual_seed(2)).cuda()
    w = torch.where(y == -1, torch.zeros_like(w), w)
    outs, launches = [], []
    lib.register("arb_set_relu_bits", None, [ctypes.c_int32])
    for bits in (0, 1):
        lib.lib().arb_set_relu_bits(bits)
        try:
            n0 = lib.launch_count()
            outs.append(_run(model, x, y, w, pack))
            launches.append(lib.launch_count() - n0)
        finally:
            lib.lib().arb_set_relu_bits(lib.default_relu_bits())
    assert launches[1] == launches[0] - 4, launches      # one kernel instead of two, per direction and layer
    assert torch.equal(outs[0][0], outs[1][0])
    (_, g0), (_, g1) = outs
    b1 = torch.zeros_like(g0, dtype=torch.bool)
    for o, n in _b1_offsets(model):
        b1[o:o + n] = True
    assert torch.equal(g0[~b1], g1[~b1])
    gap = (g0[b1] - g1[b1]).abs().max().item()
    assert gap <= 4e-6 * g0.abs().max().item(), gap
    assert g1.abs().max().item() > 0


def _b1_offsets(model):
    """(offset, length) of every FFN b1 in the flat parameter (and gradient) buffer"""
    base = model.flat_parameters.data_ptr()
    out = [((p.data_ptr() - base) // 4, p.numel()) for name, p in model.named_parameters()
           if name.endswith("feed_forward.w_1.bias")]
    assert len(out) == 2, [n for n, _ in model.named_parameters()]
    return out
