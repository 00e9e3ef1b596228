"""The summation order of the fused attention backward's QKV bias gradient, pinned bit for bit.

The key-projection bias has a mathematically zero gradient, so what the kernel returns for it is pure rounding noise,
and Adam turns any change of that noise into full-size parameter steps (DESIGN.md section 4.3).  The order is part of
the kernel's contract: per CTA, items in the order the CTA walks them (blockIdx.x, + gridDim.x, ...), per item its
128-row tiles in order, per tile and output column the tile's rows in order starting from 0.f, the tile's sum then
added to the CTA's accumulator; the CTA slots are then reduced by det_reduce_kernel (groups of 64 slots, 8 warp-strided
partial sums each added in sequence, the partials added in warp order, repeated over the groups until one is left) and
added to the incoming bias gradient.

The test restates that order on the host in float32 over the kernel's own dQ, dK, dV (fp32 or bf16 as stored) and
compares the result bitwise with the returned bias gradient, through arb_attention_backward (dense layout).  Cases have
more items than SMs, one- and two-tile extents, dk 16 and 32, dropout, the bf16 gradients, and both schedules (one
CTA per SM, one CTA per item)."""
import numpy as np
import pytest
import torch

from tests.test_gpu_attention_kernels import lib, make_dctx, make_inputs, run_bwd, run_fwd  # noqa: F401

pytestmark = pytest.mark.gpu

F32 = np.float32


def det_reduce(parts):
    """det_reduce_kernel's order over slots [n, elems]."""
    n = parts.shape[0]
    groups = []
    for s0 in range(0, n, 64):
        s1 = min(n, s0 + 64)
        warps = []
        for w in range(8):
            t = np.zeros(parts.shape[1], F32)
            for s in range(s0 + w, s1, 8):
                t = t + parts[s]
            warps.append(t)
        v = warps[0]
        for w in range(1, 8):
            v = v + warps[w]
        groups.append(v)
    return groups[0] if len(groups) == 1 else det_reduce(np.stack(groups))


def emulate_bias(d_qkv, extents, S, h, dk, n_ctas, db0):
    B = len(extents)
    g = d_qkv.float().cpu().numpy().reshape(B, S, 3, h, dk).transpose(0, 3, 1, 2, 4)   # [B, h, S, 3, dk]
    rows = np.array([(max(1, min(S, e)) + 15) // 16 * 16 for e in extents])
    n_tiles = (S + 127) // 128
    # per (item, tile, output column): the tile's rows in order, from 0.f
    tsum = np.zeros((B, h, n_tiles, 3, dk), F32)
    for tile in range(n_tiles):
        s = np.zeros((B, h, 3, dk), F32)
        for r in range(128 * tile, min(S, 128 * tile + 128)):
            s = np.where((r < rows)[:, None, None, None], s + g[:, :, r], s)
        tsum[:, :, tile] = s
    # per CTA: its items in order, each item's tiles in order
    items = B * h
    acc = np.zeros((n_ctas, 3, h, dk), F32)
    ci = np.arange(n_ctas)
    for r0 in range(0, items, n_ctas):
        it = r0 + ci
        valid = it < items
        b, hd = np.minimum(it, items - 1) // h, np.minimum(it, items - 1) % h
        for tile in range(n_tiles):
            live = valid & (128 * tile < rows[b])
            cur = acc[ci, :, hd, :]
            acc[ci, :, hd, :] = np.where(live[:, None, None], cur + tsum[b, hd, tile], cur)
    return db0.cpu().numpy() + det_reduce(acc.reshape(n_ctas, 3 * h * dk))


CASES = [(32, 0.1, False), (16, 0.1, False), (32, 0.0, True), (16, 0.3, True)]


@pytest.mark.parametrize("persistent", [1, 0], ids=["per-sm", "per-item"])
@pytest.mark.parametrize("dk,p,bf16", CASES, ids=[f"dk{dk}-p{p}" + ("-bf16" if b else "") for dk, p, b in CASES])
def test_bias_gradient_summation_order(lib, dk, p, bf16, persistent):
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    S, h = 256, 2
    cycle = [256, 200, 17, 129, 128, 1, 100, 240, 33, 144, 16]
    B = n_sm + 7                                   # about two items per SM and some with three
    ex = [cycle[(3 * b + b // 5) % len(cycle)] for b in range(B)]
    qkv, mask, ext = make_inputs(ex, S, h, dk, seed=40 + dk)
    ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, dk, p, bf16=bf16)
    d_ctx = make_dctx(ex, S, h * dk, 41 + dk)
    db0 = torch.randn(3 * h * dk, generator=torch.Generator().manual_seed(42)).cuda()
    try:
        lib.lib().arb_set_attention_bwd_persistent(persistent)
        d_qkv, dbias = run_bwd(lib, qkv, ctx, d_ctx, mask, ext, smax, ssum, B, S, h, dk, p, db0)
    finally:
        lib.lib().arb_set_attention_bwd_persistent(1)
    assert torch.isfinite(d_qkv).all()
    items = B * h
    want = emulate_bias(d_qkv, ex, S, h, dk, min(items, n_sm) if persistent else items, db0)
    got = dbias.cpu().numpy()
    diff = np.nonzero(got.view(np.int32) != want.view(np.int32))[0]
    assert diff.size == 0, f"{diff.size} bias columns differ from the emulated order, first {diff[:4].tolist()}: " \
                           f"{got[diff[:4]].tolist()} vs {want[diff[:4]].tolist()}"
