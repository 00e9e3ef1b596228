"""The fused attention kernels (attn_fwd_kernel, attn_bwd_kernel + attn_delta_kernel) against a plain fp64 restatement of
the attention operation, head by head, through arb_attention_forward / arb_attention_backward -- the scorer's own
launch descriptors (csrc/scorer.cu: attn_fwd_args / attn_bwd_args).

Reference: attention() of transformer.py:137-156 and its gradient, per (slate, head), in float64 on the device, on the
inputs rounded to TF32 as the kernels round them (cvt.rn: nearest, ties to even; the tensor core truncates under
arb_set_tf32_round_on_load(0)).  What remains is the kernels' own rounding of P and dS to TF32 (one rounding, 2^-11
relative), the fp32 accumulation of the logits (dk 2^-24 of sum |q||k| each) and fp32 sums.  Every element is bounded
on its own by the same computation over absolute values:
    O      tau * sum_j P_ij D_ij r_ij |V_j|                          (D: the scaled dropout mask)
    dV     tau * sum_i P_ij D_ij r_ij |dO_i|
    dQ     tau * scale * sum_j |dS|_ij |K_j|,   dK  tau * scale * sum_i |dS|_ij |Q_i|
with r_ij = 2^-11 + scale dk 2^-24 (a_ij + max_j a_ij), a = |Q||K|^T (the logit's error and the row max's), and
|dS| = P (D |dO| |V|^T + sum_e |dO_e||O_e|) r (delta = rowsum(dO * O) over the context read), so one wrong row,
key or column fails however small it is next to the whole tensor.  For a row with one dominant key the bound is
reached by a single rounding of P (ratio 1); TAU = 1.25 leaves room for ex2.approx and the fp32 sums.  Calibration on
an H100 80GB HBM3 (power limit 400 W): the worst error / bound over the module is 0.85 (O, with dropout), 0.79 (dV),
0.62 (dQ), 0.30 (dK), 0.19 (row max), 0.07 (row sum), 0.07 (QKV bias gradient); RATIOS collects them per case.
bf16 outputs must lie between the bf16 roundings of ref -/+ bound, and at least 80 % of them must equal the rounding
(nearest even) of the reference exactly: the kernels' own TF32 rounding of P and dS moves some values across a bf16
rounding boundary (observed: 96 % exact for the context, 88 % for dQ, where dS cancels), while a context or gradient
truncated to bf16 misses about half.

Outputs are pre-filled with NaN (a row no kernel writes fails), every case runs twice and must give the same bits, and
the backward's rows at or beyond its extent must be exactly +0.  Cases: head widths 16 / 32 / 64 (backward 16 / 32),
S = 256, 240, 129, 37 (TMA boxes past S), extents on both sides of every 16-row strip and 128-row tile, masked items
inside slates, large garbage in padded rows (padded keys would win every softmax if the mask were ignored), planted
dominant keys at extent - 1 and at the first / last key of a 16-row strip, an all-padded slate, a backward extent past
the key extent, null extents, dropout at p = 0, 0.1, 0.3, batches from 6 items to ~2400, extents that make a CTA's
consecutive items alternate between fitting its two-slot operand pool and not, both backward schedules, the bf16
context and gradients, and truncating TF32 operands."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle.tf32_emulation import tf32_trunc
from tests.dropout_masks import M32, SITE_ATTN_P, _mix32, _site, mask_tensor

pytestmark = pytest.mark.gpu

TAU = 1.25
U = 2.0 ** -11            # one TF32 rounding (10 explicit mantissa bits, to nearest)
FLOOR = 2.0 ** -100       # ex2.approx flushes subnormal probabilities to zero
SEED = 0xD1B54A32D192ED03  # a call seed with all 64 bits in play
LAYER = 3
RATIOS = {}               # worst error / bound per output kind (printed; the calibration of TAU)


@pytest.fixture(scope="module")
def lib():
    from allrank_b200 import _lib
    c_p, c_i, c_f, c_u = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float, ctypes.c_uint64
    _lib.register("arb_attention_forward", c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_f, c_u, c_i, c_i, c_p, c_p, c_p,
                                                 c_p])
    _lib.register("arb_attention_backward", c_i, [c_p, c_p, c_i, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_f, c_u,
                                                  c_i, c_p, c_p, c_p, c_p])
    _lib.register("arb_set_attention_bwd_persistent", None, [c_i])
    _lib.register("arb_set_tf32_round_on_load", None, [c_i])
    yield _lib
    for name, worst in sorted(RATIOS.items()):
        print(f"attention kernels: worst error / bound of {name}: {worst:.3g}")


# ------------------------------------------------------------------------------------------------ inputs
def tf32(x, mode):
    """fp32 -> TF32 as the kernels see an operand: "rne" (cvt.rn, round on load), "trunc" (the tensor core, rounding
    off) or "rna" (ties away from zero)."""
    if mode != "rne":
        return tf32_trunc(x, mode)
    b = x.float().contiguous().view(torch.int32)
    b = b + 0x0FFF + ((b >> 13) & 1)
    return (b & ~0x1FFF).view(torch.float32)


def extents_for(S):
    return sorted({e for e in (1, 15, 16, 17, 31, 33, 127, 128, 129) if e <= S} | {S - 1, S})


def make_inputs(extents, S, h, dk, seed):
    """qkv [B*S, 3d], mask [B, S] (1 = padded; masked items inside longer slates, never at extent - 1), extents [B].
    Every (slate, head) has a common query direction u: the planted keys (extent - 1, and the first and last key of
    the 16-row strip below the last one) lie along it and dominate every query's softmax by ~5 nats; the padded keys
    lie further along it (they would take ~all of the probability if the mask were ignored) and carry 8x values."""
    g = torch.Generator().manual_seed(seed)
    B, d = len(extents), h * dk
    ext = torch.tensor(extents, dtype=torch.int32)
    pos = torch.arange(S)
    mask = pos[None, :] >= ext[:, None].long()
    mask |= (torch.rand(B, S, generator=g) < 0.08) & (pos[None, :] < ext[:, None].long() - 1)
    u = torch.nn.functional.normalize(torch.randn(B, 1, h, dk, generator=g), dim=-1)
    q = 0.5 * torch.randn(B, S, h, dk, generator=g) + 2.0 * u
    k = torch.randn(B, S, h, dk, generator=g)
    v = torch.randn(B, S, h, dk, generator=g)
    gam = 2.5 * math.sqrt(dk)
    for b, e in enumerate(extents):
        keys = {e - 1}
        if e > 32:
            s0 = 16 * ((e - 1) // 16 - 1)
            keys |= {s0, s0 + 15}
        for j in keys:
            k[b, j] += gam * u[b, 0]
            mask[b, j] = False
    pad = mask[:, :, None, None]
    k = torch.where(pad, k + 4.0 * gam * u, k)
    v = torch.where(pad, 8.0 * v, v)
    qkv = torch.stack([q, k, v], dim=2).reshape(B * S, 3 * d)
    return qkv.cuda(), mask.to(torch.uint8).cuda(), ext.cuda()


def make_dctx(gext, S, d, seed):
    """d ctx [B*S, d]: random below each slate's backward extent, zero at and beyond it."""
    g = torch.Generator().manual_seed(seed)
    B = len(gext)
    do = torch.randn(B, S, d, generator=g)
    do[torch.arange(S)[None, :] >= torch.tensor(gext)[:, None]] = 0.0
    return do.reshape(B * S, d).cuda()


def drop_masks(slates, B, h, S, p):
    """The scaled keep mask of the attention probabilities for the given slates [n, h, S, S] (float64), regenerated
    by the host restatement of csrc/dropout.cuh; element ((b*h + head)*S + q)*S + key."""
    seed, thresh, _ = _site(SEED, LAYER, SITE_ATTN_P, p)
    scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))     # as make_drop_site computes it
    b = np.asarray(slates, dtype=np.uint64)[:, None]
    idx = (b * np.uint64(h * S * S) + np.arange(h * S * S, dtype=np.uint64)[None, :]).reshape(-1)
    hsh = _mix32((idx & M32) ^ seed)
    hsh = _mix32((hsh + (idx >> np.uint64(32)) * np.uint64(0x9e3779b1) + np.uint64(0x7f4a7c15)) & M32)
    keep = (hsh >= thresh).astype(np.float64) * scale
    return torch.tensor(keep.reshape(len(slates), h, S, S)).cuda()


def heads(t, B, S, h, dk):
    """[B*S, h*dk] -> [B, h, S, dk]"""
    return t.view(B, S, h, dk).permute(0, 2, 1, 3)


# ------------------------------------------------------------------------------------------------ reference
def reference(qkv, mask, B, S, h, dk, D, mode="rne"):
    """fp64 attention (transformer.py:137-156) per (slate, head) on the TF32-rounded operands, with the companions the
    bounds need.  D: [B, h, S, S] scaled keep mask or None."""
    x = qkv.view(B, S, 3, h, dk)
    q, k, v = (tf32(x[:, :, i], mode).double().permute(0, 2, 1, 3) for i in range(3))
    scale = 1.0 / math.sqrt(dk)
    s = q @ k.transpose(-1, -2)
    sa = q.abs() @ k.abs().transpose(-1, -2)
    keym = mask.bool()[:, None, None, :]
    mx = s.masked_fill(keym, float("-inf")).amax(-1)
    P = torch.exp((s.masked_fill(keym, float("-inf")) - mx[..., None]) * scale)
    l = torch.where(torch.isfinite(mx), P.sum(-1), 0.0)     # a row without keys: sum 0, NaN probabilities
    Pn = P / l[..., None]
    Pd = Pn if D is None else Pn * D
    # fp32 logits: each within dk 2^-24 sum_e |q_e||k_e| (the row max too, through its own key)
    max_b = dk * 2.0 ** -24 * sa.masked_fill(keym, 0.0).amax(-1)
    rel = U + scale * (dk * 2.0 ** -24 * sa + max_b[..., None])
    return dict(q=q, k=k, v=v, scale=scale, Pn=Pn, Pd=Pd, D=D, rel=rel, mode=mode,
                max=mx, sum=l, O=Pd @ v, O_b=(Pd * rel) @ v.abs(), max_b=max_b)


def reference_bwd(R, d_ctx, ctx, B, S, h, dk):
    """dQ, dK, dV of the reference for the incoming d ctx, with delta = rowsum(dO * O) over the context the kernels
    read (ctx: fp32 or bf16 [B*S, d])."""
    do = heads(d_ctx, B, S, h, dk).double()
    dor = heads(tf32(d_ctx, R["mode"]), B, S, h, dk).double()
    o = heads(ctx, B, S, h, dk).double()
    delta = (do * o).sum(-1)
    delta_a = (do.abs() * o.abs()).sum(-1)
    q, k, v, Pn, Pd, D, sc = R["q"], R["k"], R["v"], R["Pn"], R["Pd"], R["D"], R["scale"]
    dP = dor @ v.transpose(-1, -2)
    dPa = dor.abs() @ v.abs().transpose(-1, -2)
    if D is not None:
        dP, dPa = dP * D, dPa * D
    dS = Pn * (dP - delta[..., None])
    dSa = Pn * (dPa + delta_a[..., None]) * R["rel"]
    return dict(dQ=sc * dS @ k, dQ_b=sc * dSa @ k.abs(),
                dK=sc * dS.transpose(-1, -2) @ q, dK_b=sc * dSa.transpose(-1, -2) @ q.abs(),
                dV=Pd.transpose(-1, -2) @ dor, dV_b=(Pd * R["rel"]).transpose(-1, -2) @ dor.abs())


# ------------------------------------------------------------------------------------------------ calls
def run_fwd(L, qkv, mask, ext, B, S, h, dk, p, bf16=False):
    d = h * dk
    ctx = torch.full((B * S, d), float("nan"), device="cuda", dtype=torch.bfloat16 if bf16 else torch.float32)
    smax = torch.full((B, h, S), float("nan"), device="cuda")
    ssum = torch.full((B, h, S), float("nan"), device="cuda")
    rc = L.lib().arb_attention_forward(L.ptr(qkv), L.ptr(mask), L.ptr(ext), B, S, h, dk, p, SEED, LAYER, int(bf16),
                                       L.ptr(ctx), L.ptr(smax), L.ptr(ssum), L.stream_ptr())
    L.check(rc, "arb_attention_forward")
    torch.cuda.synchronize()
    return ctx, smax, ssum


def run_bwd(L, qkv, ctx, d_ctx, mask, ext, smax, ssum, B, S, h, dk, p, dbias0):
    bf16 = ctx.dtype == torch.bfloat16
    d_qkv = torch.full((B * S, 3 * h * dk), float("nan"), device="cuda", dtype=ctx.dtype)
    dbias = None if dbias0 is None else dbias0.clone()
    delta = torch.full((B, h, S), float("nan"), device="cuda")
    rc = L.lib().arb_attention_backward(L.ptr(qkv), L.ptr(ctx), int(bf16), L.ptr(d_ctx), L.ptr(mask), L.ptr(ext),
                                        L.ptr(smax), L.ptr(ssum), B, S, h, dk, p, SEED, LAYER, L.ptr(d_qkv),
                                        L.ptr(dbias), L.ptr(delta), L.stream_ptr())
    L.check(rc, "arb_attention_backward")
    torch.cuda.synchronize()
    return d_qkv, dbias


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


# ------------------------------------------------------------------------------------------------ checks
def _note(name, err, bound):
    r = (err / bound).nan_to_num(nan=0.0, posinf=float("inf"))
    worst = float(r.max()) if r.numel() else 0.0
    RATIOS[name] = max(RATIOS.get(name, 0.0), worst * TAU)
    return worst


def check(name, got, ref, comp, bf16=False):
    """Elementwise: |got - ref| <= TAU * comp (+ FLOOR); NaN exactly where the reference is NaN.  bf16: got lies
    between the bf16 roundings of ref -/+ the bound and nearly always equals the rounding of ref."""
    got = got.double()
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), f"{name}: NaN at {torch.nonzero(torch.isnan(got) != nan)[:4].tolist()}"
    got, ref, bound = got[~nan], ref[~nan], TAU * comp[~nan] + FLOOR
    err = (got - ref).abs()
    if not bf16:
        worst = _note(name, err, bound)
        bad = ~(err <= bound)
        assert not bad.any(), f"{name}: {int(bad.sum())} elements out of bound, worst error / bound {worst:.3g}"
        return
    lo = (ref - bound).float().bfloat16().double()
    hi = (ref + bound).float().bfloat16().double()
    out = ~((got >= lo) & (got <= hi))
    assert not out.any(), f"{name}: {int(out.sum())} bf16 elements beyond the rounding of ref -/+ bound"
    live = ref != 0
    exact = (got[live] == ref[live].float().bfloat16().double()).double().mean()
    assert exact >= 0.8, f"{name}: only {float(exact):.3f} of the bf16 elements are the rounding of the reference"


def check_forward(tag, R, ctx, smax, ssum, B, S, h, dk):
    bf16 = ctx.dtype == torch.bfloat16
    check(f"{tag} O", heads(ctx, B, S, h, dk), R["O"], R["O_b"], bf16)
    fin = torch.isfinite(R["max"])
    assert torch.equal(smax[~fin].double(), R["max"][~fin]), f"{tag}: row max of a row without keys"
    assert torch.equal(ssum[~fin].double(), R["sum"][~fin]), f"{tag}: row sum of a row without keys"
    check(f"{tag} stat_max", smax[fin], R["max"][fin], R["max_b"][fin])
    # fp32 sum of up to S unrounded probabilities (ex2.approx: 2^-22 each), all scaled by the error of the row max
    sum_b = R["sum"] * (S * 2.0 ** -24 + 2.0 ** -21 + R["scale"] * R["max_b"])
    check(f"{tag} stat_sum", ssum[fin], R["sum"][fin], sum_b[fin])


def colsum_and_bound(d_qkv, dbias0):
    """dbias0 + the column sums of the stored d qkv, and the error bound of adding its rows in fp32 in any order."""
    gd = d_qkv.double()
    rows = gd.shape[0]
    return dbias0.double() + gd.sum(0), 2.0 ** -24 * (rows + 8) * (gd.abs().sum(0) + dbias0.double().abs())


def check_backward(tag, Rb, d_qkv, dbias, dbias0, gext, B, S, h, dk):
    bf16 = d_qkv.dtype == torch.bfloat16
    g = d_qkv.view(B, S, 3, h, dk)
    for i, name in enumerate(("dQ", "dK", "dV")):
        check(f"{tag} {name}", g[:, :, i].permute(0, 2, 1, 3), Rb[name], Rb[name + "_b"], bf16)
    beyond = torch.arange(S, device="cuda")[None, :] >= torch.as_tensor(gext, device="cuda")[:, None]
    z = g.float()[beyond]
    assert torch.equal(z.view(torch.int32), torch.zeros_like(z).view(torch.int32)), \
        f"{tag}: rows at or beyond the backward extent are not +0"
    if dbias is None:
        return
    # the kernels' own stored values, summed: checks the columns (dQ | dK | dV, head-major) and the accumulation
    want, acc_b = colsum_and_bound(d_qkv, dbias0)
    check(f"{tag} dbias/own", dbias, want, acc_b / TAU)
    if not bf16:
        ref = torch.cat([Rb[n].sum((0, 2)).reshape(-1) for n in ("dQ", "dK", "dV")])
        comp = torch.cat([Rb[n + "_b"].sum((0, 2)).reshape(-1) for n in ("dQ", "dK", "dV")])
        check(f"{tag} dbias", dbias - dbias0, ref, comp + acc_b / TAU)


def fwd_case(L, extents, S, h, dk, p, bf16=False, seed=1, mode="rne"):
    B = len(extents)
    qkv, mask, ext = make_inputs(extents, S, h, dk, seed)
    D = drop_masks(range(B), B, h, S, p) if p > 0 else None
    R = reference(qkv, mask, B, S, h, dk, D, mode)
    return qkv, mask, ext, R


# ------------------------------------------------------------------------------------------------ tests
FWD = [(dk, S, p) for dk in (16, 32, 64) for S in (256, 240, 129, 37) for p in (0.0, 0.1)]


@pytest.mark.parametrize("dk,S,p", FWD, ids=[f"dk{dk}-S{S}-p{p}" for dk, S, p in FWD])
def test_forward_matches_fp64_reference(lib, dk, S, p):
    ex = extents_for(S)
    B, h = len(ex), 2
    qkv, mask, ext, R = fwd_case(lib, ex, S, h, dk, p, seed=dk * 1000 + S)
    out = run_fwd(lib, qkv, mask, ext, B, S, h, dk, p)
    again = run_fwd(lib, qkv, mask, ext, B, S, h, dk, p)
    assert all(same_bits(a, b) for a, b in zip(out, again)), "two runs differ"
    check_forward(f"fwd dk{dk} S{S} p{p}", R, *out, B, S, h, dk)


BWD = [(dk, S, p) for dk in (16, 32) for S in (256, 240, 129, 37) for p in (0.0, 0.1, 0.3)]


def bwd_case(L, extents, S, h, dk, p, seed, bf16=False, mode="rne", dbias=True, gext=None):
    """Reference forward + backward for a case; the backward reads the reference's statistics and context (so a wrong
    forward cannot hide a wrong backward).  By default every third slate gets d ctx rows past its key extent."""
    B, d = len(extents), h * dk
    qkv, mask, ext, R = fwd_case(L, extents, S, h, dk, p, seed=seed, mode=mode)
    if gext is None:
        gext = [min(S, e + 3) if b % 3 == 1 else e for b, e in enumerate(extents)]
    d_ctx = make_dctx(gext, S, d, seed + 1)
    o = R["O"].permute(0, 2, 1, 3).reshape(B * S, d).float()
    ctx = o.bfloat16() if bf16 else o
    Rb = reference_bwd(R, d_ctx, ctx, B, S, h, dk)
    gx = torch.tensor(gext, dtype=torch.int32, device="cuda")
    db0 = torch.randn(3 * d, generator=torch.Generator().manual_seed(seed + 2)).cuda() if dbias else None
    args = (qkv, ctx, d_ctx, mask, gx, R["max"].float(), R["sum"].float(), B, S, h, dk, p, db0)
    return args, Rb, gext


@pytest.mark.parametrize("dk,S,p", BWD, ids=[f"dk{dk}-S{S}-p{p}" for dk, S, p in BWD])
def test_backward_matches_fp64_reference(lib, dk, S, p):
    ex = extents_for(S)
    B, h = len(ex), 2
    args, Rb, gext = bwd_case(lib, ex, S, h, dk, p, seed=dk * 1000 + S + 7)
    d_qkv, dbias = run_bwd(lib, *args)
    d2, b2 = run_bwd(lib, *args)
    assert same_bits(d_qkv, d2) and same_bits(dbias, b2), "two runs differ"
    check_backward(f"bwd dk{dk} S{S} p{p}", Rb, d_qkv, dbias, args[-1], gext, B, S, h, dk)


BF16 = [(dk, S, p) for dk in (16, 32) for S in (240, 37) for p in (0.0, 0.1)]


@pytest.mark.parametrize("dk,S,p", BF16, ids=[f"dk{dk}-S{S}-p{p}" for dk, S, p in BF16])
def test_bf16_context_and_gradients(lib, dk, S, p):
    ex = extents_for(S)
    B, h = len(ex), 2
    qkv, mask, ext, R = fwd_case(lib, ex, S, h, dk, p, seed=dk * 100 + S)
    out = run_fwd(lib, qkv, mask, ext, B, S, h, dk, p, bf16=True)
    assert all(same_bits(a, b) for a, b in zip(out, run_fwd(lib, qkv, mask, ext, B, S, h, dk, p, bf16=True)))
    check_forward(f"bf16 fwd dk{dk} S{S}", R, *out, B, S, h, dk)
    args, Rb, gext = bwd_case(lib, ex, S, h, dk, p, seed=dk * 100 + S + 1, bf16=True)
    d_qkv, dbias = run_bwd(lib, *args)
    d2, b2 = run_bwd(lib, *args)
    assert same_bits(d_qkv, d2) and same_bits(dbias, b2), "two runs differ"
    check_backward(f"bf16 bwd dk{dk} S{S}", Rb, d_qkv, dbias, args[-1], gext, B, S, h, dk)


def test_all_padded_slate(lib):
    """Dense layout (DESIGN.md section 5): a slate without real items gets NaN context rows, as the reference, with
    row max -inf and row sum 0; its attention gradients are exactly zero.  Its neighbours are unaffected."""
    S, h, dk = 37, 2, 32
    ex = [37, 1, 20]
    B = len(ex)
    qkv, mask, _, R = fwd_case(lib, ex, S, h, dk, 0.0, seed=5)
    mask[1] = 1
    R = reference(qkv, mask, B, S, h, dk, None)
    ext = torch.tensor([37, 0, 20], dtype=torch.int32, device="cuda")
    ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, dk, 0.0)
    assert torch.isnan(ctx.view(B, S, -1)[1]).all()
    assert (smax[1] == float("-inf")).all() and (ssum[1] == 0).all()
    check_forward("all-padded fwd", R, ctx, smax, ssum, B, S, h, dk)
    # backward from the forward's own outputs; the empty slate has extent 0 and a zero d ctx
    gext = [37, 0, 20]
    d_ctx = make_dctx(gext, S, h * dk, 6)
    Rb = reference_bwd(R, d_ctx, ctx, B, S, h, dk)
    d_qkv, _ = run_bwd(lib, qkv, ctx, d_ctx, mask, ext, smax, ssum, B, S, h, dk, 0.0, None)
    g = d_qkv.view(B, S, 3 * h * dk)
    assert torch.equal(bits(g[1]), torch.zeros_like(bits(g[1]))), "gradients of the all-padded slate are not +0"
    keep = torch.tensor([0, 2], device="cuda")
    sub = {k: v[keep] for k, v in Rb.items()}
    check_backward("all-padded bwd", sub, d_qkv.view(B, S, -1)[keep].reshape(2 * S, -1), None, None, [37, 20],
                   2, S, h, dk)


@pytest.mark.parametrize("dk,S", [(16, 129), (32, 256), (64, 240), (32, 37)])
def test_null_extent_gives_the_same_bits(lib, dk, S):
    """Without extents the kernels run every key and query; the work the extents skip adds exact zeros (probability 0
    for a masked key, zero d ctx rows), so context, statistics, gradients and bias gradient are bit-identical."""
    ex = extents_for(S)
    B, h = len(ex), 2
    qkv, mask, ext, _ = fwd_case(lib, ex, S, h, dk, 0.1, seed=dk + S)
    a = run_fwd(lib, qkv, mask, ext, B, S, h, dk, 0.1)
    b = run_fwd(lib, qkv, mask, None, B, S, h, dk, 0.1)
    assert all(same_bits(x, y) for x, y in zip(a, b))
    if dk > 32:
        return
    args, _, _ = bwd_case(lib, ex, S, h, dk, 0.1, seed=dk + S)
    ga, ba = run_bwd(lib, *args)
    args = args[:4] + (None,) + args[5:]
    gb, bb = run_bwd(lib, *args)
    assert same_bits(ga, gb) and same_bits(ba, bb)


def _pool_extents(n_sm, rounds, cycle):
    """h = 1: CTA c runs items c, c + n_sm, ...; round r of CTA c gets cycle[(r + c % 3) % len(cycle)]."""
    return [cycle[(r + c % 3) % len(cycle)] for r in range(rounds) for c in range(n_sm)]


def _sample(n_sm, rounds, ctas=(0, 1, 5)):
    return [r * n_sm + c for c in ctas for r in range(rounds)]


def test_forward_pool_alternates_between_fitting_and_not(lib):
    """dk = 64 at S = 256: the operand pool holds one full item; two items fit side by side only when both extents are
    small, so consecutive items of a CTA alternate between prefetching beside the current item and waiting for it."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    S, h, dk, rounds = 256, 1, 64, 6
    ex = _pool_extents(n_sm, rounds, [256, 16, 33, 1, 200, 17, 64, 129])
    B = len(ex)
    qkv, mask, ext = make_inputs(ex, S, h, dk, seed=21)
    out = run_fwd(lib, qkv, mask, ext, B, S, h, dk, 0.1)
    idx = _sample(n_sm, rounds)
    sl = torch.tensor(idx, device="cuda")
    R = reference(qkv.view(B, S, -1)[sl].reshape(len(idx) * S, -1), mask[sl], len(idx), S, h, dk,
                  drop_masks(idx, B, h, S, 0.1))
    check_forward("fwd pool", R, out[0].view(B, S, -1)[sl].reshape(len(idx) * S, -1), out[1][sl], out[2][sl],
                  len(idx), S, h, dk)
    assert torch.isfinite(out[0]).all()


def test_backward_schedules_against_reference_and_each_other(lib):
    """The backward's pool holds 352 rows: consecutive items alternate between fitting side by side (prefetch) and
    not.  Persistent (one CTA per SM) and one CTA per item both match the reference and give the same dQ, dK, dV bits;
    the bias gradient is summed over a different number of CTA slots, so it agrees to fp32 summation order only."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    S, h, dk, rounds = 256, 1, 32, 6
    ex = _pool_extents(n_sm, rounds, [256, 240, 17, 200, 100, 256, 1, 129])
    B = len(ex)
    qkv, mask, ext = make_inputs(ex, S, h, dk, seed=22)
    idx = _sample(n_sm, rounds)
    sl = torch.tensor(idx, device="cuda")
    Rq = reference(qkv.view(B, S, -1)[sl].reshape(len(idx) * S, -1), mask[sl], len(idx), S, h, dk,
                   drop_masks(idx, B, h, S, 0.1))
    # statistics and context of the kernels' own forward, d ctx on every real row plus a few past the extent
    ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, dk, 0.1)
    gext = [min(S, e + (b % 2)) for b, e in enumerate(ex)]
    d_ctx = make_dctx(gext, S, h * dk, 23)
    gx = torch.tensor(gext, dtype=torch.int32, device="cuda")
    db0 = torch.zeros(3 * h * dk, device="cuda")
    outs = {}
    try:
        for pers in (1, 0):
            lib.lib().arb_set_attention_bwd_persistent(pers)
            outs[pers] = run_bwd(lib, qkv, ctx, d_ctx, mask, gx, smax, ssum, B, S, h, dk, 0.1, db0)
    finally:
        lib.lib().arb_set_attention_bwd_persistent(1)
    assert same_bits(outs[0][0], outs[1][0]), "dQ, dK, dV differ between the backward schedules"
    for pers in (1, 0):
        want, acc_b = colsum_and_bound(outs[pers][0], db0)
        check(f"bwd pool persistent={pers} dbias/own", outs[pers][1], want, acc_b / TAU)
    Rb = reference_bwd(Rq, d_ctx.view(B, S, -1)[sl].reshape(len(idx) * S, -1),
                       ctx.view(B, S, -1)[sl].reshape(len(idx) * S, -1), len(idx), S, h, dk)
    for pers in (1, 0):
        g = outs[pers][0].view(B, S, -1)[sl].reshape(len(idx) * S, -1)
        check_backward(f"bwd pool persistent={pers}", Rb, g, None, None, [gext[i] for i in idx], len(idx), S, h, dk)
    beyond = torch.arange(S, device="cuda")[None, :] >= gx[:, None]
    assert (outs[1][0].view(B, S, -1)[beyond] == 0).all() and torch.isfinite(outs[1][0]).all()


@pytest.mark.parametrize("B,h", [(3, 2), (66, 2), (600, 4)], ids=["6-items", "one-wave", "2400-items"])
def test_batch_sizes(lib, B, h):
    """Fewer items than SMs, about one wave, and many items per CTA: a seeded sample of slates against the reference,
    the rest finite with zero gradients past the extents."""
    S, dk, p = 129, 32, 0.1
    g = torch.Generator().manual_seed(B)
    cyc = extents_for(S)
    ex = [cyc[int(i)] for i in torch.randint(0, len(cyc), (B,), generator=g)]
    qkv, mask, ext = make_inputs(ex, S, h, dk, seed=B + 30)
    ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, dk, p)
    gext = [min(S, e + 2) if b % 4 == 0 else e for b, e in enumerate(ex)]
    d_ctx = make_dctx(gext, S, h * dk, B + 31)
    gx = torch.tensor(gext, dtype=torch.int32, device="cuda")
    db0 = torch.zeros(3 * h * dk, device="cuda")
    d_qkv, dbias = run_bwd(lib, qkv, ctx, d_ctx, mask, gx, smax, ssum, B, S, h, dk, p, db0)
    idx = sorted(set(torch.randperm(B, generator=g)[:min(B, 24)].tolist()))
    sl = torch.tensor(idx, device="cuda")
    n = len(idx)
    R = reference(qkv.view(B, S, -1)[sl].reshape(n * S, -1), mask[sl], n, S, h, dk, drop_masks(idx, B, h, S, p))
    check_forward(f"fwd B{B}", R, ctx.view(B, S, -1)[sl].reshape(n * S, -1), smax[sl], ssum[sl], n, S, h, dk)
    Rb = reference_bwd(R, d_ctx.view(B, S, -1)[sl].reshape(n * S, -1), ctx.view(B, S, -1)[sl].reshape(n * S, -1),
                       n, S, h, dk)
    check_backward(f"bwd B{B}", Rb, d_qkv.view(B, S, -1)[sl].reshape(n * S, -1), None, None, [gext[i] for i in idx],
                   n, S, h, dk)
    assert torch.isfinite(ctx).all() and torch.isfinite(d_qkv).all() and torch.isfinite(dbias).all()
    beyond = torch.arange(S, device="cuda")[None, :] >= gx[:, None]
    assert (d_qkv.view(B, S, -1)[beyond] == 0).all()
    want, acc_b = colsum_and_bound(d_qkv, db0)
    check(f"bwd B{B} dbias/own", dbias, want, acc_b / TAU)


def test_tf32_operand_rounding_mode(lib):
    """Rounding on load (default): the kernels agree with the nearest-even emulation better than with truncation;
    arb_set_tf32_round_on_load(0): the reverse, and within the elementwise bounds of the truncation emulation."""
    S, h, dk, p = 129, 2, 32, 0.0
    ex = extents_for(S)
    B = len(ex)
    errs = {}
    try:
        for rnd in (1, 0):
            lib.lib().arb_set_tf32_round_on_load(rnd)
            # the backward reads statistics and context of the emulation of its own operand rounding
            args, _, gext = bwd_case(lib, ex, S, h, dk, p, seed=77, mode="rne" if rnd else "trunc")
            qkv, mask = args[0], args[3]
            ctx, smax, ssum = run_fwd(lib, qkv, mask, args[4], B, S, h, dk, p)
            d_qkv, _ = run_bwd(lib, *args)
            for mode in ("rne", "rna", "trunc"):
                R = reference(qkv, mask, B, S, h, dk, None, mode)
                Rb = reference_bwd(R, args[2], args[1], B, S, h, dk)
                gq = d_qkv.view(B, S, 3, h, dk)[:, :, 0].permute(0, 2, 1, 3)
                errs[rnd, mode] = (float((heads(ctx, B, S, h, dk) - R["O"]).abs().sum()),
                                   float((gq - Rb["dQ"]).abs().sum()))
                if (rnd, mode) in ((1, "rne"), (0, "trunc")):
                    check_forward(f"round={rnd} fwd", R, ctx, smax, ssum, B, S, h, dk)
                    check_backward(f"round={rnd} bwd", Rb, d_qkv, None, None, gext, B, S, h, dk)
    finally:
        lib.lib().arb_set_tf32_round_on_load(1)
    for i in range(2):
        assert errs[1, "rne"][i] < errs[1, "trunc"][i] and errs[1, "rna"][i] < errs[1, "trunc"][i], errs
        assert errs[0, "trunc"][i] < errs[0, "rna"][i] and errs[0, "trunc"][i] < errs[0, "rne"][i], errs


def test_host_dropout_restatement_matches_mask_tensor():
    """The per-slate mask generator above keeps and drops what tests/dropout_masks.mask_tensor (the scorer tests'
    restatement) does, for every slate and for a subset."""
    B, h, S, p = 3, 2, 37, 0.3
    full = mask_tensor((B, h, S, S), SEED, LAYER, SITE_ATTN_P, p).double().cuda()
    assert 0.25 < float((full == 0).double().mean()) < 0.35
    for sl, want in (([0, 1, 2], full), ([2], full[2:])):
        got = drop_masks(sl, B, h, S, p)
        assert torch.equal(got == 0, want == 0) and torch.allclose(got, want, rtol=1e-6, atol=0)
