"""The SIMT row kernels of the scorer (csrc/scorer_kernels.cu: LayerNorm forward / backward, final norm + head forward /
backward, the multi-output head, the bias column sums and the unfused key-masked softmax) against a plain fp64
restatement of the same operations, element by element, through the arb_layernorm_* / arb_head_* / arb_column_sums /
arb_softmax_* entry points -- the scorer's own launchers, so that the steps per warp, the row layout (LPR lanes per row,
NJ float4 per lane) and the reduction slots are the ones the scorer gets for the same row count.

Reference, in float64 on the fp32 inputs: the reference's LayerNorm a (x - mean) / (std_unbiased + eps) + b
(transformer.py:73-81) and its analytic gradient, nn.LayerNorm (biased variance, eps under the root) in torch mode,
act(w . LN(x) + b) with and without the norm, the multi-output head, column sums, the key-masked row softmax and
dS = P (dP - sum P dP).  The backward references take the saved statistics (the fp32 roundings of the reference's)
as given, as the kernels do.  A constant row (std = 0) is pinned to the kernels' convention, stated analytically:
y = b bit for bit, and the std term of the backward is 0 (the reference's autograd gives NaN there: d std / dx = 0/0).
Dropout masks are tests/dropout_masks.py's restatement, evaluated on the device (keep_mask; checked against mask_tensor).

Bound, per element: tau times an absolute-value bound built from the kernel's own summation structure.  A row sum
has depth 4 NJ (a lane's sequential terms) + log2(LPR) (shuffle steps); a column sum over the rows of a launch has
depth (rows per lane) + log2(32 / LPR) (the row-group fold) + 8 (the block's warps) + 16 per DetParts level + 1 (the
accumulation); each depth is multiplied by 2^-24 and by the sum of the absolute values of its terms, plus one rounding
for the reciprocal and for each product.  A variance takes the mean's error squared (its first-order term cancels), so
rows with |mean| / std up to 1e3 keep a relative bound near depth * 2^-24 on the variance; the mean's own error
enters each output through |a| r dm.  Calibration on an H100 80GB HBM3 (power limit 700 W): the worst error / bound
per output kind is printed at the end of the module (RATIOS), TAU = 1: LayerNorm dx_masked 0.87, head dx 0.75,
softmax P 0.52, LayerNorm dx 0.49, LayerNorm std 0.42, softmax dS 0.35, multi-output dxf 0.32, multi-output score 0.31,
head score 0.26, LayerNorm y 0.24, every column sum below 0.16.

Exact properties (no tolerance): outputs are pre-filled with NaN, so a row no kernel writes fails, and rows at or
beyond rows_dev and destinations with rowmap < 0 must still hold it; repeat runs give the same bits; a row's outputs do
not depend on the launch size (the same rows inside a launch below 2^17 rows and inside one of 2^17 + 37 / + 38
rows, where the forward walks 4 steps per warp with the next step's loads in flight and the backward takes 32 rows per
warp instead of 8); row-mapped calls equal the plain call scattered / gathered through the row map; y16 / dy16_out
are the nearest-even bf16 of the fp32 outputs of the same call; dy16_in gives the bits fp32 dy with the same values
gives; dx_masked is dx times the regenerated mask; gradient buffers end up holding prefill + the gradient.

Planted rows: the first and last row of the launch, of each warp's rows and so of each block carry a 10^3 times larger
dy / dscore; dropping one of them from a column sum, or adding it twice, moves the sum far outside its bound."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests.dropout_masks import SITE_ATTN_P, SITE_FC, SITE_FFN_OUT, mask_tensor

pytestmark = pytest.mark.gpu

TAU = 1.0
U = 2.0 ** -24
FLOOR = 1e-37
SEED = 0x9E3779B97F4A7C15
LAYER = 2
BIG = 1 << 17             # r_fwd_steps / r_bwd_rows_per_warp: the large-launch path from here on
ACT_NONE, ACT_TANH, ACT_SIGMOID, ACT_RELU = 0, 1, 2, 3
ARB_E_UNSUPPORTED = -2
WIDTHS = [4, 8, 32, 124, 128, 132, 200, 256, 260, 300, 508, 512, 516, 1000, 1024]
RATIOS = {}               # worst error / bound per output kind (printed; the calibration of TAU)
DEV = "cuda"


@pytest.fixture(scope="module")
def lib():
    from allrank_b200 import _lib
    p, i, f, u, q = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float, ctypes.c_uint64, ctypes.c_int64
    _lib.register("arb_layernorm_forward", i, [p, p, p, f, i, q, i, p, p, p, p, p, p, p])
    _lib.register("arb_layernorm_backward", i, [p, p, p, p, p, p, f, i, p, q, i, p, p, p, p, p, p, f, u, i, i, p, p, p])
    _lib.register("arb_head_forward", i, [p, p, p, f, p, p, i, i, q, i, p, p, p, p, p, p])
    _lib.register("arb_head_backward", i, [p, p, p, p, p, p, p, f, p, i, i, q, i, p, p, p, p, p, p, p, p, f, u, i, i,
                                           p, p, p])
    _lib.register("arb_head_multi_forward", i, [p, p, p, i, q, i, i, p, p])
    _lib.register("arb_head_multi_backward", i, [p, p, p, p, i, q, i, i, p, p, p, p, p, f, u, i, i, p])
    _lib.register("arb_column_sums", i, [p, q, i, q, p, p])
    _lib.register("arb_softmax_forward", i, [p, p, i, i, i, i, f, u, i, p])
    _lib.register("arb_softmax_backward", i, [p, p, q, i, i, f, u, i, p])
    yield _lib
    for name, worst in sorted(RATIOS.items()):
        print(f"row kernels: worst error / bound of {name}: {worst:.3g}")


# ------------------------------------------------------------------------------------------------ launch geometry
def layout(width):
    """(LPR, NJ) of the LayerNorm and head kernels (with_row_layout)."""
    for cap, lpr, nj in ((128, 8, 4), (256, 16, 4), (512, 32, 4), (1024, 32, 8)):
        if width <= cap:
            return lpr, nj
    raise ValueError(width)


def nv(width):
    """float4 per lane of the one-row-per-warp kernels (ARB_DISPATCH_NV)."""
    return {1: 1, 2: 2, 3: 4, 4: 4}.get((width + 127) // 128, 8)


def det_depth(slots):
    """Depth of DetParts' ordered sum over `slots` block slots: per level 8 slots per warp + the 8-warp fold, then +=."""
    levels = 1
    while slots > 64:
        slots, levels = -(-slots // 64), levels + 1
    return 16 * levels + 1


def row_depth(width):
    lpr, nj = layout(width)
    return 4 * nj + int(math.log2(lpr)) + 1      # lane terms, shuffle steps, the division by the width


def bwd_per_warp(rows):
    return 32 if rows >= BIG else 8


def col_depth(rows, width):
    """Column sums of the LayerNorm / head backward: a lane's rows, the row-group fold, 8 warps, DetParts."""
    lpr, _ = layout(width)
    rw, pw = 32 // lpr, bwd_per_warp(rows)
    return pw // rw + int(math.log2(rw)) + 8 + det_depth(-(-rows // (8 * pw)))


def wb_depth(rows, width):
    """The head's bias gradient: a lane's rows, the 32-lane warp sum, 8 warps, DetParts."""
    lpr, _ = layout(width)
    pw = bwd_per_warp(rows)
    return pw // (32 // lpr) + 5 + 8 + det_depth(-(-rows // (8 * pw)))


def planted(rows):
    """First and last row of the launch and of each warp's rows (so of each block) of the backward."""
    pw = bwd_per_warp(rows)
    r = torch.arange(rows, device=DEV)
    return (r % pw == 0) | (r % pw == pw - 1) | (r == rows - 1)


# ------------------------------------------------------------------------------------------------ inputs
def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def make_x(rows, width, seed):
    """Rows at scales 1e-3 ... 1e3, a third of them shifted so that |mean| / std reaches 1e3, every 13th row zero and
    every 13th (offset 9) exactly 0.5 (constant: the fp32 mean is exact and the std 0)."""
    g = gen(seed)
    x = torch.randn(rows, width, device=DEV, generator=g)
    scale = 10.0 ** (6.0 * torch.rand(rows, 1, device=DEV, generator=g) - 3.0)
    sign = torch.where(torch.rand(rows, 1, device=DEV, generator=g) < 0.5, -1.0, 1.0)
    shift = sign * 10.0 ** (3.0 * torch.rand(rows, 1, device=DEV, generator=g))
    shift = torch.where(torch.rand(rows, 1, device=DEV, generator=g) < 0.35, shift, 0.0)
    x = (x + shift) * scale
    r = torch.arange(rows, device=DEV)
    x[r % 13 == 5] = 0.0
    x[r % 13 == 9] = 0.5
    return x.contiguous()


def const_rows(rows):
    r = torch.arange(rows, device=DEV)
    return (r % 13 == 5) | (r % 13 == 9)


def make_gain(width, seed):
    g = gen(seed)
    return ((1.0 + 0.5 * torch.randn(width, device=DEV, generator=g)).contiguous(),
            (0.5 * torch.randn(width, device=DEV, generator=g)).contiguous())


def make_dy(rows, width, seed, big=1e3):
    dy = torch.randn(rows, width, device=DEV, generator=gen(seed))
    return torch.where(planted(rows)[:, None], dy * big, dy).contiguous()


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device=DEV, dtype=dtype)


def dev_i32(values):
    return torch.tensor(values, dtype=torch.int32, device=DEV)


def make_rowmap(rows, seed):
    """A permutation of rows + 5 destinations with every 7th row mapped nowhere (-1)."""
    n_dest = rows + 5
    rm = torch.randperm(n_dest, generator=torch.Generator().manual_seed(seed))[:rows].to(torch.int32)
    rm[torch.arange(rows) % 7 == 3] = -1
    return rm.to(DEV), n_dest


# ------------------------------------------------------------------------------------------------ dropout masks
def _mul32(h, c):
    """(h * c) mod 2^32 in int64 for 0 <= h, c < 2^32"""
    return ((h & 0xFFFF) * c + ((((h >> 16) * c) & 0xFFFF) << 16)) & 0xFFFFFFFF


def _mix32_t(h):
    h = h ^ (h >> 16)
    h = _mul32(h, 0x85EBCA6B)
    h = h ^ (h >> 13)
    h = _mul32(h, 0xC2B2AE35)
    return h ^ (h >> 16)


def site_scale(p):
    """make_drop_site's scale, computed in fp32 as the kernels get it."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


def keep_mask(r0, r1, width, site, p):
    """drop_keep of rows r0 .. r1 - 1 of a [*, width] site (element row * width + column) on the device: bool."""
    from tests.dropout_masks import _site
    seed, thresh, _ = _site(SEED, LAYER, site, p)
    idx = (torch.arange(r0, r1, device=DEV, dtype=torch.int64)[:, None] * width
           + torch.arange(width, device=DEV, dtype=torch.int64)[None, :])
    h = _mix32_t((idx & 0xFFFFFFFF) ^ int(seed))
    h = _mix32_t((h + (idx >> 32) * 0x9E3779B1 + 0x7F4A7C15) & 0xFFFFFFFF)
    return h >= int(thresh)


def masked(v, r0, width, site, p):
    """v [n, width] fp32 through the kernels' dropout: v * scale where kept (one fp32 product), +0 where dropped."""
    if p == 0:
        return v
    k = keep_mask(r0, r0 + v.shape[0], width, site, p)
    return torch.where(k, v * torch.tensor(site_scale(p), device=DEV), torch.zeros((), device=DEV))


def dmask(r0, r1, width, site, p):
    """The scaled keep mask as float64 (1 when p = 0)."""
    if p == 0:
        return torch.ones((), device=DEV, dtype=torch.float64)
    return keep_mask(r0, r1, width, site, p).double() * site_scale(p)


# ------------------------------------------------------------------------------------------------ references
def ln_ref(x, a, b, eps, torch_mode):
    """LayerNorm forward in fp64 with the bounds of y, mean and the saved std."""
    xd, W = x.double(), x.shape[1]
    a, b = a.double(), b.double()
    m = xd.mean(1, keepdim=True)
    c = xd - m
    ss = (c * c).sum(1, keepdim=True)
    dep = row_depth(W)
    dm = dep * U * xd.abs().sum(1, keepdim=True) / W + U * m.abs()
    err_ss = (dep + 3) * U * (ss + W * dm * dm) + W * dm * dm
    if torch_mode:
        v, err_v = ss / W + eps, err_ss / W + 2 * U * (ss / W + eps)
    else:
        v, err_v = ss / (W - 1), err_ss / (W - 1) + U * ss / (W - 1)
    sd = v.sqrt()
    err_sd = (v + err_v).sqrt() - sd + U * sd
    den = sd if torch_mode else sd + eps
    err_den = err_sd + U * den
    r = 1.0 / den
    err_r = r * r * err_den / (1.0 - (err_den * r).clamp(max=0.5)) + U * r
    y = a * c * r + b
    y_b = a.abs() * (c.abs() * err_r + r * dm) + 4 * U * ((a * c * r).abs() + b.abs())
    return dict(y=y, y_b=y_b, mean=m[:, 0], mean_b=dm[:, 0], sd=sd[:, 0], sd_b=err_sd[:, 0])


def norm_bwd_ref(g, g_b, x, a, m, s, eps, torch_mode):
    """d x of the LayerNorm for the incoming d y = g (fp64, error bound g_b), given the saved mean m and std s
    [rows]: r (g a - mean(g a)) - K (sum_k g_k a_k c_k) c with c = x - m, r = 1 / (s + eps) and K = r^2 / ((W-1) s)
    (K = 0 where s = 0: the kernels' constant-row convention), or r^3 / W in torch mode (eps = 0)."""
    W = x.shape[1]
    a = a.double()
    m, s = m.double()[:, None], s.double()[:, None]
    c = x.double() - m
    r = 1.0 / (s + eps)
    if torch_mode:
        K = r ** 3 / W
    else:
        K = torch.where(s > 0, r * r / ((W - 1) * torch.where(s > 0, s, 1.0)), 0.0)
    dxh = g * a
    A = dxh.abs()
    dx = r * (dxh - dxh.sum(1, keepdim=True) / W) - K * (dxh * c).sum(1, keepdim=True) * c
    def spread(A):      # |d x| of a change A = |d (g a)| of the incoming gradient
        return r * (A + A.sum(1, keepdim=True) / W) + K * (A * c.abs()).sum(1, keepdim=True) * c.abs()
    dx_b = (row_depth(W) + 8) * U * spread(A) + U * dx.abs()
    if torch.is_tensor(g_b):
        dx_b = dx_b + spread(g_b * a.abs())
    return dx, dx_b, c, r


def act_ref(z, act):
    return {ACT_NONE: z, ACT_TANH: torch.tanh(z), ACT_SIGMOID: torch.sigmoid(z), ACT_RELU: z.clamp(min=0)}[act]


def act_grad(out, act):
    """act'(z) from the output, as the kernels take it"""
    return {ACT_NONE: torch.ones_like(out), ACT_TANH: 1 - out * out, ACT_SIGMOID: out * (1 - out),
            ACT_RELU: (out > 0).double()}[act]


def act_bound(zb, s, act):
    lip = {ACT_NONE: 1.0, ACT_TANH: 1.0, ACT_SIGMOID: 0.25, ACT_RELU: 1.0}[act]
    return lip * zb + (4 * U * s.abs() if act in (ACT_TANH, ACT_SIGMOID) else U * s.abs())


def head_ref(x, a, b, eps, w, wb, has_norm, act):
    W = x.shape[1]
    if has_norm:
        R = ln_ref(x, a, b, eps, 0)
        xf, xf_b = R["y"], R["y_b"]
    else:
        R, xf = {}, x.double()
        xf_b = torch.zeros_like(xf)
    wd = w.double()
    z = xf @ wd + float(wb[0])
    zb = (xf_b * wd.abs()).sum(1) + (row_depth(W) + 2) * U * (xf.abs() @ wd.abs() + abs(float(wb[0])))
    s = act_ref(z, act)
    return dict(R, score=s, score_b=act_bound(zb, s, act))


# ------------------------------------------------------------------------------------------------ calls
def call(L, name, *args):
    rc = getattr(L.lib(), name)(*args, L.stream_ptr())
    L.check(rc, name)
    torch.cuda.synchronize()


def ln_fwd(L, x, a, b, eps, tm, rows=None, bf16=False, rows_dev=None, rowmap=None, n_dest=None):
    rows = x.shape[0] if rows is None else rows
    W = x.shape[1]
    y = nan(n_dest or rows, W, dtype=torch.bfloat16 if bf16 else torch.float32)
    mean, sd = nan(rows), nan(rows)
    P = L.ptr
    call(L, "arb_layernorm_forward", P(x), P(a), P(b), eps, tm, rows, W, None if bf16 else P(y), P(y) if bf16 else None,
         P(mean), P(sd), P(rows_dev), P(rowmap))
    return y, mean, sd


def ln_bwd(L, dy, x, a, mean, sd, eps, tm, p=0.0, dres=None, g0=None, bf16_out=False, dy16_in=None, rows_dev=None,
           rowmap=None, site=SITE_FFN_OUT):
    """g0: (grad_a, grad_b, colsum) prefills (copied) or None (not computed)."""
    rows, W = x.shape
    out = dict(dx=nan(rows, W), dx_masked=nan(rows, W) if p > 0 else None,
               dy16=nan(rows, W, dtype=torch.bfloat16) if bf16_out else None)
    ga, gb, cs = (None, None, None) if g0 is None else (t.clone() for t in g0)
    P = L.ptr
    call(L, "arb_layernorm_backward", P(dy), P(dy16_in), P(x), P(a), P(mean), P(sd), 0.0 if tm else eps, tm, P(dres),
         rows, W, P(out["dx"]), P(ga), P(gb), P(out["dx_masked"]), P(out["dy16"]), P(cs), p, SEED, LAYER, site,
         P(rows_dev), P(rowmap))
    out.update(grad_a=ga, grad_b=gb, colsum=cs)
    return out


def head_fwd(L, x, a, b, eps, w, wb, has_norm, act, rows=None, rows_dev=None, rowmap=None, n_dest=None):
    rows = x.shape[0] if rows is None else rows
    score, mean, sd = nan(n_dest or rows), nan(rows), nan(rows)
    P = L.ptr
    call(L, "arb_head_forward", P(x), P(a) if has_norm else None, P(b) if has_norm else None, eps, P(w), P(wb),
         has_norm, act, rows, x.shape[1], P(score), P(mean), P(sd), P(rows_dev), P(rowmap))
    return score, mean, sd


def head_bwd(L, dscore, score, x, a, b, mean, sd, eps, w, has_norm, act, p=0.0, g0=None, bf16_out=False,
             rows_dev=None, rowmap=None):
    """g0: (grad_a, grad_b, grad_w, grad_wb, colsum) prefills (copied)."""
    rows, W = x.shape
    out = dict(dx=nan(rows, W), dx_masked=nan(rows, W) if p > 0 else None,
               dy16=nan(rows, W, dtype=torch.bfloat16) if bf16_out else None)
    ga, gb, gw, gwb, cs = (t.clone() for t in g0)
    P = L.ptr
    call(L, "arb_head_backward", P(dscore), P(score), P(x), P(a) if has_norm else None, P(b) if has_norm else None,
         P(mean) if has_norm else None, P(sd) if has_norm else None, eps, P(w), has_norm, act, rows, W, P(out["dx"]),
         P(ga), P(gb), P(gw), P(gwb), P(out["dx_masked"]), P(out["dy16"]), P(cs), p, SEED, LAYER, SITE_FC,
         P(rows_dev), P(rowmap))
    out.update(grad_a=ga, grad_b=gb, grad_w=gw, grad_wb=gwb, colsum=cs)
    return out


# ------------------------------------------------------------------------------------------------ checks
def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def all_nan(t):
    return bool(torch.isnan(t.float()).all())


def check(name, got, ref, bound):
    """|got - ref| <= TAU * bound element by element; NaN exactly where the reference is NaN."""
    got = got.double()
    isn = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), isn), f"{name}: NaN at {torch.nonzero(torch.isnan(got) != isn)[:4].tolist()}"
    got, ref, bound = got[~isn], ref[~isn], bound.expand_as(isn)[~isn]
    err = (got - ref).abs()
    r = err / (bound + FLOOR)
    worst = float(r.max()) if r.numel() else 0.0
    RATIOS[name] = max(RATIOS.get(name, 0.0), worst)
    bad = ~(err <= TAU * bound + FLOOR)
    if bad.any():
        i = int(torch.nonzero(bad)[0, 0])
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements out of bound, worst error / bound "
                             f"{worst:.3g}; first: got {float(got[i])!r} ref {float(ref[i])!r} bound {float(bound[i])!r}")


def check_colsum(name, got, g0, rows_sum, abs_sum, depth, extra=0.0):
    """g0 + a column sum of depth `depth` (rows_sum / abs_sum: fp64 sum of the terms and of their absolute values;
    extra: the summed error bounds of the terms)."""
    ref = g0.double() + rows_sum
    check(name, got, ref, depth * U * (abs_sum + g0.double().abs()) + extra)


def check_bf16_copy(name, got16, fp32):
    assert same_bits(got16, fp32.bfloat16()), f"{name}: not the nearest-even bf16 of the fp32 output"


# ------------------------------------------------------------------------------------------------ LayerNorm
MODES = [("unbiased", 1e-6), ("unbiased", 0.1), ("torch", 1e-5)]


def row_counts(width):
    """1, 7, 33 and both sides of a block of the forward (8 warps x 32 / LPR rows) and of the backward (64 rows)."""
    lpr, _ = layout(width)
    fb, bb = 8 * (32 // lpr), 64
    return sorted({1, 7, 33, fb - 1, fb + 1, bb - 1, bb + 1, 2 * bb + 3})


def ln_fwd_checks(tag, L, x, a, b, eps, tm, out):
    y, mean, sd = out
    R = ln_ref(x, a, b, eps, tm)
    check("layernorm y", y, R["y"], R["y_b"])
    check("layernorm mean", mean, R["mean"], R["mean_b"])
    check("layernorm std", sd, R["sd"], R["sd_b"])
    cr = const_rows(x.shape[0])
    assert same_bits(y[cr], b.expand(int(cr.sum()), -1)), f"{tag}: a constant row does not give y = b"
    return R


def ln_bwd_checks(tag, rows_all, x, a, m32, s32, eps, tm, dy, dres, p, g0, out, site=SITE_FFN_OUT):
    """out of ln_bwd over the first `rows` rows live (x, dy: those rows)."""
    rows, W = x.shape
    g = dy.double()
    dx, dx_b, c, r = norm_bwd_ref(g, 0.0, x, a, m32, s32, 0.0 if tm else eps, tm)
    if dres is not None:
        dx, dx_b = dx + dres.double(), dx_b + 2 * U * dres.double().abs()
    check("layernorm dx", out["dx"][:rows], dx, dx_b)
    emitted = out["dx"][:rows]
    if p > 0:
        assert same_bits(out["dx_masked"][:rows], masked(out["dx"][:rows], 0, W, site, p)), f"{tag}: dx_masked"
        D = dmask(0, rows, W, site, p)
        check("layernorm dx_masked", out["dx_masked"][:rows], dx * D, dx_b * D)
        emitted = out["dx_masked"][:rows]
    if out["dy16"] is not None:
        check_bf16_copy(f"{tag} dy16_out", out["dy16"][:rows], emitted)
    if g0 is not None:
        cd = col_depth(rows_all, W) + 4
        gcr = g * c * r
        check_colsum("layernorm grad_a", out["grad_a"], g0[0], gcr.sum(0), gcr.abs().sum(0), cd)
        check_colsum("layernorm grad_b", out["grad_b"], g0[1], g.sum(0), g.abs().sum(0), cd)
        e = emitted.double()
        check_colsum("layernorm colsum_out", out["colsum"], g0[2], e.sum(0), e.abs().sum(0), cd)


@pytest.mark.parametrize("mode,eps", MODES, ids=[f"{m}-eps{e:g}" for m, e in MODES])
@pytest.mark.parametrize("width", WIDTHS)
def test_layernorm(lib, width, mode, eps):
    tm = int(mode == "torch")
    counts = row_counts(width)
    N = counts[-1]
    x = make_x(N, width, seed=width * 10 + tm)
    a, b = make_gain(width, seed=width + 1)
    dy = make_dy(N, width, seed=width + 2)
    dres = torch.randn(N, width, device=DEV, generator=gen(width + 3))
    g0 = tuple(torch.randn(width, device=DEV, generator=gen(width + 4 + k)) for k in range(3))
    for i, rows in enumerate(counts):
        tag = f"W{width} {mode} rows {rows}"
        xs = x[:rows].contiguous()
        out = ln_fwd(lib, xs, a, b, eps, tm)
        R = ln_fwd_checks(tag, lib, xs, a, b, eps, tm, out)
        m32, s32 = R["mean"].float(), R["sd"].float()
        p = (0.0, 0.1, 0.3)[i % 3]
        dr = dres[:rows].contiguous() if i % 2 else None
        bo = ln_bwd(lib, dy[:rows].contiguous(), xs, a, m32, s32, eps, tm, p, dr, g0, bf16_out=True)
        ln_bwd_checks(tag, rows, xs, a, m32, s32, eps, tm, dy[:rows], dr, p, g0, bo)
    # at the largest count: repeat runs, bf16 copies, row-mapped calls, live rows below the nominal count
    rows = N
    y, mean, sd = ln_fwd(lib, x, a, b, eps, tm)
    assert all(same_bits(u, v) for u, v in zip((y, mean, sd), ln_fwd(lib, x, a, b, eps, tm))), "two runs differ"
    y16, mean16, sd16 = ln_fwd(lib, x, a, b, eps, tm, bf16=True)
    check_bf16_copy("y16", y16, y)
    assert same_bits(mean16, mean) and same_bits(sd16, sd)
    rm, n_dest = make_rowmap(rows, seed=width)
    ym, meanm, sdm = ln_fwd(lib, x, a, b, eps, tm, rowmap=rm, n_dest=n_dest)
    hit = rm >= 0
    assert same_bits(ym[rm[hit].long()], y[hit]) and same_bits(meanm, mean) and same_bits(sdm, sd)
    untouched = torch.ones(n_dest, dtype=torch.bool, device=DEV)
    untouched[rm[hit].long()] = False
    assert all_nan(ym[untouched]), "a destination without a row was written"
    live = rows - 3
    yl, meanl, sdl = ln_fwd(lib, x, a, b, eps, tm, rows_dev=dev_i32([live]))
    assert same_bits(yl[:live], y[:live]) and same_bits(meanl[:live], mean[:live]) and same_bits(sdl[:live], sd[:live])
    assert all_nan(yl[live:]) and all_nan(meanl[live:]) and all_nan(sdl[live:]), "rows at or beyond rows_dev written"

    R = ln_ref(x, a, b, eps, tm)
    m32, s32 = R["mean"].float(), R["sd"].float()
    full = ln_bwd(lib, dy, x, a, m32, s32, eps, tm, 0.1, dres, g0, bf16_out=True)
    again = ln_bwd(lib, dy, x, a, m32, s32, eps, tm, 0.1, dres, g0, bf16_out=True)
    for k in ("dx", "dx_masked", "dy16", "grad_a", "grad_b", "colsum"):
        assert same_bits(full[k], again[k]), f"two runs differ: {k}"
    # gradients accumulate onto the prefill: prefill + (the gradients computed from zero)
    zero = tuple(torch.zeros(width, device=DEV) for _ in range(3))
    z = ln_bwd(lib, dy, x, a, m32, s32, eps, tm, 0.1, dres, zero)
    for k, i in (("grad_a", 0), ("grad_b", 1), ("colsum", 2)):
        assert same_bits(full[k], g0[i] + z[k]), f"{k} is not prefill + gradient"
    # bf16 dy: the same results as fp32 dy holding the same values
    dy16 = dy.bfloat16()
    f16 = ln_bwd(lib, None, x, a, m32, s32, eps, tm, 0.1, dres, g0, dy16_in=dy16)
    f32 = ln_bwd(lib, dy16.float(), x, a, m32, s32, eps, tm, 0.1, dres, g0)
    for k in ("dx", "dx_masked", "grad_a", "grad_b", "colsum"):
        assert same_bits(f16[k], f32[k]), f"dy16_in: {k}"
    # row-mapped gradient = the plain call on the gathered gradient (rowmap < 0: zero)
    dyd = torch.randn(n_dest, width, device=DEV, generator=gen(width + 9))
    gathered = torch.where(hit[:, None], dyd[rm.clamp(min=0).long()], 0.0)
    fm = ln_bwd(lib, dyd, x, a, m32, s32, eps, tm, 0.3, None, g0, rowmap=rm)
    fp = ln_bwd(lib, gathered, x, a, m32, s32, eps, tm, 0.3, None, g0)
    # (the row-mapped kernel is its own instantiation: at W = 512 the compiler contracts dx's products into FMAs
    # differently, so dx agrees with the plain call to within its bound, not bit for bit)
    for k in ("grad_a", "grad_b"):
        assert same_bits(fm[k], fp[k]), f"row-mapped backward: {k}"
    ln_bwd_checks(f"W{width} row-mapped", rows, x, a, m32, s32, eps, tm, gathered, None, 0.3, g0, fm)
    # live rows: the rows below are the full call's, the rest untouched, the sums over the live rows only
    fl = ln_bwd(lib, dy, x, a, m32, s32, eps, tm, 0.1, dres, g0, bf16_out=True, rows_dev=dev_i32([live]))
    for k in ("dx", "dx_masked", "dy16"):
        assert same_bits(fl[k][:live], full[k][:live]) and all_nan(fl[k][live:]), f"rows_dev: {k}"
    ln_bwd_checks(f"W{width} live", rows, x[:live], a, m32[:live], s32[:live], eps, tm, dy[:live], dres[:live], 0.1,
                  g0, fl)


# ------------------------------------------------------------------------------------------------ final norm + head
def dz_ref(dscore, score, act):
    """dz = dscore act'(z) from the fp32 output and its bound: act' costs two roundings, and 1 - out^2 (tanh) the
    rounding of out^2 on top, absolute where it cancels."""
    ag = act_grad(score.double(), act)
    dz = dscore.double() * ag
    return dz, dscore.double().abs() * (3 * U * ag.abs() + (U if act == ACT_TANH else 0.0))


def head_bwd_ref(dscore, score, x, a, b, m32, s32, eps, w, has_norm, act):
    """dx, its bound, and the per-row terms of the parameter gradients (fp64) of the head backward, with the parts of
    their bounds that dz's error adds (*_e)."""
    dz, dz_b = dz_ref(dscore, score, act)
    wd = w.double()
    gy = dz[:, None] * wd                                 # d loss / d xf
    gy_b = dz_b[:, None] * wd.abs() + U * gy.abs()
    H = dict(dz=dz, dz_e=dz_b)
    if not has_norm:
        xd = x.double()
        return dict(H, dx=gy, dx_b=gy_b, gw=dz[:, None] * xd, gw_a=(dz[:, None] * xd).abs(), gw_e=dz_b[:, None] * xd.abs())
    dx, dx_b, c, r = norm_bwd_ref(gy, gy_b, x, a, m32, s32, eps, 0)
    xh = c * r
    xf = a.double() * xh + b.double()
    xfa = (a.double() * xh).abs() + b.double().abs()
    return dict(H, dx=dx, dx_b=dx_b, gw=dz[:, None] * xf, gw_a=dz.abs()[:, None] * xfa, gw_e=dz_b[:, None] * xfa,
                ga=gy * xh, ga_e=gy_b * xh.abs(), gb=gy, gb_e=gy_b)


def head_bwd_checks(tag, rows_all, x, a, b, m32, s32, eps, w, has_norm, act, dscore, score, p, g0, out):
    rows, W = x.shape
    H = head_bwd_ref(dscore, score, x, a, b, m32, s32, eps, w, has_norm, act)
    check("head dx", out["dx"][:rows], H["dx"], H["dx_b"])
    emitted = out["dx"][:rows]
    if p > 0:
        assert same_bits(out["dx_masked"][:rows], masked(out["dx"][:rows], 0, W, SITE_FC, p)), f"{tag}: dx_masked"
        emitted = out["dx_masked"][:rows]
    if out["dy16"] is not None:
        check_bf16_copy(f"{tag} dy16_out", out["dy16"][:rows], emitted)
    cd = col_depth(rows_all, W) + 8
    check_colsum("head grad_w", out["grad_w"], g0[2], H["gw"].sum(0), H["gw_a"].sum(0), cd, H["gw_e"].sum(0))
    dz = H["dz"]
    check_colsum("head grad_wb", out["grad_wb"], g0[3], dz.sum(0, keepdim=True), dz.abs().sum(0, keepdim=True),
                 wb_depth(rows_all, W) + 4, H["dz_e"].sum(0, keepdim=True))
    e = emitted.double()
    check_colsum("head colsum_out", out["colsum"], g0[4], e.sum(0), e.abs().sum(0), cd)
    if has_norm:
        check_colsum("head grad_a", out["grad_a"], g0[0], H["ga"].sum(0), H["ga"].abs().sum(0), cd, H["ga_e"].sum(0))
        check_colsum("head grad_b", out["grad_b"], g0[1], H["gb"].sum(0), H["gb"].abs().sum(0), cd, H["gb_e"].sum(0))
    else:
        assert same_bits(out["grad_a"], g0[0]) and same_bits(out["grad_b"], g0[1]), "FC-only head wrote norm grads"


def head_inputs(width, rows, seed):
    x = make_x(rows, width, seed)
    a, b = make_gain(width, seed + 1)
    w = (torch.randn(width, device=DEV, generator=gen(seed + 2)) / math.sqrt(width)).contiguous()
    wb = torch.tensor([0.25], device=DEV)
    dscore = torch.randn(rows, device=DEV, generator=gen(seed + 3))
    dscore = torch.where(planted(rows), dscore * 1e3, dscore)
    g0 = tuple(torch.randn(n, device=DEV, generator=gen(seed + 4 + k)) for k, n in enumerate((width,) * 3 + (1, width)))
    return x, a, b, w, wb, dscore, g0


ACTS = [ACT_NONE, ACT_TANH, ACT_SIGMOID, ACT_RELU]


@pytest.mark.parametrize("act", ACTS, ids=["identity", "tanh", "sigmoid", "relu"])
@pytest.mark.parametrize("width", WIDTHS)
def test_head(lib, width, act):
    eps = 1e-6 if act % 2 else 0.1
    counts = row_counts(width)
    N = counts[-1]
    x, a, b, w, wb, dscore, g0 = head_inputs(width, N, seed=width * 7 + act)
    for has_norm in (1, 0):
        for i, rows in enumerate(counts):
            tag = f"head W{width} act{act} norm{has_norm} rows {rows}"
            xs = x[:rows].contiguous()
            score, mean, sd = head_fwd(lib, xs, a, b, eps, w, wb, has_norm, act)
            H = head_ref(xs, a, b, eps, w, wb, has_norm, act)
            check("head score", score, H["score"], H["score_b"])
            if has_norm:
                check("head mean", mean, H["mean"], H["mean_b"])
                check("head std", sd, H["sd"], H["sd_b"])
                m32, s32 = H["mean"].float(), H["sd"].float()
            else:
                assert all_nan(mean) and all_nan(sd), f"{tag}: FC-only head wrote statistics"
                m32 = s32 = None
            s32c = H["score"].float()
            p = (0.0, 0.1, 0.3)[i % 3]
            out = head_bwd(lib, dscore[:rows].contiguous(), s32c, xs, a, b, m32, s32, eps, w, has_norm, act, p, g0,
                           bf16_out=True)
            head_bwd_checks(tag, rows, xs, a, b, m32, s32, eps, w, has_norm, act, dscore[:rows], s32c, p, g0, out)
    # at the largest count: repeat runs, row-mapped scores, live rows
    rows, has_norm = N, 1
    score, mean, sd = head_fwd(lib, x, a, b, eps, w, wb, has_norm, act)
    assert all(same_bits(u, v) for u, v in zip((score, mean, sd), head_fwd(lib, x, a, b, eps, w, wb, has_norm, act)))
    rm, n_dest = make_rowmap(rows, seed=width + act)
    hit = rm >= 0
    sm, meanm, sdm = head_fwd(lib, x, a, b, eps, w, wb, has_norm, act, rowmap=rm, n_dest=n_dest)
    assert same_bits(sm[rm[hit].long()], score[hit]) and same_bits(meanm, mean) and same_bits(sdm, sd)
    untouched = torch.ones(n_dest, dtype=torch.bool, device=DEV)
    untouched[rm[hit].long()] = False
    assert all_nan(sm[untouched]), "a score without a row was written"
    live = rows - 3
    sl, meanl, sdl = head_fwd(lib, x, a, b, eps, w, wb, has_norm, act, rows_dev=dev_i32([live]))
    assert same_bits(sl[:live], score[:live]) and all_nan(sl[live:]) and all_nan(meanl[live:])
    H = head_ref(x, a, b, eps, w, wb, has_norm, act)
    m32, s32, sc = H["mean"].float(), H["sd"].float(), H["score"].float()
    full = head_bwd(lib, dscore, sc, x, a, b, m32, s32, eps, w, has_norm, act, 0.1, g0)
    again = head_bwd(lib, dscore, sc, x, a, b, m32, s32, eps, w, has_norm, act, 0.1, g0)
    for k in ("dx", "dx_masked", "grad_a", "grad_b", "grad_w", "grad_wb", "colsum"):
        assert same_bits(full[k], again[k]), f"two runs differ: {k}"
    zero = tuple(torch.zeros_like(t) for t in g0)
    z = head_bwd(lib, dscore, sc, x, a, b, m32, s32, eps, w, has_norm, act, 0.1, zero)
    for i, k in enumerate(("grad_a", "grad_b", "grad_w", "grad_wb", "colsum")):
        assert same_bits(full[k], g0[i] + z[k]), f"{k} is not prefill + gradient"
    ds_dest = torch.randn(n_dest, device=DEV, generator=gen(width + 11))
    sc_dest = torch.rand(n_dest, device=DEV, generator=gen(width + 12))
    fm = head_bwd(lib, ds_dest, sc_dest, x, a, b, m32, s32, eps, w, has_norm, act, 0.1, g0, rowmap=rm)
    idx = rm.clamp(min=0).long()
    fp = head_bwd(lib, torch.where(hit, ds_dest[idx], 0.0), torch.where(hit, sc_dest[idx], 0.0), x, a, b, m32, s32,
                  eps, w, has_norm, act, 0.1, g0)
    for k in ("dx", "dx_masked", "grad_a", "grad_b", "grad_w", "grad_wb", "colsum"):
        assert same_bits(fm[k], fp[k]), f"row-mapped head backward: {k}"
    fl = head_bwd(lib, dscore, sc, x, a, b, m32, s32, eps, w, has_norm, act, 0.1, g0, rows_dev=dev_i32([live]))
    for k in ("dx", "dx_masked"):
        assert same_bits(fl[k][:live], full[k][:live]) and all_nan(fl[k][live:]), f"rows_dev: {k}"
    head_bwd_checks(f"head W{width} live", rows, x[:live], a, b, m32[:live], s32[:live], eps, w, has_norm, act,
                    dscore[:live], sc[:live], 0.1, g0, fl)


# ------------------------------------------------------------------------------------------------ large launches
LARGE = [(w, t) for w in (124, 256, 300, 1000) for t in (37, 38)]
CHUNK = 1 << 14


@pytest.mark.parametrize("width,tail", LARGE, ids=[f"W{w}-2^17+{t}" for w, t in LARGE])
def test_large_launch(lib, width, tail):
    """2^17 + 37 / + 38 rows: 4 forward steps per warp with the next step's loads in flight (the launch's last row is a
    prefetch: +37 in the 8- and 16-lane layouts, +38 in the 32-lane ones), 32 backward rows per warp.  Every element
    against the reference (in chunks of rows); the first and last 4099 rows launched alone give the same bits; a
    nominal launch of this size with 100 003 live rows leaves the rest untouched."""
    rows, eps, p, act, small = BIG + tail, 1e-6, 0.1, ACT_SIGMOID, 4099
    x = make_x(rows, width, seed=width + tail)
    a, b = make_gain(width, seed=width)
    # LayerNorm forward
    y, mean, sd = ln_fwd(lib, x, a, b, eps, 0)
    m32, s32 = torch.empty(rows, device=DEV), torch.empty(rows, device=DEV)
    for r0 in range(0, rows, CHUNK):
        sl = slice(r0, min(rows, r0 + CHUNK))
        R = ln_ref(x[sl], a, b, eps, 0)
        check("layernorm y", y[sl], R["y"], R["y_b"])
        check("layernorm mean", mean[sl], R["mean"], R["mean_b"])
        check("layernorm std", sd[sl], R["sd"], R["sd_b"])
        m32[sl], s32[sl] = R["mean"].float(), R["sd"].float()
    for sl in (slice(0, small), slice(rows - small, rows)):
        o = ln_fwd(lib, x[sl].contiguous(), a, b, eps, 0)
        assert all(same_bits(u, v[sl]) for u, v in zip(o, (y, mean, sd))), f"forward rows {sl} depend on the launch"
    live = 100003
    if tail == 37:
        o = ln_fwd(lib, x, a, b, eps, 0, rows_dev=dev_i32([live]))
        assert all(same_bits(u[:live], v[:live]) and all_nan(u[live:]) for u, v in zip(o, (y, mean, sd)))
    del y, o
    # LayerNorm backward, with planted rows
    dy = make_dy(rows, width, seed=width + tail + 1)
    g0 = tuple(torch.randn(width, device=DEV, generator=gen(width + k)) for k in range(3))
    out = ln_bwd(lib, dy, x, a, m32, s32, eps, 0, p, None, g0, bf16_out=True)
    acc = {k: torch.zeros(width, device=DEV, dtype=torch.float64) for k in ("a", "aa", "b", "ba", "c", "ca")}
    for r0 in range(0, rows, CHUNK):
        sl = slice(r0, min(rows, r0 + CHUNK))
        g = dy[sl].double()
        dx, dx_b, c, r = norm_bwd_ref(g, 0.0, x[sl], a, m32[sl], s32[sl], eps, 0)
        check("layernorm dx", out["dx"][sl], dx, dx_b)
        assert same_bits(out["dx_masked"][sl], masked(out["dx"][sl], r0, width, SITE_FFN_OUT, p)), "dx_masked"
        check_bf16_copy("dy16_out", out["dy16"][sl], out["dx_masked"][sl])
        gcr, e = g * c * r, out["dx_masked"][sl].double()
        for k, v in (("a", gcr), ("b", g), ("c", e)):
            acc[k] += v.sum(0)
            acc[k + "a"] += v.abs().sum(0)
    cd = col_depth(rows, width) + 4
    check_colsum("layernorm grad_a", out["grad_a"], g0[0], acc["a"], acc["aa"], cd)
    check_colsum("layernorm grad_b", out["grad_b"], g0[1], acc["b"], acc["ba"], cd)
    check_colsum("layernorm colsum_out", out["colsum"], g0[2], acc["c"], acc["ca"], cd)
    for sl in (slice(0, small), slice(rows - small, rows)):
        o = ln_bwd(lib, dy[sl].contiguous(), x[sl].contiguous(), a, m32[sl], s32[sl], eps, 0, p, None, None,
                   bf16_out=True)
        assert same_bits(o["dx"], out["dx"][sl]), f"backward rows {sl} depend on the launch"
        if sl.start == 0:      # (the dropout counter is the row index of the launch)
            assert same_bits(o["dx_masked"], out["dx_masked"][sl]) and same_bits(o["dy16"], out["dy16"][sl])
    if tail == 37:
        o = ln_bwd(lib, dy, x, a, m32, s32, eps, 0, p, None, None, bf16_out=True, rows_dev=dev_i32([live]))
        for k in ("dx", "dx_masked", "dy16"):
            assert same_bits(o[k][:live], out[k][:live]) and all_nan(o[k][live:]), f"rows_dev: {k}"
    del out, o, dy
    # final norm + head
    w = (torch.randn(width, device=DEV, generator=gen(width + 5)) / math.sqrt(width)).contiguous()
    wb = torch.tensor([0.25], device=DEV)
    score, hmean, hsd = head_fwd(lib, x, a, b, eps, w, wb, 1, act)
    sc = torch.empty(rows, device=DEV)
    for r0 in range(0, rows, CHUNK):
        sl = slice(r0, min(rows, r0 + CHUNK))
        H = head_ref(x[sl], a, b, eps, w, wb, 1, act)
        check("head score", score[sl], H["score"], H["score_b"])
        check("head mean", hmean[sl], H["mean"], H["mean_b"])
        check("head std", hsd[sl], H["sd"], H["sd_b"])
        sc[sl] = H["score"].float()
    for sl in (slice(0, small), slice(rows - small, rows)):
        o = head_fwd(lib, x[sl].contiguous(), a, b, eps, w, wb, 1, act)
        assert all(same_bits(u, v[sl]) for u, v in zip(o, (score, hmean, hsd))), f"head rows {sl} depend on the launch"
    dscore = torch.randn(rows, device=DEV, generator=gen(width + 6))
    dscore = torch.where(planted(rows), dscore * 1e3, dscore)
    hg0 = tuple(torch.randn(n, device=DEV, generator=gen(width + 7 + k))
                for k, n in enumerate((width,) * 3 + (1, width)))
    out = head_bwd(lib, dscore, sc, x, a, b, m32, s32, eps, w, 1, act, p, hg0)
    acc = {k: 0.0 for k in ("a", "aa", "ae", "b", "ba", "be", "w", "wa", "we", "wb", "wba", "wbe", "c", "ca", "ce")}
    for r0 in range(0, rows, CHUNK):
        sl = slice(r0, min(rows, r0 + CHUNK))
        H = head_bwd_ref(dscore[sl], sc[sl], x[sl], a, b, m32[sl], s32[sl], eps, w, 1, act)
        check("head dx", out["dx"][sl], H["dx"], H["dx_b"])
        want = masked(out["dx"][sl], r0, width, SITE_FC, p)
        if not same_bits(out["dx_masked"][sl], want):
            bad = torch.nonzero(bits(out["dx_masked"][sl]) != bits(want))
            i, j = (int(v) for v in bad[0])
            raise AssertionError(f"head dx_masked: {bad.shape[0]} differ, first row {r0 + i} col {j}: "
                                 f"dx {float(out['dx'][r0 + i, j])!r} dx_masked {float(out['dx_masked'][r0 + i, j])!r}"
                                 f" want {float(want[i, j])!r}; rows {sorted(set((bad[:, 0] + r0).tolist()))[:8]}")
        e = out["dx_masked"][sl].double()
        for k, v, va, ve in (("a", H["ga"], H["ga"].abs(), H["ga_e"]), ("b", H["gb"], H["gb"].abs(), H["gb_e"]),
                             ("w", H["gw"], H["gw_a"], H["gw_e"]),
                             ("wb", H["dz"][:, None], H["dz"].abs()[:, None], H["dz_e"][:, None]),
                             ("c", e, e.abs(), 0.0 * e)):
            acc[k] = acc[k] + v.sum(0)
            acc[k + "a"] = acc[k + "a"] + va.sum(0)
            acc[k + "e"] = acc[k + "e"] + ve.sum(0)
    cd = col_depth(rows, width) + 8
    for i, (name, k) in enumerate((("grad_a", "a"), ("grad_b", "b"), ("grad_w", "w"))):
        check_colsum(f"head {name}", out[name], hg0[i], acc[k], acc[k + "a"], cd, acc[k + "e"])
    check_colsum("head grad_wb", out["grad_wb"], hg0[3], acc["wb"], acc["wba"], wb_depth(rows, width) + 4, acc["wbe"])
    check_colsum("head colsum_out", out["colsum"], hg0[4], acc["c"], acc["ca"], cd)
    for sl in (slice(0, small), slice(rows - small, rows)):
        o = head_bwd(lib, dscore[sl].contiguous(), sc[sl].contiguous(), x[sl].contiguous(), a, b, m32[sl], s32[sl],
                     eps, w, 1, act, p, hg0)
        assert same_bits(o["dx"], out["dx"][sl]), f"head backward rows {sl} depend on the launch"
        if sl.start == 0:
            assert same_bits(o["dx_masked"], out["dx_masked"][sl])


# ------------------------------------------------------------------------------------------------ multi-output head
MULTI = [(w, 2 + i % 4) for i, w in enumerate(WIDTHS)]


@pytest.mark.parametrize("width,n", MULTI, ids=[f"W{w}-n{n}" for w, n in MULTI])
def test_head_multi(lib, width, n):
    act = ACTS[width % 4 if width > 8 else n % 4]
    P = lib.ptr
    for i, rows in enumerate((1, 7, 63, 65, 300)):
        p = (0.0, 0.1, 0.3)[i % 3]
        xf = make_x(rows, width, seed=width + rows)
        w = (torch.randn(n, width, device=DEV, generator=gen(width + n)) / math.sqrt(width)).contiguous()
        wb = torch.randn(n, device=DEV, generator=gen(width + n + 1))
        score = nan(rows, n)
        call(lib, "arb_head_multi_forward", P(xf), P(w), P(wb), act, rows, width, n, P(score))
        xd = xf.double()
        z = xd @ w.double().T + wb.double()
        zb = (4 * nv(width) + 7) * U * (xd.abs() @ w.double().abs().T + wb.double().abs())
        s = act_ref(z, act)
        check("multi score", score, s, act_bound(zb, s, act))
        # backward from the reference's scores
        s32 = s.float()
        ds = torch.randn(rows, n, device=DEV, generator=gen(width + rows + 1))
        ds[planted(rows)] *= 1e3
        dxf, dxm = nan(rows, width), nan(rows, width) if p > 0 else None
        gw0 = torch.randn(n, width, device=DEV, generator=gen(3))
        gwb0 = torch.randn(n, device=DEV, generator=gen(4))
        cs0 = torch.randn(width, device=DEV, generator=gen(5))
        gw, gwb, cs = gw0.clone(), gwb0.clone(), cs0.clone()
        call(lib, "arb_head_multi_backward", P(ds), P(s32), P(xf), P(w), act, rows, width, n, P(dxf), P(gw), P(gwb),
             P(dxm), P(cs), p, SEED, LAYER, SITE_FC)
        dz, dz_b = dz_ref(ds, s32, act)
        ref = dz @ w.double()
        check("multi dxf", dxf, ref, (n + 4) * U * (dz.abs() @ w.double().abs()) + dz_b @ w.double().abs())
        emitted = dxf
        if p > 0:
            assert same_bits(dxm, masked(dxf, 0, width, SITE_FC, p)), "multi dx_masked"
            emitted = dxm
        cd = 8 + 8 + det_depth(-(-rows // 64)) + 4
        for j in range(n):
            t = dz[:, j:j + 1] * xd
            check_colsum("multi grad_w", gw[j], gw0[j], t.sum(0), t.abs().sum(0), cd, (dz_b[:, j:j + 1] * xd.abs()).sum(0))
        check_colsum("multi grad_wb", gwb, gwb0, dz.sum(0), dz.abs().sum(0), cd, dz_b.sum(0))
        e = emitted.double()
        check_colsum("multi colsum_out", cs, cs0, e.sum(0), e.abs().sum(0), cd)


# ------------------------------------------------------------------------------------------------ column sums
@pytest.mark.parametrize("width", WIDTHS)
def test_column_sums(lib, width):
    """ld = width and ld > width; row counts that are not multiples of the 32-row warp pass or of the 256-row block,
    and more than 64 blocks (two DetParts levels)."""
    P = lib.ptr
    for rows in (1, 31, 33, 255, 257, 1000, 20011):
        for ld in (width, width + 12):
            src = torch.randn(rows, ld, device=DEV, generator=gen(rows + ld))
            src[planted(rows)] *= 1e3
            src[:, width:] = float("nan")          # columns beyond the width are never read
            out0 = torch.randn(width, device=DEV, generator=gen(width))
            out = out0.clone()
            call(lib, "arb_column_sums", P(src), rows, width, ld, P(out))
            t = src[:, :width].double()
            check_colsum("column sums", out, out0, t.sum(0), t.abs().sum(0), 32 + 8 + det_depth(-(-rows // 256)))


# ------------------------------------------------------------------------------------------------ softmax
SOFTMAX = [(S, pitch) for S in (1, 31, 32, 33, 240, 257, 1251, 1536) for pitch in (-(-S // 4) * 4, S + 13)]


def softmax_inputs(S, pitch, B, h, seed):
    """logits [B, h, S, pitch] (beyond S: NaN, never read), mask [B, S] with ~10 % masked keys and slate 1 all masked."""
    g = gen(seed)
    sc = 3.0 * torch.randn(B, h, S, pitch, device=DEV, generator=g)
    sc[..., S:] = float("nan")
    mask = (torch.rand(B, S, device=DEV, generator=g) < 0.1).to(torch.uint8)
    mask[0, 0] = 0
    if B > 1:
        mask[1] = 1
    return sc, mask


@pytest.mark.parametrize("p", [0.0, 0.1, 0.3])
@pytest.mark.parametrize("S,pitch", SOFTMAX, ids=[f"S{S}-pitch{p}" for S, p in SOFTMAX])
def test_softmax(lib, S, pitch, p):
    B, h = (3, 2) if S <= 257 else (2, 1)
    P = lib.ptr
    sc, mask = softmax_inputs(S, pitch, B, h, seed=S + pitch)
    out = sc.clone()
    call(lib, "arb_softmax_forward", P(out), P(mask), B, h, S, pitch, p, SEED, LAYER)
    again = sc.clone()
    call(lib, "arb_softmax_forward", P(again), P(mask), B, h, S, pitch, p, SEED, LAYER)
    assert same_bits(out, again), "two runs differ"
    assert same_bits(out[..., S:], sc[..., S:]), "columns beyond S written"
    rows = B * h * S
    s = sc[..., :S].double().masked_fill(mask.bool()[:, None, None, :], float("-inf"))
    mx = s.amax(-1, keepdim=True)
    e = torch.exp(s - mx)
    Pn = e / e.sum(-1, keepdim=True)                        # an all-masked slate: NaN rows, as the reference's
    D = dmask(0, rows, S, SITE_ATTN_P, p).reshape(B, h, S, S) if p > 0 else 1.0
    rel = (8 + -(-S // 32)) * U + U * (s - mx).abs().nan_to_num(posinf=0.0)
    rel_z = (Pn * rel).sum(-1, keepdim=True)
    got = out[..., :S]
    # (a dropped probability is +0 even in an all-masked slate's NaN rows: the kernel selects, it does not multiply)
    ref = torch.where(torch.as_tensor(D, device=DEV) == 0, 0.0, Pn * D)
    check("softmax P", got, ref, (Pn * (rel + rel_z) * D).nan_to_num(nan=0.0))
    if B > 1:
        assert torch.isnan(got[1][ref[1] != 0]).all() and torch.isnan(got[1]).any()
    # backward from the reference's undropped probabilities (0 for the all-masked slate)
    Pb = torch.where(torch.isnan(Pn), 0.0, Pn).float()
    dpt = torch.randn(B, h, S, S, device=DEV, generator=gen(S + 1))
    prob = torch.full((B, h, S, pitch), float("nan"), device=DEV)
    prob[..., :S] = Pb
    dprob = torch.full((B, h, S, pitch), float("nan"), device=DEV)
    dprob[..., :S] = dpt
    call(lib, "arb_softmax_backward", P(dprob), P(prob), rows, S, pitch, p, SEED, LAYER)
    assert all_nan(dprob[..., S:]) and all_nan(prob[..., S:]), "columns beyond S written"
    Pd, gv = Pb.double(), dpt.double() * D
    t = (Pd * gv).sum(-1, keepdim=True)
    dS = Pd * (gv - t)
    dS_b = (-(-S // 32) + 10) * U * Pd * (gv.abs() + (Pd * gv).abs().sum(-1, keepdim=True))
    check("softmax dS", dprob[..., :S], dS, dS_b)
    if p > 0:
        keep = keep_mask(0, rows, S, SITE_ATTN_P, p).reshape(B, h, S, S)
        want = torch.where(keep, Pb * torch.tensor(site_scale(p), device=DEV), torch.zeros((), device=DEV))
        assert same_bits(prob[..., :S], want), "prob is not overwritten with the dropped probabilities"
    else:
        assert same_bits(prob[..., :S], Pb)


# ------------------------------------------------------------------------------------------------ arguments, masks
def test_unsupported_shapes(lib):
    L, P = lib.lib(), lib.ptr
    x = torch.zeros(8, 1028, device=DEV)
    v = torch.zeros(1028, device=DEV)
    o = torch.zeros(8, 1028, device=DEV)
    r = torch.zeros(8, device=DEV)
    st = lib.stream_ptr()
    assert L.arb_layernorm_forward(P(x), P(v), P(v), 1e-6, 0, 8, 1028, P(o), None, P(r), P(r), None, None,
                                   st) == ARB_E_UNSUPPORTED
    assert L.arb_layernorm_backward(P(o), None, P(x), P(v), P(r), P(r), 1e-6, 0, None, 8, 1028, P(o), None, None,
                                    None, None, None, 0.0, SEED, LAYER, SITE_FFN_OUT, None, None,
                                    st) == ARB_E_UNSUPPORTED
    assert L.arb_head_forward(P(x), P(v), P(v), 1e-6, P(v), P(v), 1, 0, 8, 1028, P(r), P(r), P(r), None, None,
                              st) == ARB_E_UNSUPPORTED
    assert L.arb_head_backward(P(r), P(r), P(x), P(v), P(v), P(r), P(r), 1e-6, P(v), 1, 0, 8, 1028, P(o), None, None,
                               None, None, None, None, None, 0.0, SEED, LAYER, SITE_FC, None, None,
                               st) == ARB_E_UNSUPPORTED
    assert L.arb_head_multi_forward(P(x), P(v), P(v), 0, 8, 1028, 1, P(r), st) == ARB_E_UNSUPPORTED
    assert L.arb_head_multi_backward(P(r), P(r), P(x), P(v), 0, 8, 1028, 1, P(o), None, None, None, None, 0.0, SEED,
                                     LAYER, SITE_FC, st) == ARB_E_UNSUPPORTED
    assert L.arb_column_sums(P(x), 8, 1028, 1028, P(v), st) == ARB_E_UNSUPPORTED
    assert L.arb_layernorm_forward(P(x), P(v), P(v), 1e-6, 0, 8, 130, P(o), None, None, P(r), None, None, st) == -1
    assert L.arb_layernorm_forward(P(x), P(v), P(v), 1e-6, 0, 8, 6, P(o), None, P(r), P(r), None, None,
                                   st) == ARB_E_UNSUPPORTED
    sc = torch.zeros(1537 * 1540, device=DEV)
    mask = torch.zeros(1537, dtype=torch.uint8, device=DEV)
    assert L.arb_softmax_forward(P(sc), P(mask), 1, 1, 1537, 1540, 0.0, SEED, LAYER, st) == ARB_E_UNSUPPORTED
    assert L.arb_softmax_backward(P(sc), P(sc), 1537, 1537, 1540, 0.0, SEED, LAYER, st) == ARB_E_UNSUPPORTED
    assert L.arb_softmax_forward(P(sc), P(mask), 1, 1, 33, 32, 0.0, SEED, LAYER, st) == -1
    torch.cuda.synchronize()


def test_device_masks_match_mask_tensor():
    """keep_mask (the device evaluation used above) keeps and drops what tests/dropout_masks.mask_tensor does, at a
    row offset too."""
    for shape, site, p in (((37, 124), SITE_FFN_OUT, 0.1), ((5, 1000), SITE_FC, 0.3), ((40, 33), SITE_ATTN_P, 0.3)):
        want = mask_tensor(shape, SEED, LAYER, site, p).cuda() != 0
        assert torch.equal(keep_mask(0, shape[0], shape[1], site, p), want)
        assert torch.equal(keep_mask(3, shape[0], shape[1], site, p), want[3:])


def test_references_are_the_autograd_gradients():
    """norm_bwd_ref / head_bwd_ref restate what autograd gives for the fp64 LayerNorm (both kinds) and head, at the
    reference's own statistics (rows with a non-zero std)."""
    g = gen(1)
    x = (torch.randn(6, 36, device=DEV, generator=g) * 3 + 1).double().requires_grad_()
    a, b = (t.double() for t in make_gain(36, 2))
    dy = torch.randn(6, 36, device=DEV, generator=g).double()
    for tm, eps in ((0, 0.1), (1, 1e-5)):
        if tm:
            y = torch.nn.functional.layer_norm(x, (36,), a, b, eps)
        else:
            y = a * (x - x.mean(1, keepdim=True)) / (x.std(1, keepdim=True) + eps) + b
        (gx,) = torch.autograd.grad(y, x, dy)
        m = x.detach().mean(1)
        s = (x.detach().var(1, unbiased=not tm) + (eps if tm else 0.0)).sqrt()
        dx, _, _, _ = norm_bwd_ref(dy, 0.0, x.detach(), a, m, s, 0.0 if tm else eps, tm)
        assert torch.allclose(dx, gx, rtol=1e-10, atol=1e-12)
    w = torch.randn(36, device=DEV, generator=g).double()
    ds = torch.randn(6, device=DEV, generator=g).double()
    xn = a * (x - x.mean(1, keepdim=True)) / (x.std(1, keepdim=True) + 0.1) + b
    for act in ACTS:
        s = act_ref(xn @ w + 0.25, act)
        (gx,) = torch.autograd.grad(s, x, ds, retain_graph=True)
        H = head_bwd_ref(ds, s.detach(), x.detach(), a, b, x.detach().mean(1), x.detach().std(1), 0.1, w, 1, act)
        assert torch.allclose(H["dx"], gx, rtol=1e-10, atol=1e-12), act
