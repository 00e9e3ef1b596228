"""The twelve activation classes after None / ReLU / Tanh / Sigmoid on the GPU (include/allrank_b200.h ARB_ACT_*):
LeakyReLU, ELU, CELU, SELU, Softplus, Softsign, Hardtanh, ReLU6, Hardsigmoid, LogSigmoid, Hardshrink and Softshrink at
torch's default arguments, as the FC activation and as the output activation.

Kernels, through the arb_activation_* and arb_head_* entry points:
- forward against fp64 of the same fp32 z, within FWD_ULP ulp (the spacing of fp32 at the larger of the two values).  The bounds follow the CUDA
  Math API's maximum errors (expf 2 ulp, expm1f 1, log1pf 1, IEEE division and products 0.5) and the fp32 constants:
  1 for the products with 0.01 and lambda; ELU / CELU, expm1f alone: 2 (its documented ulp is met to within 0.12 ulp
  in this measure over a million samples); SELU's negative branch expm1f times fl(lambda alpha): 3;
  Softsign's |z| + 1 and division: 2; Hardsigmoid's z + 3 and the product with fl(1 / 6): 2; Softplus and LogSigmoid,
  expf's 2 ulp carried through log1p with a factor of at most 1, then log1pf's 1 ulp and a rounding: 4; the clamps and
  shrinks are exact but for Softshrink's one rounded subtraction (1).  At the kink values (0, +-0.5, +-1, +-3, 6, 20,
  -0.0, +-inf) the output equals torch's own fp32 forward.
- backward: act'(z) read off the output.  Away from the kinks within BWD_ABS units of 2^-24 times max(1, |act'|) of
  the fp64 derivative: the forward's error of at most 4 ulp of y passes through a derivative whose slope in y is at
  most 1 (SELU's y reaches lambda alpha ~ 1.76, hence 16).  At the kink values it equals torch autograd's derivative
  on the same fp32 z.  Under dropout every saturated element of Hardtanh, ReLU6 and Hardsigmoid gets exactly 0, and the
  column sums follow the kernel's order (tests/test_gpu_scorer_simt.colsum_emulation) bit for bit.
- head forward / backward with and without the final LayerNorm, and the multi-output head, against fp64.
Models: golden vectors of the unmodified reference (tests/golden/scorer_activations.npz,
tools/make_golden_activations.py) in the packed-row and dense layouts; train mode under the regenerated dropout masks
against oracle/tf32_emulation.py (its activation table extended here by the torch classes of the same names); x.grad
and prepare_for_output against oracle/scorer_ref.py; a loss + FlatAdam step; a graphed dropout step equal to the
eager one; and an unmodified allrank.main.run() under patch_allrank() with LeakyReLU and Softplus."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.dropout_masks import SITE_FC, mask_tensor
from tests.test_gpu_fc_block import build_pair
from tests.test_gpu_scorer_simt import P, bits, call, colsum_emulation, lib, nan, same_bits, site_scale  # noqa: F401

pytestmark = pytest.mark.gpu

DEV = "cuda"
SEED = 0x5DEECE66D
LAYER = 1
NAMES = ["LeakyReLU", "ELU", "CELU", "SELU", "Softplus", "Softsign", "Hardtanh", "ReLU6", "Hardsigmoid", "LogSigmoid",
         "Hardshrink", "Softshrink"]
ID = {n: 5 + i for i, n in enumerate(NAMES)}
FWD_ULP = {"LeakyReLU": 1, "ELU": 2, "CELU": 2, "SELU": 3, "Softplus": 4, "Softsign": 2, "Hardtanh": 0, "ReLU6": 0,
           "Hardsigmoid": 2, "LogSigmoid": 4, "Hardshrink": 0, "Softshrink": 1}
BWD_ABS = 16
LAM, ALPHA = 1.0507009873554805, 1.6732632423543772
KINKS = [0.0, -0.0, 0.5, -0.5, 1.0, -1.0, 3.0, -3.0, 6.0, -6.0, 20.0, -20.0, float("inf"), float("-inf")]
SHAPES = [(1, 4), (255, 12), (256, 64), (16385, 100), (255, 1000), (2 ** 17 + 3, 8)]
SATURATING = ["Hardtanh", "ReLU6", "Hardsigmoid"]
EXACT_FWD = ["LeakyReLU", "Hardtanh", "ReLU6", "Hardshrink", "Softshrink"]   # the same fp32 operations as torch's CPU
PIECEWISE = ["LeakyReLU", "Hardtanh", "ReLU6", "Hardsigmoid", "Hardshrink", "Softshrink"]   # constant derivatives
# a jump at |z| = 0.5: TF32 products move a few pre-activations across it, so the model-level comparisons of these
# cases bound the share of values off by more than the tolerance (5 %: a flip in one layer moves every value of the
# next a little, and some of those across the jump again) and take the gradients within 2e-1
JUMP = ("Hardshrink",)
# derivatives that jump (at 0 for LeakyReLU and SELU, at the bounds of the clamps and shrinks): the same pre-activations
# flip a few derivatives, so the model-level gradient comparisons of these cases allow 2e-1 instead of 5e-2
DERIV_JUMP = ("LeakyReLU", "SELU", "Hardtanh", "ReLU6", "Hardsigmoid", "Hardshrink", "Softshrink")


def f64(z, name):
    """the activation in fp64"""
    if name == "LeakyReLU":
        return np.where(z > 0, z, 0.01 * z)
    if name in ("ELU", "CELU"):
        return np.where(z > 0, z, np.expm1(np.minimum(z, 0)))
    if name == "SELU":
        return LAM * np.where(z > 0, z, ALPHA * np.expm1(np.minimum(z, 0)))
    if name == "Softplus":
        return np.where(z > 20, z, np.logaddexp(0, np.minimum(z, 20)))
    if name == "Softsign":
        return z / (1 + np.abs(z))
    if name == "Hardtanh":
        return np.clip(z, -1, 1)
    if name == "ReLU6":
        return np.clip(z, 0, 6)
    if name == "Hardsigmoid":
        return np.clip(z / 6 + 0.5, 0, 1)
    if name == "LogSigmoid":
        return -np.logaddexp(0, -z)
    if name == "Hardshrink":
        return np.where(np.abs(z) > 0.5, z, 0.0)
    return np.where(z > 0.5, z - 0.5, np.where(z < -0.5, z + 0.5, 0.0))


def d64(z, name):
    """its derivative in fp64 (away from the kinks)"""
    if name == "LeakyReLU":
        return np.where(z > 0, 1.0, 0.01)
    if name in ("ELU", "CELU"):
        return np.where(z > 0, 1.0, np.exp(np.minimum(z, 0)))
    if name == "SELU":
        return np.where(z > 0, LAM, LAM * ALPHA * np.exp(np.minimum(z, 0)))
    if name == "Softplus":
        return np.where(z > 20, 1.0, 1 / (1 + np.exp(-z)))
    if name == "Softsign":
        return 1 / (1 + np.abs(z)) ** 2
    if name == "Hardtanh":
        return ((z > -1) & (z < 1)).astype(np.float64)
    if name == "ReLU6":
        return ((z > 0) & (z < 6)).astype(np.float64)
    if name == "Hardsigmoid":
        return ((z > -3) & (z < 3)) / 6.0
    if name == "LogSigmoid":
        return 1 / (1 + np.exp(z))
    return (np.abs(z) > 0.5).astype(np.float64)


def dout64(y, name):
    """its derivative as the kernels read it off the output y (include/allrank_b200.h ARB_ACT_*), in fp64"""
    if name == "LeakyReLU":
        return np.where(y > 0, 1.0, 0.01)
    if name in ("ELU", "CELU"):
        return np.where(y > 0, 1.0, y + 1)
    if name == "SELU":
        return np.where(y > 0, LAM, y + LAM * ALPHA)
    if name == "Softplus":
        return np.where(y > 20, 1.0, -np.expm1(-y))
    if name == "Softsign":
        return (1 - np.abs(y)) ** 2
    if name == "Hardtanh":
        return ((y > -1) & (y < 1)).astype(np.float64)
    if name == "ReLU6":
        return ((y > 0) & (y < 6)).astype(np.float64)
    if name == "Hardsigmoid":
        return ((y > 0) & (y < 1)) / 6.0
    if name == "LogSigmoid":
        return -np.expm1(y)
    return (y != 0).astype(np.float64)


def torch_act(name):
    return getattr(torch.nn, name)()


def act_forward(lib, z, act, p, rows_dev=None):
    h = z.clone()
    call(lib, "arb_activation_forward", P(h), h.shape[0], h.shape[1], act, p, SEED, LAYER, P(rows_dev))
    return h


def act_backward(lib, dh, h, act, p, mul=1.0, cs=None):
    dz = nan(*h.shape)
    call(lib, "arb_activation_backward", P(dh), P(h), P(dz), h.shape[0], h.shape[1], act, p, SEED, LAYER, mul, P(cs),
         None)
    return dz


def ulp32(x64):
    return np.spacing(np.abs(x64.astype(np.float32))).astype(np.float64)


def inputs(rows, width, name, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    z = torch.randn(rows, width, device=DEV, generator=g) * 4
    if name == "ReLU6":
        z = z + 3
    return z.float()


def kink_tensor():
    z = torch.tensor(KINKS, dtype=torch.float32)
    z = torch.cat([z, torch.zeros(-len(KINKS) % 4)]).view(-1, 4)
    return z


# ------------------------------------------------------------------------------------------------ activation kernels
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("rows,width", SHAPES)
def test_activation_forward(lib, name, rows, width):
    act = ID[name]
    z = inputs(rows, width, name, rows * 7 + width + act)
    y0 = act_forward(lib, z, act, 0.0)
    assert same_bits(y0, act_forward(lib, z, act, 0.0)), "two calls differ"
    r64 = f64(z.double().cpu().numpy(), name)
    y = y0.double().cpu().numpy()
    err = np.abs(y - r64) / np.maximum(ulp32(np.maximum(np.abs(y), np.abs(r64))), 2.0 ** -149)
    assert err.max() <= max(FWD_ULP[name], 0.5), f"{err.max():.2f} ulp"
    for p in (0.1, 0.5):
        h = act_forward(lib, z, act, p)
        assert same_bits(h, act_forward(lib, z, act, p))
        keep = mask_tensor((rows, width), SEED, LAYER, SITE_FC, p).to(DEV) != 0
        assert torch.equal(bits(h)[~keep], torch.zeros_like(bits(h)[~keep])), "dropped elements must be +0.0"
        assert same_bits(h[keep], (y0 * torch.tensor(site_scale(p), device=DEV))[keep])


@pytest.mark.parametrize("name", NAMES)
def test_activation_forward_at_the_kinks_equals_torch(lib, name):
    z = kink_tensor()
    y = act_forward(lib, z.to(DEV), ID[name], 0.0).cpu()
    want = torch_act(name)(z)
    assert torch.allclose(y, want, rtol=2.0 ** -21, atol=0.0, equal_nan=True), (z, y, want)
    if name in EXACT_FWD:
        assert torch.equal(y, want)


@pytest.mark.parametrize("name", NAMES)
def test_activation_forward_rows_dev(lib, name):
    rows, width, live = 700, 36, 333
    z = inputs(rows, width, name, 5)
    z[live:] = float("nan")
    dev = torch.tensor([live], dtype=torch.int32, device=DEV)
    h = act_forward(lib, z, ID[name], 0.1, dev)
    assert same_bits(h[:live], act_forward(lib, z[:live].contiguous(), ID[name], 0.1))
    assert torch.isnan(h[live:]).all()


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("rows,width", SHAPES)
def test_activation_backward_against_fp64(lib, name, rows, width):
    act = ID[name]
    z = inputs(rows, width, name, rows + 3 * width + act)
    h = act_forward(lib, z, act, 0.0)
    one = torch.ones_like(z)
    d0 = act_backward(lib, one, h, act, 0.0)
    assert same_bits(d0, act_backward(lib, one, h, act, 0.0)), "two calls differ"
    d = d0.double().cpu().numpy()
    want = d64(z.double().cpu().numpy(), name)
    err = np.abs(d - want) / (2.0 ** -24 * np.maximum(1.0, np.abs(want)))
    assert err.max() <= BWD_ABS, f"{err.max():.2f} units of 2^-24"


@pytest.mark.parametrize("name", NAMES)
def test_activation_backward_at_the_kinks_equals_torch_autograd(lib, name):
    z = kink_tensor()
    h = act_forward(lib, z.to(DEV), ID[name], 0.0)
    got = act_backward(lib, torch.ones_like(h), h, ID[name], 0.0).cpu()
    zr = z.clone().requires_grad_(True)
    torch_act(name)(zr).sum().backward()
    want = zr.grad
    n = len(KINKS)
    g, w = got.flatten()[:n], want.flatten()[:n]
    assert torch.allclose(g, w, rtol=0.0, atol=BWD_ABS * 2.0 ** -24, equal_nan=True), (z.flatten()[:n], g, w)
    if name in PIECEWISE:
        assert torch.equal(g, w), (z.flatten()[:n], g, w)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("p", [0.1, 0.3, 0.5])
def test_activation_backward_under_dropout(lib, name, p):
    """Kept elements: ((dh * mul) * scale) * act', where Hardtanh, ReLU6 and Hardsigmoid decide saturation on the
    stored h; a saturated element gets exactly 0 whatever the rounding of h * (1 / scale).  Column sums in order."""
    act = ID[name]
    rows, width = 20000, 36
    z = inputs(rows, width, name, 77 + act)
    h = act_forward(lib, z, act, p)
    y0 = act_forward(lib, z, act, 0.0)
    g = torch.Generator(device=DEV).manual_seed(3)
    dh = torch.randn(rows, width, device=DEV, generator=g)
    cs0 = torch.randn(width, device=DEV, generator=g)
    outs = []
    for _ in range(2):
        cs = cs0.clone()
        outs.append((act_backward(lib, dh, h, act, p, 2.0, cs), cs))
    assert same_bits(outs[0][0], outs[1][0]) and same_bits(outs[0][1], outs[1][1])
    dz, cs = outs[0]
    keep = mask_tensor((rows, width), SEED, LAYER, SITE_FC, p).to(DEV) != 0
    assert torch.equal(bits(dz)[~keep], torch.zeros_like(bits(dz)[~keep]))
    # the derivative the kernel applied to each kept element, against the p = 0 derivative of the same output
    scale = torch.tensor(site_scale(p), device=DEV)
    base = (dh * 2.0) * scale
    d_p0 = act_backward(lib, torch.ones_like(y0), y0, act, 0.0)
    if name in SATURATING:
        lo, hi = {"Hardtanh": (-1.0, 1.0), "ReLU6": (0.0, 6.0), "Hardsigmoid": (0.0, 1.0)}[name]
        sat = keep & ((y0 <= lo) | (y0 >= hi))
        assert sat.sum() > 100
        assert bool((dz[sat] == 0).all()), "a saturated element got a gradient"   # (+0 or -0: 0 times dh's sign)
        # (an output within 2 ulp of the upper bound may round to bound * scale in h: left out)
        inside = keep & (y0 > lo) & (y0 < hi) & (hi - y0 > 2.0 ** -22 * hi)
        assert same_bits(dz[inside], (base * d_p0)[inside])
    else:
        z64 = z.double().cpu().numpy()
        want = base.double().cpu().numpy() * d64(z64, name)
        k = keep.cpu().numpy()
        tol = (BWD_ABS + 8) * 2.0 ** -24 * np.abs(base.double().cpu().numpy()) * np.maximum(1.0, np.abs(d64(z64, name)))
        assert np.all(np.abs(dz.double().cpu().numpy() - want)[k] <= tol[k] + 1e-30)
    want_cs = (cs0.cpu().numpy() + colsum_emulation(dz.cpu().numpy(), width)).astype(np.float32)
    assert np.array_equal(cs.cpu().numpy().view(np.int32), want_cs.view(np.int32)), "column sums differ from the order"


def test_unknown_activation_ids_are_refused(lib):
    from tests.test_gpu_scorer_simt import refused
    h = torch.zeros(8, 8, device=DEV)
    for act in (4, 17, -1):
        refused(lib, "arb_activation_forward", P(h), 8, 8, act, 0.0, SEED, LAYER, None)


# ------------------------------------------------------------------------------------------------ head kernels
@pytest.fixture(scope="module")
def hlib(lib):
    import ctypes
    p, i, f, u, q = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float, ctypes.c_uint64, ctypes.c_int64
    lib.register("arb_head_forward", i, [p, p, p, f, p, p, i, i, q, i, p, p, p, p, p])
    lib.register("arb_head_backward", i, [p, p, p, p, p, p, p, f, p, i, i, q, i, p, p, p, p, p, p, p, p, f, u, i, i,
                                          p, p])
    lib.register("arb_head_multi_forward", i, [p, p, p, i, q, i, i, p])
    lib.register("arb_head_multi_backward", i, [p, p, p, p, i, q, i, i, p, p, p, p, p, f, u, i, i])
    return lib


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("has_norm", [0, 1])
def test_head_forward_and_backward_against_fp64(hlib, name, has_norm):
    rows, width, eps = 3001, 96, 1e-6
    g = torch.Generator(device=DEV).manual_seed(ID[name] * 2 + has_norm)
    x = torch.randn(rows, width, device=DEV, generator=g)
    a = 1 + 0.1 * torch.randn(width, device=DEV, generator=g)
    b = 0.1 * torch.randn(width, device=DEV, generator=g)
    w = torch.randn(width, device=DEV, generator=g) * (0.5 if has_norm else 0.3)
    wb = torch.tensor([0.4], device=DEV)
    score, mean, sd = nan(rows), nan(rows), nan(rows)
    call(hlib, "arb_head_forward", P(x), P(a), P(b), eps, P(w), P(wb), has_norm, ID[name], rows, width, P(score),
         P(mean), P(sd), None, None)
    X, A, Bv, W = (t.double().cpu() for t in (x, a, b, w))
    if has_norm:
        xf = A * (X - X.mean(-1, keepdim=True)) / (X.std(-1, keepdim=True) + eps) + Bv
    else:
        xf = X
    z = (xf @ W + 0.4).numpy()
    s64 = f64(z, name)
    bound = 1e-5 * (1 + (xf.abs() @ W.abs()).numpy())
    ok = np.abs(np.abs(z) - 0.5) > bound if name in JUMP else np.ones(rows, bool)
    assert np.all((np.abs(score.double().cpu().numpy() - s64) <= bound)[ok])
    dscore = torch.randn(rows, device=DEV, generator=g)
    dx, ga, gbb, gw, gwb = nan(rows, width), torch.zeros(width, device=DEV), torch.zeros(width, device=DEV), \
        torch.zeros(width, device=DEV), torch.zeros(1, device=DEV)
    call(hlib, "arb_head_backward", P(dscore), P(score), P(x), P(a), P(b), P(mean), P(sd), eps, P(w), has_norm,
         ID[name], rows, width, P(dx), P(ga), P(gbb), P(gw), P(gwb), None, None, None, 0.0, SEED, 0, 0, None, None)
    # (act' read off the kernel's own score: a z within rounding of a kink may sit on either side)
    dz = dscore.double().cpu().numpy() * dout64(score.double().cpu().numpy(), name)
    assert _rel(gwb.cpu().numpy(), [dz.sum()]) <= 3e-4
    assert _rel(gw.cpu().numpy(), dz @ xf.numpy()) <= 3e-4
    if has_norm:
        Xr = X.clone().requires_grad_(True)
        xr = A * (Xr - Xr.mean(-1, keepdim=True)) / (Xr.std(-1, keepdim=True) + eps) + Bv
        (xr @ W * torch.from_numpy(dz)).sum().backward()
        assert _rel(dx.cpu().numpy(), Xr.grad.numpy()) <= 3e-4
    else:
        assert _rel(dx.cpu().numpy(), dz[:, None] * W.numpy()[None, :]) <= 3e-4


@pytest.mark.parametrize("name", NAMES)
def test_multi_output_head_against_fp64(hlib, name):
    rows, width, n = 2049, 64, 4
    g = torch.Generator(device=DEV).manual_seed(ID[name])
    xf = torch.randn(rows, width, device=DEV, generator=g)
    w = torch.randn(n, width, device=DEV, generator=g) * 0.3
    wb = torch.randn(n, device=DEV, generator=g) * 0.2
    score = nan(rows, n)
    call(hlib, "arb_head_multi_forward", P(xf), P(w), P(wb), ID[name], rows, width, n, P(score))
    X, W = xf.double().cpu().numpy(), w.double().cpu().numpy()
    z = X @ W.T + wb.double().cpu().numpy()
    bound = 1e-5 * (1 + np.abs(X) @ np.abs(W).T)
    ok = np.abs(np.abs(z) - 0.5) > bound if name in JUMP else np.ones(z.shape, bool)
    assert np.all((np.abs(score.double().cpu().numpy() - f64(z, name)) <= bound)[ok])
    dscore = torch.randn(rows, n, device=DEV, generator=g)
    dxf, gw, gwb = nan(rows, width), torch.zeros(n, width, device=DEV), torch.zeros(n, device=DEV)
    call(hlib, "arb_head_multi_backward", P(dscore), P(score), P(xf), P(w), ID[name], rows, width, n, P(dxf), P(gw),
         P(gwb), None, None, 0.0, SEED, 0, 0)
    dz = dscore.double().cpu().numpy() * dout64(score.double().cpu().numpy(), name)
    assert _rel(dxf.cpu().numpy(), dz @ W) <= 3e-4
    assert _rel(gw.cpu().numpy(), dz.T @ X) <= 3e-4
    assert _rel(gwb.cpu().numpy(), dz.sum(0)) <= 3e-4


# ------------------------------------------------------------------------------------------------ models
def golden_model(g, name):
    """make_model under the generator's seeds (tools/make_golden_activations.py)"""
    from allrank_b200.model import make_model
    m = json.loads(str(g[name + ":model"]))
    torch.manual_seed(87)
    model = make_model(fc_model=m["fc_model"], transformer=m["transformer"], post_model=m["post_model"],
                       n_features=int(g[name + ":F"]))
    gen = torch.Generator().manual_seed(88)
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    return model


def _check_scores(out, ref, valid, tol, jump):
    err = (out - ref)[valid].abs()
    tol = tol * max(1.0, ref[valid].abs().max().item())
    if jump:
        assert (err > tol).float().mean().item() <= 0.05, err.max().item()
    else:
        assert err.max().item() <= tol, err.max().item()


GOLDEN = [f"fc_{n}" for n in NAMES] + [f"out_{n}" for n in NAMES] + ["enc_Softplus", "enc_SELU", "enc_Hardtanh",
                                                                     "d4_Hardsigmoid"]


@pytest.fixture(params=["packed", "dense"])
def layout(request):
    from allrank_b200 import _lib
    lib = _lib.lib()
    lib.arb_set_pack_rows(1 if request.param == "packed" else 0)
    yield request.param
    lib.arb_set_pack_rows(_lib.default_pack_rows())


@pytest.mark.parametrize("name", GOLDEN)
def test_eval_matches_the_reference_golden_vectors(golden, name, layout):
    g = golden("scorer_activations")
    model = golden_model(g, name)
    for k, v in model.state_dict().items():
        assert np.array_equal([v.double().sum().item(), v.double().abs().sum().item()], g[name + ":c:" + k]), k
    model = model.cuda().eval()
    F = int(g[name + ":F"])
    x, y = torch.tensor(g[f"x{F}"]).cuda(), torch.tensor(g[f"y{F}"]).cuda()
    out = model(x, y == -1, None)
    ref = torch.tensor(g[name + ":scores"])
    valid = (y != -1).cpu()
    jump = name.endswith(JUMP)
    _check_scores(out.detach().cpu(), ref, valid, 5e-3, jump)
    gtol = 2e-1 if name.endswith(DERIV_JUMP) else 5e-2
    (out * torch.tensor(g[name + ":w"]).cuda()).sum().backward()
    params = dict(model.named_parameters())
    rms_max = max(float(g[name + ":n:" + k]) / np.sqrt(p.numel()) for k, p in params.items())
    for k, p in params.items():
        n = p.numel()
        gi = torch.arange(n) if n <= 256 else torch.linspace(0, n - 1, 256).long()
        got = p.grad.detach().flatten().cpu()[gi].double().numpy()
        want = g[name + ":g:" + k].astype(np.float64)
        fro = np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-2 * rms_max * np.sqrt(len(gi)))
        nrm = abs(p.grad.norm().item() - float(g[name + ":n:" + k])) / max(float(g[name + ":n:" + k]),
                                                                           1e-2 * rms_max * np.sqrt(n))
        assert fro <= gtol and nrm <= gtol, (k, fro, nrm)


# F, sizes, act, input_norm, N, h, dff, positional, d_output, out_act
MODEL_CASES = [(46, [50, 30], n, False, 0, 1, 4, None, 1, None) for n in NAMES] + \
    [(46, [50, 30], "ReLU", False, 0, 1, 4, None, 1, n) for n in NAMES] + \
    [(46, [64], "Softplus", False, 2, 4, 128, None, 1, None), (46, [64], "SELU", False, 2, 4, 128, None, 1, "Tanh"),
     (46, [64], "Hardtanh", False, 1, 4, 128, None, 4, "Hardsigmoid")]
MODEL_IDS = [f"{c[2]}-N{c[4]}-o{c[8]}{c[9]}" for c in MODEL_CASES]


def _slates(B, S, F, seed):
    from allrank_b200.synth import make_slates
    return make_slates(B, S, n_features=F, seed=seed, mean_len=int(0.6 * S), std_len=S // 5)


@pytest.fixture
def emulated_activations(monkeypatch):
    """oracle/tf32_emulation.py's activation table, extended by the torch classes of the other names"""
    from oracle import tf32_emulation
    base = tf32_emulation._activation
    monkeypatch.setattr(tf32_emulation, "_activation",
                        lambda t, name: base(t, name) if name in (None, "ReLU", "Tanh", "Sigmoid")
                        else torch_act(name)(t))


@pytest.mark.parametrize("case", MODEL_CASES, ids=MODEL_IDS)
def test_train_mode_matches_the_tf32_emulation(case, emulated_activations):
    from oracle.tf32_emulation import scorer_forward
    from tests.dropout_masks import scorer_masks
    Fn, sizes, act, inorm, N, h, dff, pos, n_out, out_act = case
    p, p_fc = (0.2 if N else 0.0), 0.25
    _, mine = build_pair(case, p=p, p_fc=p_fc)
    mine.train()
    B, S = 3, 240
    x, y, idx = _slates(B, S, Fn, seed=9)
    mask = y == -1
    torch.manual_seed(31)
    call_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    torch.manual_seed(31)
    xm = x.cuda().requires_grad_(True)
    out = mine(xm, mask.cuda(), None)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(6))
    (out * w.cuda()).sum().backward()
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in mine.state_dict().items()}
    xe = x.clone().requires_grad_(True)
    ref = scorer_forward(sd, xe, mask, N, h, out_act, "rna", drop=scorer_masks(call_seed, B, S, sizes, N, h, dff, p,
                                                                               p_fc), fc_act=act)
    (ref * w).sum().backward()
    valid = ~mask
    jump = act in JUMP or out_act in JUMP
    _check_scores(out.detach().cpu(), ref.detach(), valid, 3e-3, jump)
    tol = 2e-1 if jump else (3e-2 if N == 0 else 1e-1)
    floor = 1e-2 * max(v.grad.abs().max().item() for v in sd.values())
    for k, q in mine.named_parameters():
        a, r = q.grad.cpu().double().numpy(), sd[k].grad.double().numpy()
        rel = np.linalg.norm(a - r) / max(np.linalg.norm(r), floor * np.sqrt(r.size))
        assert rel <= tol, (k, rel)
    rel = (xm.grad.cpu() - xe.grad).norm().item() / max(xe.grad.norm().item(), 1e-6)
    assert rel <= tol, ("x.grad", rel)


@pytest.mark.parametrize("case", MODEL_CASES, ids=MODEL_IDS)
def test_input_gradient_and_prepare_for_output_match_the_oracle(case, dense_rows):
    ref, mine = build_pair(case)
    ref.eval(); mine.eval()
    B, S = 4, 120
    x, y, idx = _slates(B, S, case[0], seed=8)
    mask = y == -1
    valid = ~mask
    xr = x.clone().requires_grad_(True)
    xm = x.cuda().requires_grad_(True)
    out_ref, out = ref(xr, mask, idx), mine(xm, mask.cuda(), idx.cuda())
    w = torch.randn(out_ref.shape, generator=torch.Generator().manual_seed(12))
    (out_ref * w).sum().backward()
    (out * w.cuda()).sum().backward()
    jump = case[2] in JUMP or case[9] in JUMP
    _check_scores(out.detach().cpu(), out_ref.detach(), valid, 5e-3, jump)
    gx, rx = xm.grad.cpu()[valid], xr.grad[valid]
    assert (gx - rx).norm().item() <= (2e-1 if jump else 5e-2) * max(rx.norm().item(), 1e-6), "x.grad"
    with torch.no_grad():
        hid = mine.prepare_for_output(x.cuda(), mask.cuda(), idx.cuda()).cpu()
        hid_ref = ref.prepare_for_output(x, mask, idx)
    assert hid.shape == hid_ref.shape == (B, S, case[1][-1])
    _check_scores(hid, hid_ref, valid, 5e-3, jump)


@pytest.mark.parametrize("case", MODEL_CASES[:12], ids=MODEL_IDS[:12])
def test_a_loss_and_flat_adam_step_trains(case):
    from allrank_b200 import losses
    from allrank_b200.optim import FlatAdam
    _, mine = build_pair(case, p_fc=0.25)
    mine.train()
    opt = FlatAdam(mine, lr=1e-2)
    before = [q.detach().clone() for q in mine.parameters()]
    x, y, _ = _slates(8, 120, case[0], seed=40)
    loss = losses.approxNDCGLoss(mine.score(x.cuda(), (y == -1).cuda(), None), y.cuda())
    opt.zero_grad()
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss)
    assert all(q.grad is not None and bool(q.grad.isfinite().all()) for q in mine.parameters())
    assert all(bool(q.isfinite().all()) for q in mine.parameters())
    assert any(not torch.equal(a, q.detach()) for a, q in zip(before, mine.parameters()))


@pytest.mark.parametrize("name", ["Hardtanh", "Softplus"])
def test_graphed_dropout_step_equals_the_eager_step(name, monkeypatch):
    from allrank_b200 import losses
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.optim import FlatAdam
    case = (46, [50, 30], name, False, 0, 1, 4, None, 1, None)
    batches = [_slates(8, 240, 46, seed=20 + k)[:2] for k in range(2)] * 2
    batches = [(x.cuda(), y.cuda()) for x, y in batches]
    s = 977
    _, eager = build_pair(case, p_fc=0.25)
    eager.train()
    opt = FlatAdam(eager, lr=1e-3, capturable=True)
    eager_losses = []
    for k, (x, y) in enumerate(batches, start=1):
        monkeypatch.setattr(eager, "_draw_seed", lambda k=k: s + k)
        loss = losses.approxNDCGLoss(eager(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        eager_losses.append(loss.item())
    _, graphed = build_pair(case, p_fc=0.25)
    graphed.train()
    gopt = FlatAdam(graphed, lr=1e-3, capturable=True)
    init = {k: v.clone() for k, v in graphed.state_dict().items()}
    monkeypatch.setattr(graphed, "_draw_seed", lambda: pytest.fail("the graphed step drew a host seed"))
    step = GraphedTrainStep(graphed, losses.approxNDCGLoss, gopt, *batches[0], warmup=2, dropout_seed=s)
    graphed.load_state_dict(init)
    gopt.exp_avg.zero_(); gopt.exp_avg_sq.zero_(); gopt._dev_state.zero_()
    graph_losses = [step(x, y).item() for x, y in batches]
    assert graph_losses == eager_losses
    assert torch.equal(graphed.flat_parameters, eager.flat_parameters)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "allrank", "main.py"))


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
def test_unmodified_main_trains_leaky_relu_and_softplus_under_patch(tmp_path):
    """allrank.main.run() under patch_allrank() on the reference's dummy data, FC activation LeakyReLU and output
    activation Softplus: the run finishes on the native library with the reference's parameter count."""
    with open(os.path.join(ROOT, "tests", "configs", "baseline_cfg1.json")) as f:
        cfg = json.load(f)
    cfg["model"]["fc_model"].update({"sizes": [64, 32], "activation": "LeakyReLU", "dropout": 0.1})
    cfg["model"]["post_model"]["output_activation"] = "Softplus"
    cfg["training"]["epochs"] = 2
    path = tmp_path / "activations_cfg.json"
    path.write_text(json.dumps(cfg))
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    cmd = [sys.executable, os.path.join(ROOT, "oracle", "run_reference_main.py"), "--workdir", str(tmp_path),
           "--config", str(path), "--run-id", "gpu", "--patched"]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])
    assert res["native_so_loaded"]
    assert np.isfinite(res["val_metrics/ndcg_5"]) and res["val_metrics/ndcg_5"] > 0.0
