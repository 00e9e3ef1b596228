"""Head widths d_model / h that are not a multiple of 4: the scorer pads every head to hs = round_up(w, 4) columns with
exact zeros (DESIGN.md 4.15) and runs the existing fused kernels at width hs with the scale 1/sqrt(w).

Kernel level, through arb_attention_padded_forward / arb_attention_padded_backward (the scorer's descriptors), against
the fp64 reference of tests/test_gpu_attention_kernels.py at the real width w (same per-element bounds, TAU,
NaN-prefilled outputs, every case run twice for identical bits): widths 1 ... 255 that reach every DK (16, 32, 64, 96,
128, 192, 256), S from 1 to 4096, the pad columns of the context and of dQ | dK | dV exactly +0, and the padded QKV
bias gradient +0 in its pads.  At widths that are multiples of 4 the padded entry points are the unpadded ones, bit for
bit.  On an H100 80GB HBM3 (power limit 700 W) the worst error / bound over the kernel cases is 0.98 (row max at width
2, where the bound's 2 * 2^-24 sum |q||k| is tightest; width 1 is exact), 0.96 (O), 0.79 (dV), 0.71 (dK), 0.69 (dQ)
and 0.40 (QKV bias gradient); the whole file takes about 3 minutes there.

Scorer: d 144 / h 8 (w 18), d 96 / h 32 (w 3), d 200 / h 8 (w 25) and d 260 / h 2 (w 130) in train mode with dropout,
attention modes 0, 1 and 2 against the TF32 emulation under the regenerated masks and against each other (the bounds of
test_gpu_attention_narrow.py), training at S = 2048 and 4096, repeated steps, a graphed dropout step, frozen
parameters, and the golden vectors of the unmodified reference (tests/golden/scorer_odd_heads.npz, written by
tools/make_golden_odd_heads.py)."""
import ctypes
import json

import numpy as np
import pytest
import torch

from tests.test_gpu_attention_kernels import (  # noqa: F401  (lib: the module's fixture)
    SEED, LAYER, bwd_case, check_backward, check_forward, fwd_case, lib, run_bwd, run_fwd, same_bits)
from tests.test_gpu_attention_narrow import _emulate, narrow_extents
from tests.test_gpu_attention_wide import _model, _rel, _set_attention_mode, _slates

gpu = pytest.mark.gpu
pytestmark = gpu


@pytest.fixture(scope="module")
def plib(lib):
    c_p, c_i, c_f, c_u = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float, ctypes.c_uint64
    lib.register("arb_attention_padded_forward", c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_f, c_u, c_i, c_p, c_p, c_p,
                                                       c_p])
    lib.register("arb_attention_padded_backward", c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_f, c_u,
                                                        c_i, c_p, c_p, c_p, c_p])
    return lib


def hs_of(w):
    return (w + 3) // 4 * 4


def pad_heads(t, n, h, w):
    """[rows, n*h*w] -> [rows, n*h*hs]: every head followed by hs - w zero columns."""
    rows, hs = t.shape[0], hs_of(w)
    out = torch.zeros(rows, n, h, hs, dtype=t.dtype, device=t.device)
    out[..., :w] = t.view(rows, n, h, w)
    return out.reshape(rows, n * h * hs)


def split_heads(t, n, h, w):
    """[rows, n*h*hs] -> (real [rows, n*h*w], pads [rows, n, h, hs - w])"""
    v = t.view(t.shape[0], n, h, hs_of(w))
    return v[..., :w].reshape(t.shape[0], n * h * w), v[..., w:]


def assert_pos_zero(t, what):
    z = t.float().contiguous()
    assert torch.equal(z.view(torch.int32), torch.zeros_like(z).view(torch.int32)), f"{what} are not +0"


def run_pfwd(L, qkv_p, mask, ext, B, S, h, w, p):
    dp = h * hs_of(w)
    ctx = torch.full((B * S, dp), float("nan"), device="cuda")
    smax = torch.full((B, h, S), float("nan"), device="cuda")
    ssum = torch.full((B, h, S), float("nan"), device="cuda")
    rc = L.lib().arb_attention_padded_forward(L.ptr(qkv_p), L.ptr(mask), L.ptr(ext), B, S, h, w, p, SEED, LAYER,
                                              L.ptr(ctx), L.ptr(smax), L.ptr(ssum), L.stream_ptr())
    L.check(rc, "arb_attention_padded_forward")
    torch.cuda.synchronize()
    return ctx, smax, ssum


def run_pbwd(L, qkv_p, ctx_p, dctx_p, mask, ext, smax, ssum, B, S, h, w, p, dbias_p):
    dp = h * hs_of(w)
    d_qkv = torch.full((B * S, 3 * dp), float("nan"), device="cuda")
    dbias = dbias_p.clone()
    delta = torch.full((B, h, S), float("nan"), device="cuda")
    rc = L.lib().arb_attention_padded_backward(L.ptr(qkv_p), L.ptr(ctx_p), L.ptr(dctx_p), L.ptr(mask), L.ptr(ext),
                                               L.ptr(smax), L.ptr(ssum), B, S, h, w, p, SEED, LAYER, L.ptr(d_qkv),
                                               L.ptr(dbias), L.ptr(delta), L.stream_ptr())
    L.check(rc, "arb_attention_padded_backward")
    torch.cuda.synchronize()
    return d_qkv, dbias


# ------------------------------------------------------------------------------------------------ kernels
WIDTHS = [1, 2, 3, 5, 6, 7, 9, 17, 18, 25, 33, 50, 66, 101, 126, 130, 191, 255]
KCASES = [(w, S, p) for w in WIDTHS for S in (1, 37, 240, 256, 257, 1024) for p in (0.0, 0.1)]
KCASES += [(3, 4096, 0.1), (18, 4096, 0.0), (130, 4096, 0.1)]


@pytest.mark.parametrize("w,S,p", KCASES, ids=[f"w{w}-S{S}-p{p}" for w, S, p in KCASES])
def test_padded_kernels_match_fp64_reference(plib, w, S, p):
    ex = narrow_extents(S)
    B = len(ex)
    h = (3 if S <= 1024 else 2) if w <= 32 else (2 if S <= 1024 else 1)
    seed = w * 10000 + S + int(p * 10) + 555
    qkv, mask, ext, R = fwd_case(plib, ex, S, h, w, p, seed=seed)
    qkv_p = pad_heads(qkv, 3, h, w)
    out = run_pfwd(plib, qkv_p, mask, ext, B, S, h, w, p)
    again = run_pfwd(plib, qkv_p, mask, ext, B, S, h, w, p)
    assert all(same_bits(a, b) for a, b in zip(out, again)), "two forward runs differ"
    ctx, cpad = split_heads(out[0], 1, h, w)
    assert_pos_zero(cpad, "pad columns of the context")
    check_forward(f"padded fwd w{w} S{S} p{p}", R, ctx, out[1], out[2], B, S, h, w)
    del R
    torch.cuda.empty_cache()
    # backward on the reference's statistics and context (a wrong forward cannot hide a wrong backward)
    args, Rb, gext = bwd_case(plib, ex, S, h, w, p, seed=seed + 7)
    qkv, ctx, d_ctx, mask, gx, smax, ssum = args[:7]
    db0 = args[-1]
    pargs = (pad_heads(qkv, 3, h, w), pad_heads(ctx, 1, h, w), pad_heads(d_ctx, 1, h, w), mask, gx, smax, ssum,
             B, S, h, w, p, pad_heads(db0[None], 3, h, w)[0])
    d_qkv, dbias = run_pbwd(plib, *pargs)
    d2, b2 = run_pbwd(plib, *pargs)
    assert same_bits(d_qkv, d2) and same_bits(dbias, b2), "two backward runs differ"
    g, gpad = split_heads(d_qkv, 3, h, w)
    assert_pos_zero(gpad, "pad columns of dQ | dK | dV")
    b, bpad = split_heads(dbias[None], 3, h, w)
    assert_pos_zero(bpad, "pad entries of the QKV bias gradient")
    check_backward(f"padded bwd w{w} S{S} p{p}", Rb, g, b[0], db0, gext, B, S, h, w)


@pytest.mark.parametrize("w,S,p", [(4, 37, 0.1), (16, 240, 0.1), (72, 1024, 0.0), (256, 257, 0.1)])
def test_padded_entry_points_are_the_plain_ones_at_multiples_of_4(plib, w, S, p):
    ex = narrow_extents(S)
    B, h = len(ex), 2
    args, _, _ = bwd_case(plib, ex, S, h, w, p, seed=w + S)
    qkv, mask, gx = args[0], args[3], args[4]
    a = run_fwd(plib, qkv, mask, gx, B, S, h, w, p)
    b = run_pfwd(plib, qkv, mask, gx, B, S, h, w, p)
    assert all(same_bits(x, y) for x, y in zip(a, b))
    ga, ba = run_bwd(plib, *args)
    gb, bb = run_pbwd(plib, *args)
    assert same_bits(ga, gb) and same_bits(ba, bb)


@pytest.mark.parametrize("w", [0, 257])
def test_padded_entry_points_refuse_widths_outside_1_to_256(plib, w):
    x = torch.zeros(16, device="cuda")
    m = torch.zeros(16, dtype=torch.uint8, device="cuda")
    rc = plib.lib().arb_attention_padded_forward(plib.ptr(x), plib.ptr(m), None, 1, 1, 1, w, 0.0, 1, 0, plib.ptr(x),
                                                 plib.ptr(x), plib.ptr(x), plib.stream_ptr())
    assert rc != 0 and "[1, 256]" in plib.lib().arb_last_error().decode()


# ------------------------------------------------------------------------------------------------ scorer
# (d_model, n_heads, N, d_ff)
MODELS = {"d144h8": (144, 8, 2, 576), "d96h32": (96, 32, 2, 384), "d200h8": (200, 8, 2, 400), "d260h2": (260, 2, 1, 520)}


def _odd_model(name, p, seed=29, N=None):
    d, h, n, dff = MODELS[name]
    return _model(136, d, N or n, h, dff, p, seed=seed)


@pytest.mark.parametrize("name", list(MODELS))
def test_scorer_matches_the_unfused_path_and_the_emulation(name, monkeypatch):
    """Train mode at S = 240 with attention dropout 0.1: modes 2, 1 and 0 against the TF32 emulation run with the same
    dropout masks (scores, prepare_for_output, x.grad, every parameter gradient) and modes 1 and 2 against mode 0, with
    the tolerances of test_gpu_attention_narrow's scorer test."""
    from tests.dropout_masks import scorer_masks
    B, S, F, p = 4, 240, 136, 0.1
    d, h, N, dff = MODELS[name]
    seed = 0x5DEECE66D
    model = _odd_model(name, p)
    monkeypatch.setattr(model, "_draw_seed", lambda: seed)
    x0, y = _slates(B, S, F, seed=13)
    mask = y == -1
    g = torch.Generator(device="cuda").manual_seed(3)
    w = torch.randn(B, S, device="cuda", generator=g) * (~mask).float()
    wh = torch.randn(B, S, d, device="cuda", generator=g)
    out = {}
    try:
        for mode in (0, 1, 2):
            _set_attention_mode(mode)
            model.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(True)
            s = model(x, mask, None)
            (s * w).sum().backward()
            grads = {k: q.grad.clone() for k, q in model.named_parameters()}
            xs = x.grad.clone()
            flat = model.flat_gradients.clone()
            x = x0.clone().requires_grad_(True)
            hid = model.prepare_for_output(x, mask, None)
            (hid * wh).sum().backward()
            out[mode] = (s.detach().clone(), flat, xs, hid.detach().clone(), x.grad.clone(), grads)
    finally:
        _set_attention_mode(2)
    drop = {k: None if v is None else v.cuda() for k, v in scorer_masks(seed, B, S, [d], N, h, dff, p, 0.0).items()}
    es, egrads, exs, eh, exh = _emulate(model, x0, mask, w, wh, N, h, drop)
    real = ~mask
    for mode in (0, 1, 2):
        s1, _, xs1, h1, xh1, grads = out[mode]
        rs, rx, rh, rxh = _rel(s1[real], es[real]), _rel(xs1, exs), _rel(h1[real], eh[real]), _rel(xh1, exh)
        worst = {}
        for k, q in grads.items():
            r = egrads[k]
            if r is None or ".self_attn.linears.1.bias" in k:   # the key bias gradient is analytically zero
                continue
            worst[k] = _rel(q, r)
        print(name, "mode", mode, "vs emulation: scores", rs, "x.grad", rx, "hidden", rh, "x.grad (hidden)", rxh,
              "worst param", max(worst.items(), key=lambda kv: kv[1]))
        assert rs <= 1e-3 and rh <= 1e-3 and rx <= 5e-2 and rxh <= 5e-2, (mode, rs, rh, rx, rxh)
        for k, e in worst.items():
            assert e <= (1e-1 if ".feed_forward.w_1." in k else 5e-2), (mode, k, e)
    for mode in (1, 2):
        s0, g0, xs0, h0, xh0, _ = out[0]
        s1, g1, xs1, h1, xh1, _ = out[mode]
        assert (s0 - s1).abs().max().item() <= 2e-3 * max(1.0, s0.abs().max().item())
        assert (h0 - h1).abs().max().item() <= 2e-3 * max(1.0, h0.abs().max().item())
        assert _rel(xs1, xs0) <= 5e-2 and _rel(xh1, xh0) <= 5e-2
    g0, g1, g2 = out[0][1], out[1][1], out[2][1]
    assert _rel(g2, g1) <= 1.5e-2, "the fused backward's flat gradient against the unfused backward's"
    assert _rel(g2, g0) <= max(1.5e-2, 1.1 * _rel(g1, g0))


@pytest.mark.parametrize("S", [2048, 4096])
def test_training_beyond_the_unfused_limit(S):
    """S > 1536 at width 18: a training step's scores, x.grad and parameter gradients against the TF32 emulation,
    then an optimiser step."""
    from allrank_b200.optim import FlatAdam
    from oracle.tf32_emulation import scorer_forward
    F, B, N = 136, 2, 1
    _, h, _, _ = MODELS["d144h8"]
    model = _odd_model("d144h8", 0.0, N=N)
    x0, y = _slates(B, S, F, seed=17)
    mask = y == -1
    w = torch.randn(B, S, generator=torch.Generator().manual_seed(4)).cuda() * (~mask).float()
    x = x0.clone().requires_grad_(True)
    s = model(x, mask, None)
    (s * w).sum().backward()
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    xe = x0.clone().requires_grad_(True)
    ref = scorer_forward(sd, xe, mask, N, h, None, "rna")
    (ref * w).sum().backward()
    real = ~mask
    es, ex = _rel(s.detach()[real], ref.detach()[real]), _rel(x.grad, xe.grad)
    print("d144h8", S, "scores rel err", es, "x.grad rel err", ex)
    assert es <= 1e-3 and ex <= 1e-2, (es, ex)
    for k, q in model.named_parameters():
        r = sd[k].grad
        if r is None or ".self_attn.linears.1.bias" in k:
            continue
        e = _rel(q.grad, r)
        assert e <= (1e-1 if ".feed_forward.w_1." in k else 5e-2), (k, e)
    del sd, xe, ref
    before = model.flat_parameters.clone()
    FlatAdam(model, lr=1e-3).step()
    assert torch.isfinite(model.flat_parameters).all() and not torch.equal(before, model.flat_parameters)


@pytest.mark.parametrize("name,S", [("d96h32", 240), ("d200h8", 1024)])
def test_two_training_steps_give_the_same_bits(name, S, monkeypatch):
    """The same step twice from the same state, with attention dropout: scores and flat gradients are the same bits
    (the padded gradients reach the flat buffer in a fixed order)."""
    from allrank_b200 import losses
    x, y = _slates(8, S, 136, seed=23)
    model = _odd_model(name, 0.1)
    monkeypatch.setattr(model, "_draw_seed", lambda: 4242)
    out = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        s = model(x, y == -1, None)
        losses.approxNDCGLoss(s, y).backward()
        out.append((s.detach().clone(), model.flat_gradients.clone()))
    assert same_bits(out[0][0], out[1][0]) and same_bits(out[0][1], out[1][1])


def test_graphed_dropout_training_at_width_18(monkeypatch):
    """GraphedTrainStep(dropout_seed=s) at width 18, S = 240: replay k equals an eager step seeded s + k."""
    from allrank_b200 import losses
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.optim import FlatAdam
    batches = [_slates(8, 240, 136, seed=20 + k) for k in range(2)] * 2
    s = 977

    eager = _odd_model("d144h8", 0.3)
    opt = FlatAdam(eager, lr=1e-3, capturable=True)
    eager_losses = []
    for k, (x, y) in enumerate(batches, start=1):
        monkeypatch.setattr(eager, "_draw_seed", lambda k=k: s + k)
        loss = losses.approxNDCGLoss(eager(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        eager_losses.append(loss.item())

    graphed = _odd_model("d144h8", 0.3)
    gopt = FlatAdam(graphed, lr=1e-3, capturable=True)
    init = {k: v.clone() for k, v in graphed.state_dict().items()}
    monkeypatch.setattr(graphed, "_draw_seed", lambda: pytest.fail("the graphed step drew a host seed"))
    step = GraphedTrainStep(graphed, losses.approxNDCGLoss, gopt, *batches[0], warmup=2, dropout_seed=s)
    graphed.load_state_dict(init)
    gopt.exp_avg.zero_(); gopt.exp_avg_sq.zero_(); gopt._dev_state.zero_()
    graph_losses = [step(x, y).item() for x, y in batches]
    assert graph_losses == eager_losses
    assert torch.equal(graphed.flat_parameters, eager.flat_parameters)


def test_frozen_parameters_give_x_grad_only():
    """Every parameter frozen: no parameter gradient is computed, and x.grad is the same bits as with gradients on."""
    model = _odd_model("d96h32", 0.0).eval()
    x0, y = _slates(4, 240, 136, seed=41)
    mask = y == -1
    w = torch.randn(4, 240, generator=torch.Generator().manual_seed(5)).cuda()
    x = x0.clone().requires_grad_(True)
    (model(x, mask, None) * w).sum().backward()
    want = x.grad.clone()
    for q in model.parameters():
        q.requires_grad_(False)
    x = x0.clone().requires_grad_(True)
    (model(x, mask, None) * w).sum().backward()
    assert same_bits(x.grad, want)


# ------------------------------------------------------------------------------------------------ golden vectors
def _golden_model(g, name):
    from allrank_b200.model import make_model
    m = json.loads(str(g[name + ":model"]))
    torch.manual_seed(87)
    model = make_model(fc_model=m["fc_model"], transformer=m["transformer"], post_model=m["post_model"], n_features=136)
    gen = torch.Generator().manual_seed(88)
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    return model


@pytest.mark.parametrize("name", ["d144h8", "d96h32"])
def test_eval_matches_the_reference_golden_vectors(golden, name):
    """The unmodified reference's scores within the TF32 bound (5e-3 at unit scale) and every parameter gradient
    (sampled positions and norm) within 5 % of the largest per-element gradient scale, as test_shipped_configs."""
    g = golden("scorer_odd_heads")
    model = _golden_model(g, name)
    for k, v in model.state_dict().items():      # the same initialisation as the reference's
        got = np.array([v.double().sum().item(), v.double().abs().sum().item()])
        assert np.array_equal(got, g[name + ":c:" + k]), k
    model = model.cuda().eval()
    x, y = torch.tensor(g["x"]).cuda(), torch.tensor(g["y"]).cuda()
    out = model(x, y == -1, None)
    ref = torch.tensor(g[name + ":scores"])
    valid = (y != -1).cpu()
    err = (out.detach().cpu() - ref)[valid].abs().max().item()
    assert err <= 5e-3 * max(1.0, ref[valid].abs().max().item()), err
    (out * torch.tensor(g[name + ":w"]).cuda()).sum().backward()
    params = dict(model.named_parameters())
    rms_max = max(float(g[name + ":n:" + k]) / np.sqrt(p.numel()) for k, p in params.items())
    worst = 0.0
    for k, p in params.items():
        n = p.numel()
        gi = torch.arange(n) if n <= 1024 else torch.linspace(0, n - 1, 1024).long()
        got = p.grad.detach().flatten().cpu()[gi].double().numpy()
        want = g[name + ":g:" + k].astype(np.float64)
        floor = 1e-2 * rms_max * np.sqrt(len(gi))
        fro = np.linalg.norm(got - want) / max(np.linalg.norm(want), floor)
        nrm = abs(p.grad.norm().item() - float(g[name + ":n:" + k])) / max(float(g[name + ":n:" + k]),
                                                                           1e-2 * rms_max * np.sqrt(n))
        worst = max(worst, fro)
        assert fro <= 5e-2 and nrm <= 5e-2, (k, fro, nrm)
    print(name, "score err", err, "worst sampled gradient rel err", worst)
