"""The fused attention kernels of slates longer than 256 items (csrc/attention_long.cu: attn_long_fwd_kernel,
attn_long_dkdv_kernel, attn_long_dq_kernel) against the fp64 reference of tests/test_gpu_attention_kernels.py (same
per-element bounds, TAU, NaN-prefilled outputs, every case run twice for identical bits), against the short kernels bit
for bit on slates both serve, and through the scorer against the unfused path and the TF32 emulation, including
slates beyond the unfused path's 1536 items."""
import ctypes

import pytest
import torch

from tests.test_gpu_attention_kernels import (  # noqa: F401  (lib: the module's fixture)
    TAU, bwd_case, bits, check, check_backward, check_forward, colsum_and_bound, fwd_case, heads, lib, make_dctx,
    make_inputs, reference, reference_bwd, run_bwd, run_fwd, same_bits)

pytestmark = pytest.mark.gpu


def long_extents(S):
    """Extents on both sides of 16-row strips, 128-row tiles / key blocks and the short kernels' 256 rows."""
    cand = {1, 15, 17, 127, 128, 129, 255, 256, 257, 383, 640, 1025, S - 1, S}
    if S >= 2048:                     # the fp64 reference holds B * h * S^2 doubles per tensor
        cand = {129, 1025, S - 1, S}
    return sorted(e for e in cand if 1 <= e <= S)


CASES = [(dk, S, p) for S in (257, 300, 1024, 1536, 2048, 4096) for dk in (16, 32) for p in (0.0, 0.1, 0.3)]


@pytest.mark.parametrize("dk,S,p", CASES, ids=[f"dk{dk}-S{S}-p{p}" for dk, S, p in CASES])
def test_forward_and_backward_match_fp64_reference(lib, dk, S, p):
    ex = long_extents(S)
    B, h = len(ex), (1 if S >= 2048 else 2)
    seed = dk * 10000 + S + int(p * 10)
    qkv, mask, ext, R = fwd_case(lib, ex, S, h, dk, p, seed=seed)
    out = run_fwd(lib, qkv, mask, ext, B, S, h, dk, p)
    again = run_fwd(lib, qkv, mask, ext, B, S, h, dk, p)
    assert all(same_bits(a, b) for a, b in zip(out, again)), "two forward runs differ"
    check_forward(f"long fwd dk{dk} S{S} p{p}", R, *out, B, S, h, dk)
    del R
    torch.cuda.empty_cache()
    args, Rb, gext = bwd_case(lib, ex, S, h, dk, p, seed=seed + 7)
    d_qkv, dbias = run_bwd(lib, *args)
    d2, b2 = run_bwd(lib, *args)
    assert same_bits(d_qkv, d2) and same_bits(dbias, b2), "two backward runs differ"
    assert any(g > e for g, e in zip(gext, ex)), "no backward extent past the key extent"
    check_backward(f"long bwd dk{dk} S{S} p{p}", Rb, d_qkv, dbias, args[-1], gext, B, S, h, dk)


def test_all_padded_slate(lib):
    """A slate without real items: NaN context rows, row max -inf, row sum 0, exactly zero gradients."""
    S, h, dk = 300, 2, 32
    ex = [300, 1, 200]
    B = len(ex)
    qkv, mask, _, _ = fwd_case(lib, ex, S, h, dk, 0.0, seed=5)
    mask[1] = 1
    R = reference(qkv, mask, B, S, h, dk, None)
    ext = torch.tensor([300, 0, 200], dtype=torch.int32, device="cuda")
    ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, dk, 0.0)
    assert torch.isnan(ctx.view(B, S, -1)[1]).all()
    assert (smax[1] == float("-inf")).all() and (ssum[1] == 0).all()
    check_forward("long all-padded fwd", R, ctx, smax, ssum, B, S, h, dk)
    gext = [300, 0, 200]
    d_ctx = make_dctx(gext, S, h * dk, 6)
    Rb = reference_bwd(R, d_ctx, ctx, B, S, h, dk)
    d_qkv, _ = run_bwd(lib, qkv, ctx, d_ctx, mask, ext, smax, ssum, B, S, h, dk, 0.0, None)
    g = d_qkv.view(B, S, 3 * h * dk)
    assert torch.equal(bits(g[1]), torch.zeros_like(bits(g[1]))), "gradients of the all-padded slate are not +0"
    keep = torch.tensor([0, 2], device="cuda")
    sub = {k: v[keep] for k, v in Rb.items()}
    check_backward("long all-padded bwd", sub, d_qkv.view(B, S, -1)[keep].reshape(2 * S, -1), None, None, [300, 200],
                   2, S, h, dk)


def test_truncating_tf32_operands(lib):
    """arb_set_tf32_round_on_load(0): the tensor core truncates; within the bounds of the truncation emulation."""
    S, h, dk, p = 300, 2, 32, 0.1
    ex = long_extents(S)
    B = len(ex)
    try:
        lib.lib().arb_set_tf32_round_on_load(0)
        qkv, mask, ext, R = fwd_case(lib, ex, S, h, dk, p, seed=78, mode="trunc")
        check_forward("long trunc fwd", R, *run_fwd(lib, qkv, mask, ext, B, S, h, dk, p), B, S, h, dk)
        args, Rb, gext = bwd_case(lib, ex, S, h, dk, p, seed=79, mode="trunc")
        d_qkv, dbias = run_bwd(lib, *args)
        check_backward("long trunc bwd", Rb, d_qkv, dbias, args[-1], gext, B, S, h, dk)
    finally:
        lib.lib().arb_set_tf32_round_on_load(1)


def _embed(t, B, S0, S, fill):
    """[B*S0, w] rows -> [B*S, w] with rows S0 ... S-1 of every slate set to `fill`."""
    w = t.shape[-1]
    out = torch.full((B, S, w), fill, dtype=t.dtype, device=t.device)
    out[:, :S0] = t.view(B, S0, w)
    return out.reshape(B * S, w)


@pytest.mark.parametrize("dk", [16, 32])
def test_same_bits_as_the_short_kernels(lib, dk):
    """Slates of at most 256 items in an S = 256 batch (short kernels) and in S = 300 / 1024 batches (the long
    kernels): context, row statistics, dQ, dK and dV of rows 0 ... 255 are the same bits; the bias gradient is summed
    in another order and checked to its bound."""
    S0, h = 256, 2
    ex = [1, 16, 17, 100, 128, 129, 200, 255, 256, 256]
    B, d = len(ex), h * dk
    qkv0, mask0, ext = make_inputs(ex, S0, h, dk, seed=40 + dk)
    gext = [min(S0, e + 3) if b % 3 == 1 else e for b, e in enumerate(ex)]
    d_ctx0 = make_dctx(gext, S0, d, 41)
    gx = torch.tensor(gext, dtype=torch.int32, device="cuda")
    db0 = torch.zeros(3 * d, device="cuda")
    res = {}
    for S in (S0, 300, 1024):
        qkv = _embed(qkv0, B, S0, S, 7.0)          # garbage in the rows past 256: masked, beyond every extent
        mask = torch.ones(B, S, dtype=torch.uint8, device="cuda")
        mask[:, :S0] = mask0
        d_ctx = _embed(d_ctx0, B, S0, S, 0.0)
        ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, dk, 0.0)
        d_qkv, dbias = run_bwd(lib, qkv, ctx, d_ctx, mask, gx, smax, ssum, B, S, h, dk, 0.0, db0)
        res[S] = (ctx.view(B, S, d)[:, :S0], smax[..., :S0], ssum[..., :S0], d_qkv.view(B, S, 3 * d)[:, :S0],
                  dbias, d_qkv)
        if S > S0:
            assert (d_qkv.view(B, S, 3 * d)[:, S0:] == 0).all()
    for S in (300, 1024):
        for i, name in enumerate(("ctx", "stat_max", "stat_sum", "dQ|dK|dV")):
            assert same_bits(res[S][i], res[S0][i]), f"S={S}: {name} differs from the short kernels"
        want, acc_b = colsum_and_bound(res[S][5], db0)
        check(f"S={S} dbias/own", res[S][4], want, acc_b / TAU)
        check(f"S={S} dbias vs short", res[S][4], res[S0][4].double(), 2 * acc_b / TAU)   # two orders of one sum


# ------------------------------------------------------------------------------------------------ scorer
def _set_attention_mode(mode):
    from allrank_b200 import _lib
    L = _lib.lib()
    L.arb_set_attention_mode.argtypes = [ctypes.c_int32]
    L.arb_set_attention_mode(mode)


def _model(F, d, N, h, dff, p, seed=29):
    from allrank_b200.model import make_model
    torch.manual_seed(seed)
    return make_model(fc_model={"sizes": [d], "input_norm": False, "activation": None, "dropout": 0.0},
                      transformer={"N": N, "d_ff": dff, "h": h, "positional_encoding": None, "dropout": p},
                      post_model={"d_output": 1, "output_activation": None}, n_features=F).cuda().train()


def _slates(B, S, F, seed):
    from allrank_b200.synth import make_slates
    x, y, _ = make_slates(B, S, n_features=F, seed=seed, mean_len=0.6 * S, std_len=0.3 * S)
    return x.cuda(), y.cuda()


def _rel(a, b):
    return (a - b).norm().item() / max(b.norm().item(), 1e-30)


@pytest.mark.parametrize("S,p,dk", [(300, 0.0, 32), (300, 0.3, 16), (1024, 0.0, 16), (1024, 0.3, 32)])
def test_scorer_matches_the_unfused_path(S, p, dk, monkeypatch):
    """Modes 2 (fused forward and backward) and 1 (fused forward) against mode 0 (materialised S x S), train mode, the
    same dropout masks: scores and flat gradients with the tolerances of test_gpu_scorer's fused-vs-unfused test,
    prepare_for_output and x.grad as well."""
    F, d, N, B = 136, 64, 2, 4
    model = _model(F, d, N, d // dk, 128, p)
    monkeypatch.setattr(model, "_draw_seed", lambda: 0x5DEECE66D)
    x0, y = _slates(B, S, F, seed=13)
    mask = y == -1
    g = torch.Generator(device="cuda").manual_seed(3)
    w = torch.randn(B, S, device="cuda", generator=g)
    wh = torch.randn(B, S, d, device="cuda", generator=g)
    out = {}
    try:
        for mode in (0, 1, 2):
            _set_attention_mode(mode)
            model.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(True)
            s = model(x, mask, None)
            (s * w).sum().backward()
            xs = x.grad.clone()
            x = x0.clone().requires_grad_(True)
            hid = model.prepare_for_output(x, mask, None)
            (hid * wh).sum().backward()
            out[mode] = (s.detach().clone(), model.flat_gradients.clone(), xs, hid.detach().clone(), x.grad.clone())
    finally:
        _set_attention_mode(2)
    for mode in (1, 2):
        s0, g0, xs0, h0, xh0 = out[0]
        s1, g1, xs1, h1, xh1 = out[mode]
        ds = (s0 - s1).abs().max().item()
        dh = (h0 - h1).abs().max().item()
        print(S, p, dk, "mode", mode, "score diff", ds, "grad", _rel(g1, g0), "x.grad", _rel(xs1, xs0), "hidden", dh,
              "x.grad (hidden)", _rel(xh1, xh0))
        assert ds <= 2e-3 * max(1.0, s0.abs().max().item())
        assert dh <= 2e-3 * max(1.0, h0.abs().max().item())
        assert _rel(g1, g0) <= 1.5e-2
        # x.grad: the tolerance test_gpu_autograd holds it to against the reference (dropout at p = 0.3 amplifies
        # the TF32 differences of the two paths: up to 2.2e-2 observed on an H100)
        assert _rel(xs1, xs0) <= 5e-2 and _rel(xh1, xh0) <= 5e-2


@pytest.mark.parametrize("S,h", [(2048, 2), (4096, 4)])
def test_slates_beyond_the_unfused_limit(S, h):
    """S > 1536 (where the unfused softmax stops): scores, x.grad and the parameter gradients against the TF32
    emulation on the host."""
    from oracle.tf32_emulation import scorer_forward
    F, d, B = 136, 64, 2
    model = _model(F, d, 1, h, 128, 0.0).eval()
    x0, y = _slates(B, S, F, seed=17)
    mask = y == -1
    w = torch.randn(B, S, generator=torch.Generator().manual_seed(4)).cuda() * (~mask).float()
    x = x0.clone().requires_grad_(True)
    s = model(x, mask, None)
    (s * w).sum().backward()
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    xe = x0.cpu().clone().requires_grad_(True)
    ref = scorer_forward(sd, xe, mask.cpu(), 1, h, None, "rna")
    (ref * w.cpu()).sum().backward()
    real = (~mask).cpu()
    es = _rel(s.detach().cpu()[real], ref.detach()[real])
    ex = _rel(x.grad.cpu(), xe.grad)
    print(S, h, "scores rel err", es, "x.grad rel err", ex)
    assert es <= 1e-3 and ex <= 1e-2, (es, ex)
    for k, q in model.named_parameters():
        r = sd[k].grad
        if r is None or ".self_attn.linears.1.bias" in k:   # the key bias gradient is analytically zero: rounding only
            continue
        e = _rel(q.grad.cpu(), r)
        assert e <= (1e-1 if ".feed_forward.w_1." in k else 5e-2), (k, e)


def test_training_step_and_metrics_at_4096():
    from allrank_b200 import losses, metrics
    from allrank_b200.optim import FlatAdam
    S, B = 4096, 2
    x, y = _slates(B, S, 136, seed=19)
    for loss_fn in (losses.approxNDCGLoss, losses.listNet):
        model = _model(136, 64, 1, 4, 128, 0.1)
        opt = FlatAdam(model, lr=1e-3)
        params = lambda: torch.cat([q.detach().flatten() for q in model.parameters()])  # noqa: E731
        before = params()
        loss = loss_fn(model(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        assert torch.isfinite(model.flat_gradients).all() and model.flat_gradients.abs().sum() > 0
        opt.step()
        assert torch.isfinite(loss) and torch.isfinite(params()).all()
        assert not torch.equal(before, params())
        with torch.no_grad():
            nd = metrics.ndcg(model.eval()(x, y == -1, None), y, ats=[5, 60])
        assert torch.isfinite(nd).all() and (nd >= 0).all() and (nd <= 1 + 1e-6).all()


def test_workspace_drops_the_probability_buffers():
    from allrank_b200 import _lib
    F, d, N, h, B, S = 136, 64, 2, 2, 8, 1024
    model = _model(F, d, N, h, 128, 0.0)
    cfg = ctypes.byref(model._cfg)
    sizes = {}
    try:
        for mode in (0, 2):
            _set_attention_mode(mode)
            sizes[mode] = int(_lib.lib().arb_scorer_workspace_floats(cfg, B, S, 1))
    finally:
        _set_attention_mode(2)
    prob = B * h * S * ((S + 3) // 4 * 4)     # [B, h, S, round_up(S, 4)] per layer
    assert sizes[0] - sizes[2] == N * ((prob + 63) // 64 * 64), sizes


def test_graphed_dropout_training_at_1024(monkeypatch):
    """GraphedTrainStep(dropout_seed=s): replay k equals an eager step seeded s + k."""
    from allrank_b200 import losses
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.optim import FlatAdam
    batches = [_slates(4, 1024, 136, seed=20 + k) for k in range(2)] * 2
    s = 977

    eager = _model(136, 64, 1, 2, 128, 0.3)
    opt = FlatAdam(eager, lr=1e-3, capturable=True)
    eager_losses = []
    for k, (x, y) in enumerate(batches, start=1):
        monkeypatch.setattr(eager, "_draw_seed", lambda k=k: s + k)
        loss = losses.approxNDCGLoss(eager(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        eager_losses.append(loss.item())

    graphed = _model(136, 64, 1, 2, 128, 0.3)
    gopt = FlatAdam(graphed, lr=1e-3, capturable=True)
    init = {k: v.clone() for k, v in graphed.state_dict().items()}
    monkeypatch.setattr(graphed, "_draw_seed", lambda: pytest.fail("the graphed step drew a host seed"))
    step = GraphedTrainStep(graphed, losses.approxNDCGLoss, gopt, *batches[0], warmup=2, dropout_seed=s)
    graphed.load_state_dict(init)
    gopt.exp_avg.zero_(); gopt.exp_avg_sq.zero_(); gopt._dev_state.zero_()
    graph_losses = [step(x, y).item() for x, y in batches]
    assert graph_losses == eager_losses
    assert torch.equal(graphed.flat_parameters, eager.flat_parameters)


def test_bf16_context_beyond_256_is_refused(lib):
    S, h, dk = 300, 2, 32
    qkv, mask, ext = make_inputs([300], S, h, dk, seed=3)
    ctx = torch.zeros(S, h * dk, device="cuda", dtype=torch.bfloat16)
    smax = torch.zeros(1, h, S, device="cuda")
    rc = lib.lib().arb_attention_forward(lib.ptr(qkv), lib.ptr(mask), lib.ptr(ext), 1, S, h, dk, 0.0, 1, 0, 1,
                                         lib.ptr(ctx), lib.ptr(smax), lib.ptr(smax.clone()), lib.stream_ptr())
    assert rc != 0
