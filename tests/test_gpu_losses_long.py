"""Every loss kernel against the fp64 oracle (oracle/losses_ref.py) at slate lengths 1 to 4096.

The kernels are driven through the C ABI entry points allrank_b200/losses.py calls, with the gradient buffer filled
with NaN first, so an element a kernel fails to write cannot pass.  Every call runs twice and must give the same
bits, and the loss value must be the same bits without a gradient buffer.

The slate lengths straddle the warp / block switch of listNet (1280 items), the register, shared-memory and workspace
paths of neuralNDCG, the 256-thread row ownership of the pair loops and the bitonic sort's power-of-two padding.

Bounds (the contract of test_gpu_losses.py): loss within 1e-5 relative plus a 1e-7 floor, gradient within 2e-5 of
the largest reference entry on the real items (neuralNDCG 5e-4), padded items exactly 0.  Where the reference loss
is NaN (listNet or binary_listNet with an all-padded slate, rankNet or a `mean` lambdaLoss without a single pair),
the kernel must return NaN as well, and there is no gradient to compare.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

PAD = -1.0
EPS = 1e-10
SLATE_LENGTHS = [1, 2, 31, 32, 33, 127, 128, 129, 136, 255, 256, 257, 1024, 1280, 1281, 2048, 4096]
REL, FLOOR, GREL, GREL_NEURAL = 1e-5, 1e-7, 2e-5, 5e-4

LAMBDA_CASES = [
    {},
    {"weighing_scheme": "ndcgLoss1_scheme", "k": 20},
    {"weighing_scheme": "ndcgLoss2_scheme", "sigma": 2.0, "reduction_log": "natural"},
    {"weighing_scheme": "lambdaRank_scheme", "reduction": "mean", "reduction_log": "natural"},
    {"weighing_scheme": "ndcgLoss2PP_scheme", "mu": 5.0, "k": 10},
    {"weighing_scheme": "rankNet_scheme", "reduction": "mean"},
    {"weighing_scheme": "rankNetWeightedByGTDiff_scheme", "sigma": 0.5, "k": 100},
    {"weighing_scheme": "rankNetWeightedByGTDiffPowed_scheme"},
]
LOSS_CASES = ([("listNet", {}), ("listMLE", {}), ("approxNDCGLoss", {"alpha": 1.0}), ("approxNDCGLoss", {"alpha": 5.0})]
              + [("lambdaLoss", kw) for kw in LAMBDA_CASES]
              + [("rankNet", {}), ("rankNet_weightByGTDiff", {}), ("rankNet_weightByGTDiff_pow", {}),
                 ("binary_listNet", {}), ("pointwise_rmse", {"no_of_levels": 4}), ("bce", {}), ("ordinal", {"n": 4})])
NEURAL_CASES = [
    ("neuralNDCG", {}),
    ("neuralNDCG", {"k": 10, "powered_relevancies": False, "temperature": 0.5}),
    ("neuralNDCG_transposed", {}),
    ("neuralNDCG_transposed", {"k": 10, "powered_relevancies": False}),
]
TIE_FREE = ("approxNDCGLoss", "lambdaLoss")
POINTWISE = {"binary_listNet": 0, "pointwise_rmse": 1, "bce": 2}
RANKNET = {"rankNet": 0, "rankNet_weightByGTDiff": 1, "rankNet_weightByGTDiff_pow": 2}


def _id(case):
    name, kw = case
    return name + "".join(f"-{k}={v}" for k, v in kw.items())


# ------------------------------------------------------------------------------------------------ the kernels
def launch(name, kw, yp, yt, grad=True):
    """One call of the C ABI entry point behind losses.<name>.  Returns (loss, grad [B,S(,n)] or None, the per-slate
    values the kernel wrote before the batch reduction)."""
    from allrank_b200 import _lib, losses
    from allrank_b200.metrics import discount_table
    s = yp.float().contiguous().cuda()
    t = yt.float().contiguous().cuda()
    B, S = t.shape
    nan = float("nan")
    loss = torch.full((), nan, device="cuda")
    g = torch.full(s.shape, nan, device="cuda") if grad else None
    scratch = torch.full((2 * B,), nan, device="cuda")
    lib, P, st = _lib.lib(), _lib.ptr, _lib.stream_ptr(s.device)
    tail = (P(loss), P(g), P(scratch), st)
    if name == "listNet":
        rc = lib.arb_listnet(P(s), P(t), B, S, EPS, PAD, *tail)
    elif name == "listMLE":
        perm = kw["perm"].to("cuda", torch.int64).contiguous()
        order = kw["order"].to("cuda", torch.int32).contiguous()
        rc = lib.arb_listmle(P(s), P(t), B, S, EPS, PAD, P(perm), P(order), *tail)
    elif name == "approxNDCGLoss":
        rc = lib.arb_approx_ndcg(P(s), P(t), B, S, EPS, PAD, float(kw["alpha"]), *tail)
    elif name == "lambdaLoss":
        rc = lib.arb_lambda_loss(P(s), P(t), B, S, EPS, PAD, losses._SCHEMES[kw.get("weighing_scheme")],
                                 int(kw.get("k") or 0), float(kw.get("sigma", 1.0)), float(kw.get("mu", 10.0)),
                                 1 if kw.get("reduction") == "mean" else 0,
                                 1 if kw.get("reduction_log") == "natural" else 0, *tail)
    elif name.startswith("neuralNDCG"):
        powered = kw.get("powered_relevancies", True)
        mode = (1 if powered else 0) if name == "neuralNDCG" else (1 if powered else 2)
        max_iter = int(kw.get("max_iter", 50))
        ws_bytes = int(lib.arb_neural_ndcg_workspace_bytes(B, S, max_iter))
        ws = torch.full((ws_bytes // 4,), nan, device="cuda") if ws_bytes else None
        rc = lib.arb_neural_ndcg(P(s), P(t), B, S, P(discount_table(S, s.device)), PAD,
                                 float(kw.get("temperature", 1.0)), mode, int(kw.get("k") or 0), max_iter,
                                 float(kw.get("tol", 1e-6)), P(loss), P(g), P(scratch), P(ws), ws_bytes, st)
    elif name in RANKNET:
        rc = lib.arb_ranknet(P(s), P(t), B, S, PAD, RANKNET[name], *tail)
    elif name in POINTWISE:
        param = float(kw.get("no_of_levels", 0.0))
        rc = lib.arb_pointwise_loss(P(s), P(t), B, S, PAD, POINTWISE[name], param, EPS if name == "binary_listNet"
                                    else 0.0, *tail)
    elif name == "ordinal":
        rc = lib.arb_ordinal(P(s), P(t), B, S, int(kw["n"]), PAD, *tail)
    else:
        raise KeyError(name)
    _lib.check(rc, name)
    torch.cuda.synchronize()
    return loss.item(), (g.cpu().numpy() if grad else None), scratch.cpu().numpy()


def same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def run_kernel(name, kw, yp, yt):
    """Twice with a gradient (same bits), once without (same loss bits)."""
    val, grad, per = launch(name, kw, yp, yt)
    val2, grad2, per2 = launch(name, kw, yp, yt)
    val3, none, _ = launch(name, kw, yp, yt, grad=False)
    problems = []
    if not (same_bits(val, val2) and same_bits(grad, grad2) and same_bits(per, per2)):
        problems.append("two identical calls differ")
    if not same_bits(val, val3):
        problems.append(f"loss without a gradient {val3!r} != {val!r}")
    return val, grad, problems


# ------------------------------------------------------------------------------------------------ the reference
def reference(name, kw, yp, yt):
    """fp64 loss and gradient of the oracle (listMLE: the same shuffle and tie order as the kernel)."""
    from oracle import losses_ref
    p = yp.double().clone().requires_grad_(True)
    out = losses_ref.LOSSES[name](p, yt.double(), **kw)
    if out.requires_grad:
        out.backward()
    return out.item(), (p.grad if p.grad is not None else torch.zeros_like(p)).numpy()


def saturated_bce_reference(name, kw, yp, yt):
    """nn.BCELoss (what bce.py and ordinal.py call) on probabilities that include exact 0 and 1: it clamps the logs at
    -100 and its backward divides by max(p(1-p), 1e-12).  Autograd through the oracle's clamped logs gives 0 there."""
    import torch.nn.functional as F
    p = yp.double().clone().requires_grad_(True)
    valid = yt != PAD
    if name == "bce":
        target = torch.where(valid, yt, torch.zeros_like(yt)).double()
        per = F.binary_cross_entropy(p, target, reduction="none") * valid.double()
        out = per.sum() / valid.any(dim=1).double().sum()
    else:
        n = int(kw["n"])
        target = ((yt[:, :, None] >= torch.arange(1, n + 1, dtype=yt.dtype)) & valid[:, :, None]).double()
        per = F.binary_cross_entropy(p, target, reduction="none") * valid[:, :, None].double()
        out = per.sum() / valid.double().sum()
    out.backward()
    return out.item(), p.grad.numpy()


def compare(tag, val, grad, ref, gref, yt, gbound, worst):
    """Loss within REL (+FLOOR) of the reference, both NaN or neither; gradient within gbound of the largest reference
    entry on the real items, exactly 0 on the padded ones.  Returns a list of problems."""
    if math.isnan(ref) or math.isnan(val):
        return [] if math.isnan(ref) and math.isnan(val) else [f"{tag}: loss {val!r}, reference {ref!r}"]
    problems = []
    if not abs(val - ref) <= REL * abs(ref) + FLOOR:
        problems.append(f"{tag}: loss {val!r}, reference {ref!r}, rel {abs(val - ref) / max(abs(ref), 1e-30):.3g}")
    real = (yt != PAD).numpy()
    if grad.ndim == 3:
        real = np.broadcast_to(real[:, :, None], grad.shape)
    if not (grad[~real] == 0).all():
        problems.append(f"{tag}: padded items get {np.unique(grad[~real])[:4]}, not 0")
    if real.any():
        scale = float(np.abs(gref[real]).max())
        err = float(np.abs(grad[real] - gref[real]).max())        # NaN (an unwritten element) fails the tests below
        if scale == 0:
            # A reference gradient that is identically zero (listMLE with one valid item per slate: the loss does not
            # depend on the score) has no scale.  The kernel sums cancelling terms in fp32, e*C - 1 (which rounds to
            # 0) and the max-shift eps / (tail + eps), and leaves eps / B (1.56e-12 at B = 64, measured on an H100):
            # it must stay below eps.
            if not err <= EPS:
                problems.append(f"{tag}: gradient {err:.3g} where the reference gradient is 0")
            return problems
        worst[0] = max(worst[0], err / scale) if err == err else math.inf
        if not err <= gbound * scale:
            problems.append(f"{tag}: gradient error {err:.3g} against largest entry {scale:.3g} ({err / scale:.3g})")
    return problems


# ------------------------------------------------------------------------------------------------ inputs
def batch_for(S):
    """One fp64 [B,S,S] tensor of the pair-loss oracles stays at or below 2^23 elements (4096: B = 1)."""
    return max(1, min(64, 2 ** 23 // (S * S)))


def tie_free_scores(B, S, seed, scale=1.0):
    """randn scores without ties inside a slate (the oracle's sort leaves tied scores in an undefined order)."""
    while True:
        yp = torch.randn(B, S, generator=torch.Generator().manual_seed(seed), dtype=torch.float32) * scale
        if all(torch.unique(yp[b]).numel() == S for b in range(B)):
            return yp
        seed += 1000


def labels(B, S, kind, seed):
    from allrank_b200.synth import make_slates
    full = kind == "full"
    _, y, _ = make_slates(B, S, n_features=1, seed=seed, mean_len=0.6 * S, std_len=0.3 * S, full=full)
    if kind == "equal":                                         # no pair with different labels
        y = torch.where(y == PAD, y, torch.ones_like(y))
    elif kind == "edges":
        g = torch.Generator().manual_seed(seed + 1)
        for b in range(B):
            edge = b % 4
            if edge == 0:                                       # padding that is not a tail
                holes = torch.rand(S, generator=g) < 0.3
                holes[int(torch.randint(S, (1,), generator=g))] = False
                y[b] = torch.multinomial(torch.tensor([0.5, 0.3, 0.2]), S, replacement=True, generator=g).float()
                y[b][holes] = PAD
            elif edge == 1:                                     # a single valid item
                y[b] = PAD
                y[b, 0] = 2.0
            elif edge == 2:                                     # an all-padded slate among live ones
                y[b] = PAD
            else:                                               # a slate without a relevant item
                y[b] = torch.where(y[b] == PAD, y[b], torch.zeros_like(y[b]))
    return y


def kinds_for(S):
    """Inputs per slate length: random lengths and the edge batch everywhere; full slates, all-equal labels and
    scores scaled by 30 (sigmoid, eps and 1e8 clamps active; saturated probabilities) on a subset of the long ones."""
    if S <= 257:
        return ["random", "edges", "full", "equal", "scale30"]
    extra = {1024: ["equal"], 1280: ["full"], 1281: ["full", "scale30"], 2048: ["scale30"], 4096: ["full"]}
    return ["random", "edges"] + extra.get(S, [])


def inputs(name, kw, S, kind, seed=7):
    B = batch_for(S)
    y = labels(B, S, kind, seed)
    scale = 30.0 if kind == "scale30" else 1.0
    if name == "ordinal":
        n = int(kw["n"])
        z = torch.randn(B, S, n, generator=torch.Generator().manual_seed(seed + 2)) * (2.0 if scale == 1.0 else scale)
        return torch.sigmoid(z), y, {}
    yp = tie_free_scores(B, S, seed + 3, scale)
    extra = {}
    if name == "bce":
        yp = torch.sigmoid(yp)
        y = torch.where(y == PAD, y, (y > 0).float())
    elif name == "listMLE":
        from oracle.losses_ref import listMLE_realised_order
        perm = torch.randperm(S, generator=torch.Generator().manual_seed(seed + 4))
        extra = {"perm": perm, "order": listMLE_realised_order(y, perm)}
    return yp, y, extra


# ------------------------------------------------------------------------------------------------ a. the oracle
@pytest.mark.parametrize("case", LOSS_CASES, ids=_id)
def test_against_fp64_oracle_at_every_slate_length(case):
    name, kw = case
    problems, worst = [], [0.0]
    for S in SLATE_LENGTHS:
        for kind in kinds_for(S):
            yp, y, extra = inputs(name, kw, S, kind)
            if name in TIE_FREE:
                assert all(torch.unique(yp[b]).numel() == S for b in range(yp.shape[0]))
            args = dict(kw, **extra)
            val, grad, p = run_kernel(name, args, yp, y)
            problems += [f"S={S} {kind}: {m}" for m in p]
            saturated = name in ("bce", "ordinal") and kind == "scale30"
            if saturated:
                assert ((yp == 0) | (yp == 1)).any()
                ref, gref = saturated_bce_reference(name, kw, yp, y)
            else:
                ref, gref = reference(name, args, yp, y)
            problems += compare(f"S={S} {kind}", val, grad, ref, gref, y, GREL, worst)
    print(f"{_id(case)}: worst gradient error / largest entry {worst[0]:.3g}")
    assert not problems, "\n".join(problems)


def neural_inputs(S, kind, seed=7):
    """Slates for neuralNDCG.  The oracle materialises [B,n,n] per Sinkhorn iteration under autograd: B * n^2 stays
    near 2^18, and slates of 1024 items or more keep at most 600 valid items (a fully valid 4096-item slate needs a
    136 MB workspace per slate and minutes per call)."""
    B = 8 if S <= 128 else max(1, min(8, 2 ** 18 // (min(S, 600) ** 2)))
    y = labels(B, S, kind, seed)
    if S >= 1024:
        y[:, 600:] = PAD
    return tie_free_scores(B, S, seed + 3, 30.0 if kind == "scale30" else 1.0), y


def neural_kinds(S):
    return ["random", "edges", "full", "scale30"] if S <= 257 else ["random", "edges"]


def trimmed(yp, y):
    """The columns up to the last real item of any slate: the oracle on them equals the oracle on the whole slate
    (test_neural_oracle_ignores_trailing_padding)."""
    real = (y != PAD).any(dim=0).nonzero()
    w = int(real.max()) + 1 if real.numel() else 1
    return yp[:, :w], y[:, :w]


def test_neural_oracle_ignores_trailing_padding():
    """What lets the long neuralNDCG cases compare on the trimmed prefix: appending padded items changes neither the
    fp64 oracle's loss nor its gradient on the real items."""
    y = labels(4, 40, "random", 3)
    y[:, 30:] = PAD
    yp = tie_free_scores(4, 40, 5)
    for name, kw in NEURAL_CASES:
        kw = dict(kw, tol=0.0)
        a, ga = reference(name, kw, yp, y)
        b, gb = reference(name, kw, yp[:, :30], y[:, :30])
        assert a == pytest.approx(b, rel=1e-12, abs=1e-15), (name, kw)
        assert np.abs(ga[:, :30] - gb).max() <= 1e-12 * np.abs(gb).max(), (name, kw)
        assert (ga[:, 30:] == 0).all()


@pytest.mark.parametrize("case", NEURAL_CASES, ids=_id)
def test_neural_ndcg_against_fp64_oracle(case):
    """tol = 0 on both sides: both run exactly max_iter Sinkhorn iterations (the early exit is tested per slate by the
    kernel and over the batch by the reference).  S <= 128 runs the register kernel, 129 to ~140 the generic kernel in
    shared memory, longer slates the workspace; max_iter = 200 forces the generic kernel at S <= 128."""
    name, kw = case
    problems, worst = [], [0.0]
    runs = [(S, kind, 50) for S in SLATE_LENGTHS for kind in neural_kinds(S)] + [(S, "random", 200) for S in (33, 128)]
    for S, kind, iters in runs:
        yp, y = neural_inputs(S, kind)
        args = dict(kw, tol=0.0, max_iter=iters)
        val, grad, p = run_kernel(name, args, yp, y)
        problems += [f"S={S} {kind} max_iter={iters}: {m}" for m in p]
        ty, tyy = trimmed(yp, y)
        ref, gt = reference(name, args, ty, tyy)
        gref = np.zeros(grad.shape)
        gref[:, :gt.shape[1]] = gt
        problems += compare(f"S={S} {kind} max_iter={iters}", val, grad, ref, gref, y, GREL_NEURAL, worst)
    print(f"{_id(case)}: worst gradient error / largest entry {worst[0]:.3g}")
    assert not problems, "\n".join(problems)


def test_neural_ndcg_refuses_slates_beyond_4096():
    """Its per-item arrays fill the 220 KB of shared memory at exactly 4096 items: 4097 is refused, not launched."""
    from allrank_b200 import _lib
    from allrank_b200.metrics import discount_table
    S = 4097
    yp, y = torch.randn(1, S, device="cuda"), torch.ones(1, S, device="cuda")
    loss, scratch = torch.zeros((), device="cuda"), torch.zeros(2, device="cuda")
    lib, P = _lib.lib(), _lib.ptr
    before = _lib.launch_count()
    rc = lib.arb_neural_ndcg(P(yp), P(y), 1, S, P(discount_table(S, yp.device)), PAD, 1.0, 1, 0, 50, 0.0, P(loss),
                             None, P(scratch), None, 0, _lib.stream_ptr(yp.device))
    assert rc != 0 and "too long" in lib.arb_last_error().decode()
    assert _lib.launch_count() == before


# ------------------------------------------------------------------------------------------------ b. bit equality
BIT_EQUAL_CASES = ([("approxNDCGLoss", {"alpha": 1.0}), ("approxNDCGLoss", {"alpha": 5.0})]
                   + [("lambdaLoss", kw) for kw in LAMBDA_CASES]
                   + [(n, {}) for n in RANKNET] + [("ordinal", {"n": 4})]
                   + [(n, dict(kw, tol=0.0)) for n, kw in NEURAL_CASES])


@pytest.mark.parametrize("case", BIT_EQUAL_CASES, ids=_id)
def test_padding_to_longer_slates_keeps_the_bits(case):
    """130 valid items padded to 136, 240, 1024 and 4096: padded items add exact zeros in the same per-thread order,
    so the per-slate loss and the gradient of every item are the same bits.  neuralNDCG runs its generic kernel at
    all four: shared memory at 136; at 240 the host chose the workspace but the slate still fits in shared memory;
    the workspace at 1024 and 4096."""
    name, kw = case
    n, B = 130, 4
    y0 = labels(B, n, "full", 31)
    yp0 = tie_free_scores(B, n, 32)
    if name == "ordinal":
        yp0 = torch.sigmoid(2.0 * torch.randn(B, n, 4, generator=torch.Generator().manual_seed(33)))
    first = None
    for S in (136, 240, 1024, 4096):
        y = torch.cat([y0, torch.full((B, S - n), PAD)], dim=1)
        tail_shape = (B, S - n) + tuple(yp0.shape[2:])
        yp = torch.cat([yp0, torch.rand(tail_shape, generator=torch.Generator().manual_seed(S))], dim=1)
        val, grad, per = launch(name, kw, yp, y)
        assert (grad[:, n:] == 0).all(), S
        got = (val, per, grad[:, :n])
        if first is None:
            first = got
            continue
        assert same_bits(got[0], first[0]), (S, got[0], first[0])
        assert same_bits(got[1], first[1]), (S, got[1], first[1])
        assert same_bits(got[2], first[2]), (S, np.abs(got[2] - first[2]).max())


# ------------------------------------------------------------------------------------------------ c. 4096 items
@pytest.mark.parametrize("case", LOSS_CASES + NEURAL_CASES, ids=_id)
def test_every_loss_runs_at_4096(case):
    name, kw = case
    S, B = 4096, 2
    y = labels(B, S, "full", 41)
    if name.startswith("neuralNDCG"):
        y[:, 600:] = PAD
    yp = tie_free_scores(B, S, 42)
    extra = {}
    if name == "ordinal":
        yp = torch.sigmoid(torch.randn(B, S, 4, generator=torch.Generator().manual_seed(43)))
    elif name == "bce":
        yp = torch.sigmoid(yp)
        y = (y > 0).float()
    elif name == "listMLE":
        from oracle.losses_ref import listMLE_realised_order
        perm = torch.randperm(S, generator=torch.Generator().manual_seed(44))
        extra = {"perm": perm, "order": listMLE_realised_order(y, perm)}
    val, grad, _ = launch(name, dict(kw, **extra), yp, y)
    assert math.isfinite(val) and np.isfinite(grad).all(), (val, np.isnan(grad).sum())


@pytest.mark.parametrize("loss_name,activation", [("bce", "Sigmoid"), ("binary_listNet", None)])
def test_training_step_at_2048_with_pointwise_losses(loss_name, activation):
    """A scorer that trains at 2048 items trains with the losses of the pointwise family too."""
    from allrank_b200 import losses
    from allrank_b200.model import make_model
    from allrank_b200.optim import FlatAdam
    from allrank_b200.synth import make_slates
    S, B = 2048, 2
    x, y, _ = make_slates(B, S, n_features=136, seed=23, mean_len=0.6 * S, std_len=0.3 * S)
    x, y = x.cuda(), y.cuda()
    if loss_name == "bce":
        y = torch.where(y == PAD, y, (y > 0).float())
    torch.manual_seed(29)
    model = make_model(fc_model={"sizes": [64], "input_norm": False, "activation": None, "dropout": 0.0},
                       transformer={"N": 1, "d_ff": 128, "h": 4, "positional_encoding": None, "dropout": 0.1},
                       post_model={"d_output": 1, "output_activation": activation}, n_features=136).cuda().train()
    opt = FlatAdam(model, lr=1e-3)
    before = torch.cat([q.detach().flatten() for q in model.parameters()])
    loss = getattr(losses, loss_name)(model(x, y == PAD, None), y)
    opt.zero_grad()
    loss.backward()
    assert torch.isfinite(loss) and torch.isfinite(model.flat_gradients).all()
    assert model.flat_gradients.abs().sum() > 0
    opt.step()
    after = torch.cat([q.detach().flatten() for q in model.parameters()])
    assert torch.isfinite(after).all() and not torch.equal(before, after)
