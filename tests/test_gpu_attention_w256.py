"""The fused attention kernels at head widths 132 ... 256 (csrc/attention_long.cu at DK = 192 and 256: 64-row tiles, each
16-row strip shared by two warps with half the output columns each, 32- / 16-row streamed blocks, with
attn_delta_wide_kernel) against the fp64 reference of tests/test_gpu_attention_kernels.py (same per-element bounds, TAU,
NaN-prefilled outputs, every case run twice for identical bits), for bit-identical results when the same slates sit in
batches of other S, and through the scorer against the unfused path and the TF32 emulation, with the workspace, graph
replay and a few training steps."""
import ctypes

import pytest
import torch

from tests.test_gpu_attention_kernels import (  # noqa: F401  (lib: the module's fixture)
    TAU, bits, bwd_case, check, check_backward, check_forward, colsum_and_bound, fwd_case, lib, make_dctx, make_inputs,
    reference, reference_bwd, run_bwd, run_fwd, same_bits)
from tests.test_gpu_attention_wide import _embed, _model, _rel, _set_attention_mode, _slates

pytestmark = pytest.mark.gpu


def w256_extents(S):
    """Extents on both sides of 16-row strips, 16- and 32-row streamed blocks, 64-row tiles and the short kernels' 256
    rows."""
    cand = {1, 15, 16, 17, 31, 32, 33, 47, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 640, 1025, S - 1, S}
    if S >= 2048:                     # the fp64 reference holds B * h * S^2 doubles per tensor
        cand = {33, 65, 129, 1025, S - 1, S}
    return sorted(e for e in cand if 1 <= e <= S)


CASES = [(w, S, p) for w in (192, 256) for S in (1, 37, 129, 240, 256, 257, 1024, 4096) for p in (0.0, 0.1, 0.3)]
CASES += [(w, S, p) for w, p in ((132, 0.1), (136, 0.0), (160, 0.3), (196, 0.1), (200, 0.3)) for S in (240, 1024)]


@pytest.mark.parametrize("w,S,p", CASES, ids=[f"w{w}-S{S}-p{p}" for w, S, p in CASES])
def test_forward_and_backward_match_fp64_reference(lib, w, S, p):
    ex = w256_extents(S)
    B, h = len(ex), (1 if S >= 1024 else 2)
    seed = w * 10000 + S + int(p * 10)
    qkv, mask, ext, R = fwd_case(lib, ex, S, h, w, p, seed=seed)
    out = run_fwd(lib, qkv, mask, ext, B, S, h, w, p)
    again = run_fwd(lib, qkv, mask, ext, B, S, h, w, p)
    assert all(same_bits(a, b) for a, b in zip(out, again)), "two forward runs differ"
    check_forward(f"w256 fwd w{w} S{S} p{p}", R, *out, B, S, h, w)
    del R
    torch.cuda.empty_cache()
    args, Rb, gext = bwd_case(lib, ex, S, h, w, p, seed=seed + 7)
    d_qkv, dbias = run_bwd(lib, *args)
    d2, b2 = run_bwd(lib, *args)
    assert same_bits(d_qkv, d2) and same_bits(dbias, b2), "two backward runs differ"
    if S > 1:
        assert any(g > e for g, e in zip(gext, ex)), "no backward extent past the key extent"
    check_backward(f"w256 bwd w{w} S{S} p{p}", Rb, d_qkv, dbias, args[-1], gext, B, S, h, w)


@pytest.mark.parametrize("w,S", [(256, 65), (256, 300), (192, 129), (136, 300)])
def test_all_padded_slate(lib, w, S):
    """A slate without real items beside one of extent 1: NaN context rows, row max -inf, row sum 0, exactly zero
    gradients."""
    h = 2
    ex = [S, 1, 50]
    B = len(ex)
    qkv, mask, _, _ = fwd_case(lib, ex, S, h, w, 0.0, seed=5)
    mask[1] = 1
    R = reference(qkv, mask, B, S, h, w, None)
    ext = torch.tensor([S, 0, 50], dtype=torch.int32, device="cuda")
    ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, w, 0.0)
    assert torch.isnan(ctx.view(B, S, -1)[1]).all()
    assert (smax[1] == float("-inf")).all() and (ssum[1] == 0).all()
    check_forward("w256 all-padded fwd", R, ctx, smax, ssum, B, S, h, w)
    gext = [S, 0, 50]
    d_ctx = make_dctx(gext, S, h * w, 6)
    Rb = reference_bwd(R, d_ctx, ctx, B, S, h, w)
    d_qkv, _ = run_bwd(lib, qkv, ctx, d_ctx, mask, ext, smax, ssum, B, S, h, w, 0.0, None)
    g = d_qkv.view(B, S, 3 * h * w)
    assert torch.equal(bits(g[1]), torch.zeros_like(bits(g[1]))), "gradients of the all-padded slate are not +0"
    keep = torch.tensor([0, 2], device="cuda")
    sub = {k: v[keep] for k, v in Rb.items()}
    check_backward("w256 all-padded bwd", sub, d_qkv.view(B, S, -1)[keep].reshape(2 * S, -1), None, None, [S, 50],
                   2, S, h, w)


@pytest.mark.parametrize("w,S", [(256, 240), (192, 1024), (132, 257)])
def test_null_extent_gives_the_same_bits(lib, w, S):
    """Without extents the kernels run every key and query; the work the extents skip adds exact zeros, so context,
    statistics, gradients and the bias gradient are bit-identical."""
    ex = w256_extents(S)
    B, h = len(ex), 1
    qkv, mask, ext, _ = fwd_case(lib, ex, S, h, w, 0.1, seed=w + S)
    a = run_fwd(lib, qkv, mask, ext, B, S, h, w, 0.1)
    b = run_fwd(lib, qkv, mask, None, B, S, h, w, 0.1)
    assert all(same_bits(x, y) for x, y in zip(a, b))
    args, _, _ = bwd_case(lib, ex, S, h, w, 0.1, seed=w + S)
    ga, ba = run_bwd(lib, *args)
    args = args[:4] + (None,) + args[5:]
    gb, bb = run_bwd(lib, *args)
    assert same_bits(ga, gb) and same_bits(ba, bb)


@pytest.mark.parametrize("w,h", [(256, 1), (136, 2)])
def test_padding_gives_the_same_bits(lib, w, h):
    """The same slates of at most 256 items in batches with S = 256, 300 and 1024, without dropout (its counter is
    indexed by S): keys beyond a slate's extent are never streamed, so the context, row statistics and dQ / dK / dV of
    the real rows are the same bits.  The QKV bias gradient may be summed in another association: it is held to the
    bound of adding the stored rows in any order."""
    S0 = 256
    ex = [1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 191, 193, 200, 255, 256]
    B, d = len(ex), h * w
    qkv0, mask0, ext = make_inputs(ex, S0, h, w, seed=143)
    gext = [min(S0, e + 3) if b % 3 == 1 else e for b, e in enumerate(ex)]
    dctx0 = make_dctx(gext, S0, d, 144)
    gx = torch.tensor(gext, dtype=torch.int32, device="cuda")
    db0 = torch.randn(3 * d, generator=torch.Generator().manual_seed(145)).cuda()
    res = {}
    for S in (S0, 300, 1024):
        qkv = _embed(qkv0, B, S0, S, 7.0)          # garbage in the rows past 256: masked, beyond every extent
        mask = torch.ones(B, S, dtype=torch.uint8, device="cuda")
        mask[:, :S0] = mask0
        ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, w, 0.0)
        d_ctx = _embed(dctx0, B, S0, S, 0.0)
        d_qkv, dbias = run_bwd(lib, qkv, ctx, d_ctx, mask, gx, smax, ssum, B, S, h, w, 0.0, db0)
        want, acc_b = colsum_and_bound(d_qkv, db0)
        check(f"w256 padding w{w} S{S} dbias", dbias, want, acc_b / TAU)
        res[S] = (ctx.view(B, S, d)[:, :S0], smax[..., :S0], ssum[..., :S0], d_qkv.view(B, S, 3 * d)[:, :S0])
    for S in (300, 1024):
        for i, name in enumerate(("ctx", "stat_max", "stat_sum", "d_qkv")):
            assert same_bits(res[S][i], res[S0][i]), f"S={S}: {name} differs from S={S0}"


# ------------------------------------------------------------------------------------------------ scorer
# (d_model, n_heads, N, d_ff): head widths 136, 192, 256 (one head: the neuralNDCG-paper model widened) and 160, 256
MODELS = {"d136h1": (136, 1, 2, 384), "d192h1": (192, 1, 2, 384), "d256h1": (256, 1, 2, 512),
          "d320h2": (320, 2, 1, 640), "d512h2": (512, 2, 1, 1024)}


def _w256_model(name, p, seed=29):
    d, h, N, dff = MODELS[name]
    return _model(136, d, N, h, dff, p, seed=seed)


# d 512 has no unfused backward (its QKV bias column sum spans 3 d = 1536 > 1024 columns): the TF32 emulation checks it
SCORER = [(n, S, p) for n in MODELS if n != "d512h2" for S, p in ((240, 0.0), (240, 0.1), (1024, 0.1))]


@pytest.mark.parametrize("name,S,p", SCORER, ids=[f"{n}-S{S}-p{p}" for n, S, p in SCORER])
def test_scorer_matches_the_unfused_path(name, S, p, monkeypatch):
    """Modes 2 (fused forward and backward) and 1 (fused forward, unfused backward) against mode 0 (materialised
    S x S), train mode, the same dropout masks: scores, prepare_for_output, flat gradients and x.grad with the
    tolerances and reasoning of test_gpu_attention_wide's scorer test -- with attention dropout, mode 2's flat gradient
    is held to 1.5e-2 against mode 1's and to mode 1's own distance from mode 0."""
    B, F = 4, 136
    model = _w256_model(name, p)
    monkeypatch.setattr(model, "_draw_seed", lambda: 0x5DEECE66D)
    x0, y = _slates(B, S, F, seed=13)
    mask = y == -1
    g = torch.Generator(device="cuda").manual_seed(3)
    w = torch.randn(*model(x0, mask, None).shape, device="cuda", generator=g)
    out = {}
    try:
        for mode in (0, 1, 2):
            _set_attention_mode(mode)
            model.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(True)
            s = model(x, mask, None)
            (s * w).sum().backward()
            with torch.no_grad():
                pfo = model.prepare_for_output(x0, mask, None).clone()
            out[mode] = (s.detach().clone(), model.flat_gradients.clone(), x.grad.clone(), pfo)
    finally:
        _set_attention_mode(2)
    for mode in (1, 2):
        s0, g0, xs0, _ = out[0]
        s1, g1, xs1, _ = out[mode]
        print(name, S, p, "mode", mode, "score diff", (s0 - s1).abs().max().item(), "grad", _rel(g1, g0), "x.grad",
              _rel(xs1, xs0))
    for mode in (1, 2):
        s0, _, xs0, p0 = out[0]
        s1, _, xs1, p1 = out[mode]
        assert (s0 - s1).abs().max().item() <= 2e-3 * max(1.0, s0.abs().max().item())
        assert (p0 - p1).abs().max().item() <= 2e-3 * max(1.0, p0.abs().max().item())
        assert _rel(xs1, xs0) <= 5e-2
    g0, g1, g2 = out[0][1], out[1][1], out[2][1]
    assert _rel(g2, g1) <= 1.5e-2, "the fused backward's flat gradient against the unfused backward's"
    assert _rel(g2, g0) <= max(1.5e-2, 1.1 * _rel(g1, g0))


EMUL = [("d136h1", 2048), ("d256h1", 2048), ("d512h2", 240), ("d512h2", 1024), ("d512h2", 2048), ("d256h1", 4096)]


@pytest.mark.parametrize("name,S", EMUL, ids=[f"{n}-S{S}" for n, S in EMUL])
def test_scorer_matches_the_tf32_emulation(name, S):
    """S > 1536 (where the unfused softmax stops), and d 512 at every S (no unfused backward there): scores, x.grad and
    the parameter gradients against the TF32 emulation on the host."""
    from oracle.tf32_emulation import scorer_forward
    F, B = 136, 2
    _, h, N, _ = MODELS[name]
    model = _w256_model(name, 0.0).eval()
    x0, y = _slates(B, S, F, seed=17)
    mask = y == -1
    w = torch.randn(B, S, generator=torch.Generator().manual_seed(4)).cuda() * (~mask).float()
    x = x0.clone().requires_grad_(True)
    s = model(x, mask, None)
    (s * w).sum().backward()
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    xe = x0.cpu().clone().requires_grad_(True)
    ref = scorer_forward(sd, xe, mask.cpu(), N, h, None, "rna")
    (ref * w.cpu()).sum().backward()
    real = (~mask).cpu()
    es = _rel(s.detach().cpu()[real], ref.detach()[real])
    ex = _rel(x.grad.cpu(), xe.grad)
    print(name, S, "scores rel err", es, "x.grad rel err", ex)
    # at S = 240 x.grad has the unfused comparison's bound: on these two slates the width-128 model d 512, h 4 (kernels
    # older than widths above 128) already lies 1.0e-2 from the emulation
    assert es <= 1e-3 and ex <= (5e-2 if S <= 256 else 1e-2), (es, ex)
    for k, q in model.named_parameters():
        r = sd[k].grad
        if r is None or ".self_attn.linears.1.bias" in k:   # the key bias gradient is analytically zero: rounding only
            continue
        e = _rel(q.grad.cpu(), r)
        assert e <= (1e-1 if ".feed_forward.w_1." in k else 5e-2), (k, e)


@pytest.mark.parametrize("name", ["d256h1", "d512h2"])
def test_workspace_drops_the_probability_buffers(name):
    from allrank_b200 import _lib
    model = _w256_model(name, 0.1)
    _, h, N, _ = MODELS[name]
    B, S = 4, 1024
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


def test_two_training_steps_give_the_same_bits(monkeypatch):
    """The same step twice from the same state, with attention dropout: scores and flat gradients are the same bits
    (the QKV bias gradient goes through per-warp slots summed in order)."""
    from allrank_b200 import losses
    x, y = _slates(8, 1024, 136, seed=23)
    model = _w256_model("d512h2", 0.1)
    monkeypatch.setattr(model, "_draw_seed", lambda: 4242)
    out = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        s = model(x, y == -1, None)
        losses.approxNDCGLoss(s, y).backward()
        out.append((s.detach().clone(), model.flat_gradients.clone()))
    assert same_bits(out[0][0], out[1][0]) and same_bits(out[0][1], out[1][1])


def test_graphed_dropout_training_at_width_256(monkeypatch):
    """GraphedTrainStep(dropout_seed=s) at width 256, S = 1024: replay k equals an eager step seeded s + k."""
    from allrank_b200 import losses
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.optim import FlatAdam
    batches = [_slates(4, 1024, 136, seed=20 + k) for k in range(2)] * 2
    s = 977

    eager = _w256_model("d256h1", 0.3)
    opt = FlatAdam(eager, lr=1e-3, capturable=True)
    eager_losses = []
    for k, (x, y) in enumerate(batches, start=1):
        monkeypatch.setattr(eager, "_draw_seed", lambda k=k: s + k)
        loss = losses.approxNDCGLoss(eager(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        eager_losses.append(loss.item())

    graphed = _w256_model("d256h1", 0.3)
    gopt = FlatAdam(graphed, lr=1e-3, capturable=True)
    init = {k: v.clone() for k, v in graphed.state_dict().items()}
    monkeypatch.setattr(graphed, "_draw_seed", lambda: pytest.fail("the graphed step drew a host seed"))
    step = GraphedTrainStep(graphed, losses.approxNDCGLoss, gopt, *batches[0], warmup=2, dropout_seed=s)
    graphed.load_state_dict(init)
    gopt.exp_avg.zero_(); gopt.exp_avg_sq.zero_(); gopt._dev_state.zero_()
    graph_losses = [step(x, y).item() for x, y in batches]
    assert graph_losses == eager_losses
    assert torch.equal(graphed.flat_parameters, eager.flat_parameters)


def test_one_head_of_width_256_trains():
    """make_model(h=1, d_model=256) trains: a few Adam steps on one batch lower the loss."""
    from allrank_b200 import losses
    from allrank_b200.optim import FlatAdam
    model = _model(136, 256, 2, 1, 512, 0.1, seed=7)
    opt = FlatAdam(model, lr=1e-3)
    x, y = _slates(16, 240, 136, seed=41)
    hist = []
    for _ in range(8):
        loss = losses.approxNDCGLoss(model(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        hist.append(loss.item())
    assert all(v == v for v in hist), hist
    assert hist[-1] < hist[0], hist


def test_one_head_wider_than_256_is_refused():
    """h = 1, d_model = 260: a head of 260 columns raises NotImplementedError rather than fall back."""
    x, y = _slates(2, 16, 136, seed=3)
    with pytest.raises(NotImplementedError, match="256"):
        _model(136, 260, 1, 1, 520, 0.0)(x, y == -1, None)
