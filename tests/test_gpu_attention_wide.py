"""The fused attention kernels at head widths 36 ... 96 (csrc/attention_long.cu at DK = 64 and 96: attn_long_fwd_kernel,
attn_long_dkdv_kernel, attn_long_dq_kernel, with attn_delta_kernel's path for widths that are not a power of two)
against the fp64 reference of tests/test_gpu_attention_kernels.py (same per-element bounds, TAU, NaN-prefilled outputs,
every case run twice for identical bits), against attn_fwd_kernel bit for bit at width 64, and through the scorer at
the shapes of the shipped configurations (local_config 64, ordinal 72, neuralNDCG-paper 96) against the unfused path
and the TF32 emulation."""
import ctypes

import pytest
import torch

from tests.test_gpu_attention_kernels import (  # noqa: F401  (lib: the module's fixture)
    TAU, bwd_case, bits, check, check_backward, check_forward, colsum_and_bound, fwd_case, lib, make_dctx,
    make_inputs, reference, reference_bwd, run_bwd, run_fwd, same_bits)

pytestmark = pytest.mark.gpu


def wide_extents(S):
    """Extents on both sides of 16-row strips, 64-row streamed blocks, 128-row tiles and the short kernels' 256 rows."""
    cand = {1, 15, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257, 383, 640, 1025, S - 1, S}
    if S >= 2048:                     # the fp64 reference holds B * h * S^2 doubles per tensor
        cand = {63, 129, 1025, S - 1, S}
    return sorted(e for e in cand if 1 <= e <= S)


CASES = [(w, S, p) for w in (64, 72, 96) for S in (37, 129, 240, 256, 257, 1024, 4096) for p in (0.0, 0.1, 0.3)]
CASES += [(36, 240, 0.1), (36, 1024, 0.0), (84, 240, 0.3), (84, 1024, 0.1)]


@pytest.mark.parametrize("w,S,p", CASES, ids=[f"w{w}-S{S}-p{p}" for w, S, p in CASES])
def test_forward_and_backward_match_fp64_reference(lib, w, S, p):
    ex = wide_extents(S)
    B, h = len(ex), (1 if S >= 2048 else 2)
    seed = w * 10000 + S + int(p * 10)
    qkv, mask, ext, R = fwd_case(lib, ex, S, h, w, p, seed=seed)
    out = run_fwd(lib, qkv, mask, ext, B, S, h, w, p)
    again = run_fwd(lib, qkv, mask, ext, B, S, h, w, p)
    assert all(same_bits(a, b) for a, b in zip(out, again)), "two forward runs differ"
    check_forward(f"wide fwd w{w} S{S} p{p}", R, *out, B, S, h, w)
    del R
    torch.cuda.empty_cache()
    args, Rb, gext = bwd_case(lib, ex, S, h, w, p, seed=seed + 7)
    d_qkv, dbias = run_bwd(lib, *args)
    d2, b2 = run_bwd(lib, *args)
    assert same_bits(d_qkv, d2) and same_bits(dbias, b2), "two backward runs differ"
    assert any(g > e for g, e in zip(gext, ex)), "no backward extent past the key extent"
    check_backward(f"wide bwd w{w} S{S} p{p}", Rb, d_qkv, dbias, args[-1], gext, B, S, h, w)


def _embed(t, B, S0, S, fill):
    """[B*S0, c] rows -> [B*S, c] with rows S0 ... S-1 of every slate set to `fill`."""
    c = t.shape[-1]
    out = torch.full((B, S, c), fill, dtype=t.dtype, device=t.device)
    out[:, :S0] = t.view(B, S0, c)
    return out.reshape(B * S, c)


def test_long_forward_gives_the_short_forward_bits_at_width_64(lib):
    """Slates of at most 256 items in an S = 256 batch (attn_fwd_kernel) and in S = 300 / 1024 batches (the long
    forward): row statistics of rows 0 ... 255 are the same bits, and so is the context without dropout (the dropout
    counter is indexed by S, so other S draw other masks)."""
    S0, h, w = 256, 2, 64
    ex = [1, 16, 17, 63, 64, 65, 100, 128, 129, 200, 255, 256]
    B, d = len(ex), h * w
    qkv0, mask0, ext = make_inputs(ex, S0, h, w, seed=140)
    res = {}
    for p in (0.0, 0.1):
        for S in (S0, 300, 1024):
            qkv = _embed(qkv0, B, S0, S, 7.0)          # garbage in the rows past 256: masked, beyond every extent
            mask = torch.ones(B, S, dtype=torch.uint8, device="cuda")
            mask[:, :S0] = mask0
            ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, w, p)
            res[S] = (ctx.view(B, S, d)[:, :S0], smax[..., :S0], ssum[..., :S0])
        for S in (300, 1024):
            for i, name in enumerate(("ctx", "stat_max", "stat_sum")):
                if p > 0 and name == "ctx":
                    continue
                assert same_bits(res[S][i], res[S0][i]), f"p={p} S={S}: {name} differs from attn_fwd_kernel"


@pytest.mark.parametrize("w,S", [(72, 129), (96, 300)])
def test_all_padded_slate(lib, w, S):
    """A slate without real items: NaN context rows, row max -inf, row sum 0, exactly zero gradients."""
    h = 2
    ex = [S, 1, 100]
    B = len(ex)
    qkv, mask, _, _ = fwd_case(lib, ex, S, h, w, 0.0, seed=5)
    mask[1] = 1
    R = reference(qkv, mask, B, S, h, w, None)
    ext = torch.tensor([S, 0, 100], dtype=torch.int32, device="cuda")
    ctx, smax, ssum = run_fwd(lib, qkv, mask, ext, B, S, h, w, 0.0)
    assert torch.isnan(ctx.view(B, S, -1)[1]).all()
    assert (smax[1] == float("-inf")).all() and (ssum[1] == 0).all()
    check_forward("wide all-padded fwd", R, ctx, smax, ssum, B, S, h, w)
    gext = [S, 0, 100]
    d_ctx = make_dctx(gext, S, h * w, 6)
    Rb = reference_bwd(R, d_ctx, ctx, B, S, h, w)
    d_qkv, _ = run_bwd(lib, qkv, ctx, d_ctx, mask, ext, smax, ssum, B, S, h, w, 0.0, None)
    g = d_qkv.view(B, S, 3 * h * w)
    assert torch.equal(bits(g[1]), torch.zeros_like(bits(g[1]))), "gradients of the all-padded slate are not +0"
    keep = torch.tensor([0, 2], device="cuda")
    sub = {k: v[keep] for k, v in Rb.items()}
    check_backward("wide all-padded bwd", sub, d_qkv.view(B, S, -1)[keep].reshape(2 * S, -1), None, None, [S, 100],
                   2, S, h, w)


@pytest.mark.parametrize("w", [72, 96])
def test_truncating_tf32_operands(lib, w):
    """arb_set_tf32_round_on_load(0): the tensor core truncates; within the bounds of the truncation emulation."""
    S, h, p = 257, 2, 0.1
    ex = wide_extents(S)
    B = len(ex)
    try:
        lib.lib().arb_set_tf32_round_on_load(0)
        qkv, mask, ext, R = fwd_case(lib, ex, S, h, w, p, seed=78, mode="trunc")
        check_forward("wide trunc fwd", R, *run_fwd(lib, qkv, mask, ext, B, S, h, w, p), B, S, h, w)
        args, Rb, gext = bwd_case(lib, ex, S, h, w, p, seed=79, mode="trunc")
        d_qkv, dbias = run_bwd(lib, *args)
        check_backward("wide trunc bwd", Rb, d_qkv, dbias, args[-1], gext, B, S, h, w)
    finally:
        lib.lib().arb_set_tf32_round_on_load(1)


@pytest.mark.parametrize("w,S", [(64, 240), (72, 240), (96, 1024)])
def test_null_extent_gives_the_same_bits(lib, w, S):
    """Without extents the kernels run every key and query; the work the extents skip adds exact zeros, so context,
    statistics, gradients and the bias gradient are bit-identical."""
    ex = wide_extents(S)
    B, h = len(ex), 2
    qkv, mask, ext, _ = fwd_case(lib, ex, S, h, w, 0.1, seed=w + S)
    a = run_fwd(lib, qkv, mask, ext, B, S, h, w, 0.1)
    b = run_fwd(lib, qkv, mask, None, B, S, h, w, 0.1)
    assert all(same_bits(x, y) for x, y in zip(a, b))
    args, _, _ = bwd_case(lib, ex, S, h, w, 0.1, seed=w + S)
    ga, ba = run_bwd(lib, *args)
    args = args[:4] + (None,) + args[5:]
    gb, bb = run_bwd(lib, *args)
    assert same_bits(ga, gb) and same_bits(ba, bb)


def test_bf16_context_at_width_64_is_refused(lib):
    S, h, w = 240, 1, 64
    qkv, mask, ext = make_inputs([240], S, h, w, seed=3)
    ctx = torch.zeros(S, h * w, device="cuda", dtype=torch.bfloat16)
    smax = torch.zeros(1, h, S, device="cuda")
    rc = lib.lib().arb_attention_forward(lib.ptr(qkv), lib.ptr(mask), lib.ptr(ext), 1, S, h, w, 0.0, 1, 0, 1,
                                         lib.ptr(ctx), lib.ptr(smax), lib.ptr(smax.clone()), lib.stream_ptr())
    assert rc != 0
    from allrank_b200.model import make_model
    with pytest.raises(NotImplementedError):
        make_model(**SHIPPED["local_config"], n_features=136, compute_dtype="bf16")


# ------------------------------------------------------------------------------------------------ scorer
# the `model` sections of scripts/local_config.json, contextaware_web30k/ordinal.json and neuralndcg_web30k/approxndcg.json
SHIPPED = {
    "local_config": dict(fc_model={"sizes": [64], "input_norm": False, "activation": None, "dropout": 0.0},
                         transformer={"N": 1, "d_ff": 64, "h": 1, "positional_encoding": None, "dropout": 0.0},
                         post_model={"output_activation": "Sigmoid", "d_output": 4}),
    "ordinal": dict(fc_model={"sizes": [144], "input_norm": False, "activation": None, "dropout": 0.0},
                    transformer={"N": 4, "d_ff": 512, "h": 2, "positional_encoding": None, "dropout": 0.4},
                    post_model={"output_activation": "Sigmoid", "d_output": 4}),
    "approxndcg": dict(fc_model={"sizes": [96], "input_norm": False, "activation": None, "dropout": 0.0},
                       transformer={"N": 2, "d_ff": 384, "h": 1, "positional_encoding": None, "dropout": 0.1},
                       post_model={"output_activation": None, "d_output": 1}),
}


def _set_attention_mode(mode):
    from allrank_b200 import _lib
    L = _lib.lib()
    L.arb_set_attention_mode.argtypes = [ctypes.c_int32]
    L.arb_set_attention_mode(mode)


def _shipped(name, seed=29, dropout=None):
    from allrank_b200.model import make_model
    cfg = {k: dict(v) for k, v in SHIPPED[name].items()}
    if dropout is not None:
        cfg["transformer"]["dropout"] = dropout
    torch.manual_seed(seed)
    return make_model(**cfg, n_features=136).cuda().train()


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


SCORER = [("local_config", 240, None), ("local_config", 240, 0.1), ("ordinal", 240, None), ("approxndcg", 240, None),
          ("approxndcg", 1024, None)]


@pytest.mark.parametrize("name,S,p", SCORER, ids=[f"{n}-S{S}-p{p}" for n, S, p in SCORER])
def test_scorer_matches_the_unfused_path(name, S, p, monkeypatch):
    """Modes 2 (fused forward and backward) and 1 (fused forward, unfused backward) against mode 0 (materialised
    S x S), train mode with the configuration's dropout (p: another rate), the same dropout masks: scores, flat
    gradients, x.grad and prepare_for_output with the tolerances of test_gpu_attention_long's scorer test.  With
    attention dropout the flat gradients of modes 1 and 2 both lie up to ~2.2 % from mode 0's (H100: local_config at
    p = 0.1 1.77 % for both, ordinal 2.14 % for both; mode 1 at local_config runs only kernels older than the wide
    ones): the forward's TF32 differences, amplified by the dropout scale.  So mode 2's flat gradient is held to
    1.5e-2 against mode 1's -- the same forward, the unfused backward -- and to mode 1's own distance from mode 0."""
    B = 4
    model = _shipped(name, dropout=p)
    monkeypatch.setattr(model, "_draw_seed", lambda: 0x5DEECE66D)
    x0, y = _slates(B, S, 136, seed=13)
    mask = y == -1
    d = SHIPPED[name]["fc_model"]["sizes"][0]
    g = torch.Generator(device="cuda").manual_seed(3)
    w = torch.randn(*model(x0, mask, None).shape, device="cuda", generator=g)
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
        print(name, S, p, "mode", mode, "score diff", (s0 - s1).abs().max().item(), "grad", _rel(g1, g0), "x.grad",
              _rel(xs1, xs0), "hidden", (h0 - h1).abs().max().item(), "x.grad (hidden)", _rel(xh1, xh0))
    for mode in (1, 2):
        s0, g0, xs0, h0, xh0 = out[0]
        s1, g1, xs1, h1, xh1 = out[mode]
        ds = (s0 - s1).abs().max().item()
        dh = (h0 - h1).abs().max().item()
        assert ds <= 2e-3 * max(1.0, s0.abs().max().item())
        assert dh <= 2e-3 * max(1.0, h0.abs().max().item())
        assert _rel(xs1, xs0) <= 5e-2 and _rel(xh1, xh0) <= 5e-2
    g0, g1, g2 = out[0][1], out[1][1], out[2][1]
    assert _rel(g2, g1) <= 1.5e-2, "the fused backward's flat gradient against the unfused backward's"
    assert _rel(g2, g0) <= max(1.5e-2, 1.1 * _rel(g1, g0))


def test_width_96_at_2048_against_the_tf32_emulation():
    """S = 2048 (beyond the unfused softmax): scores, x.grad and the parameter gradients against the TF32 emulation on
    the host."""
    from oracle.tf32_emulation import scorer_forward
    F, d, h, B, S = 136, 96, 1, 2, 2048
    model = _model(F, d, 1, h, 384, 0.0).eval()
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
    print(S, "scores rel err", es, "x.grad rel err", ex)
    assert es <= 1e-3 and ex <= 1e-2, (es, ex)
    for k, q in model.named_parameters():
        r = sd[k].grad
        if r is None or ".self_attn.linears.1.bias" in k:   # the key bias gradient is analytically zero: rounding only
            continue
        e = _rel(q.grad.cpu(), r)
        assert e <= (1e-1 if ".feed_forward.w_1." in k else 5e-2), (k, e)


def test_workspace_drops_the_probability_buffers_at_width_72():
    from allrank_b200 import _lib
    model = _shipped("ordinal")
    N, h, B, S = 4, 2, 8, 240
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


def test_graphed_dropout_training_at_width_72(monkeypatch):
    """GraphedTrainStep(dropout_seed=s) of the ordinal configuration: replay k equals an eager step seeded s + k."""
    from allrank_b200 import losses
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.optim import FlatAdam
    batches = [_slates(8, 240, 136, seed=20 + k) for k in range(2)] * 2

    def loss_fn(s, y):
        return losses.ordinal(s, y, n=4)
    s = 977

    eager = _shipped("ordinal")
    opt = FlatAdam(eager, lr=1e-3, capturable=True)
    eager_losses = []
    for k, (x, y) in enumerate(batches, start=1):
        monkeypatch.setattr(eager, "_draw_seed", lambda k=k: s + k)
        loss = loss_fn(eager(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        eager_losses.append(loss.item())

    graphed = _shipped("ordinal")
    gopt = FlatAdam(graphed, lr=1e-3, capturable=True)
    init = {k: v.clone() for k, v in graphed.state_dict().items()}
    monkeypatch.setattr(graphed, "_draw_seed", lambda: pytest.fail("the graphed step drew a host seed"))
    step = GraphedTrainStep(graphed, loss_fn, gopt, *batches[0], warmup=2, dropout_seed=s)
    graphed.load_state_dict(init)
    gopt.exp_avg.zero_(); gopt.exp_avg_sq.zero_(); gopt._dev_state.zero_()
    graph_losses = [step(x, y).item() for x, y in batches]
    assert graph_losses == eager_losses
    assert torch.equal(graphed.flat_parameters, eager.flat_parameters)


def test_padded_items_keep_their_scores_with_packed_rows_on():
    """Packed rows (the default) serve head widths 16 and 32 only: a width-96 model still scores its padded items as
    the unfused path does, not 0."""
    from allrank_b200 import _lib
    L = _lib.lib()
    L.arb_get_pack_rows.restype = ctypes.c_int32
    L.arb_set_pack_rows.argtypes = [ctypes.c_int32]
    B, S = 6, 240
    model = _model(136, 96, 2, 1, 384, 0.0).eval()
    x, y = _slates(B, S, 136, seed=31)
    mask = y == -1
    assert mask.any()
    old = L.arb_get_pack_rows()
    out = {}
    try:
        L.arb_set_pack_rows(1)
        with torch.no_grad():
            for mode in (0, 2):
                _set_attention_mode(mode)
                out[mode] = model(x, mask, None).clone()
    finally:
        _set_attention_mode(2)
        L.arb_set_pack_rows(old)
    pad0, pad2 = out[0][mask], out[2][mask]
    assert (pad2 != 0).any(), "padded items scored 0"
    assert (out[2] - out[0]).abs().max().item() <= 2e-3 * max(1.0, out[0].abs().max().item())
    assert (pad2 - pad0).abs().max().item() <= 2e-3 * max(1.0, pad0.abs().max().item())
