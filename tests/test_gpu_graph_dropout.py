"""Dropout seeds read from device memory (LTRModel.dropout_seed_from, the arb_scorer_*_dseed entry points) and CUDA-graph
training steps with dropout (GraphedTrainStep(dropout_seed=...)).

With the same seed value the device-seeded path must apply exactly the host-seeded masks: every comparison here is
bitwise."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(fc_sizes=(64,), fc_act=None, p_fc=0.0, N=2, h=2, dff=128, p=0.3, d_output=1, out_act=None,
           compute_dtype="tf32", F=136, seed=3):
    from allrank_b200.model import make_model
    torch.manual_seed(seed)
    tcfg = {"N": N, "d_ff": dff, "h": h, "positional_encoding": None, "dropout": p} if N > 0 else None
    return make_model(fc_model={"sizes": list(fc_sizes), "input_norm": False, "activation": fc_act, "dropout": p_fc},
                      transformer=tcfg, post_model={"d_output": d_output, "output_activation": out_act},
                      n_features=F, compute_dtype=compute_dtype).cuda().train()


def _batch(B, S, F=136, seed=5):
    from allrank_b200.synth import make_slates
    x, y, _ = make_slates(B, S, n_features=F, seed=seed, mean_len=0.7 * S, std_len=0.2 * S)
    return x.cuda(), y.cuda()


def _seed_tensor(s):
    return torch.tensor([s], dtype=torch.int64, device="cuda")


def _pass(model, x, mask, ws, wh):
    """scores, x.grad through the scores, prepare_for_output, x.grad through it, the flat gradient of both backwards."""
    for q in model.parameters():
        q.grad = None
    xs = x.clone().requires_grad_(True)
    scores = model(xs, mask, None)
    (scores * ws).sum().backward()
    xh = x.clone().requires_grad_(True)
    hidden = model.prepare_for_output(xh, mask, None)
    (hidden * wh).sum().backward()
    return [scores.detach().clone(), xs.grad.clone(), hidden.detach().clone(), xh.grad.clone(),
            model.flat_gradients.clone()]


SHAPES = {   # (model arguments, B, S): every dropout site and kernel path
    "relu_mlp_fc_dropout": (dict(fc_sizes=(64, 32), fc_act="ReLU", p_fc=0.3, N=0, d_output=4, out_act="Sigmoid"), 6, 40),
    "dk32_fused_fwd_bwd": (dict(fc_sizes=(128,), p_fc=0.1, N=2, h=4, dff=256, p=0.3), 5, 64),
    "dk64_fused_fwd_unfused_bwd": (dict(fc_sizes=(128,), N=1, h=2, dff=256, p=0.3), 5, 64),
    "dk96_h1_unfused": (dict(fc_sizes=(96,), N=2, h=1, dff=384, p=0.1), 4, 48),
    "s300_unfused": (dict(fc_sizes=(64,), N=1, h=2, dff=128, p=0.3), 3, 300),
    "bf16": (dict(fc_sizes=(64,), p_fc=0.2, N=2, h=2, dff=128, p=0.3, compute_dtype="bf16"), 5, 64),
    "d_output4": (dict(fc_sizes=(64,), N=1, h=2, dff=128, p=0.4, d_output=4, out_act="Sigmoid"), 5, 48),
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_device_seed_gives_the_host_seeded_bits(shape, monkeypatch):
    kw, B, S = SHAPES[shape]
    model = _model(**kw)
    x, y = _batch(B, S)
    mask = y == -1
    g = torch.Generator(device="cuda").manual_seed(2)
    out_shape = (B, S) if model.d_output == 1 else (B, S, model.d_output)
    ws = torch.randn(out_shape, device="cuda", generator=g)
    wh = torch.randn(B, S, model.d_model, device="cuda", generator=g)
    s = 0x2545F4914F6CDD1D
    monkeypatch.setattr(model, "_draw_seed", lambda: s)
    host = _pass(model, x, mask, ws, wh)
    monkeypatch.setattr(model, "_draw_seed", lambda: s + 1)
    other = _pass(model, x, mask, ws, wh)
    monkeypatch.setattr(model, "_draw_seed", lambda: pytest.fail("the device-seeded path drew a host seed"))
    with model.dropout_seed_from(_seed_tensor(s)):
        dev = _pass(model, x, mask, ws, wh)
    names = ["scores", "x.grad (scores)", "prepare_for_output", "x.grad (prepare_for_output)", "flat_gradients"]
    for name, a, b in zip(names, host, dev):
        assert torch.equal(a, b), name
    assert not torch.equal(host[0], other[0])          # the seed reaches the masks


def test_the_seed_is_read_when_a_captured_forward_runs(monkeypatch):
    """A forward captured once applies the masks of whatever value the seed tensor holds at replay time."""
    p = 0.25
    model = _model(fc_sizes=(64,), N=0, p_fc=p, F=20)
    x, y = _batch(64, 120, F=20)
    mask = y == -1
    with torch.no_grad():
        model.output_layer.w_1.weight.zero_()
        model.output_layer.w_1.weight[0, 5] = 1.0        # scores = one column of dropout(FC(x)): the mask shows
        model.output_layer.w_1.bias.zero_()
    seed = _seed_tensor(11)
    with torch.no_grad(), model.dropout_seed_from(seed):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            model(x, mask, None)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = model(x, mask, None)
    s1, s2 = 1234567, 1234568
    replays = []
    for s in (s1, s2):
        seed.fill_(s)
        graph.replay()
        replays.append(out.clone())
    eager = []
    with torch.no_grad():
        for s in (s1, s2):
            monkeypatch.setattr(model, "_draw_seed", lambda s=s: s)
            eager.append(model(x, mask, None))
    assert torch.equal(replays[0], eager[0]) and torch.equal(replays[1], eager[1])
    assert not torch.equal(replays[0], replays[1])
    real = ~mask
    n = int(real.sum().item())
    for r in replays:
        frac = (r[real] == 0).float().mean().item()
        assert abs(frac - p) <= 5 * math.sqrt(p * (1 - p) / n), (frac, n)


CONFIGS = {   # the models and losses of the shipped configurations, at a smaller batch
    "ndcgloss2pp": (dict(fc_sizes=(128,), N=4, h=4, dff=512, p=0.3), "lambdaLoss",
                    {"weighing_scheme": "ndcgLoss2PP_scheme", "k": None, "mu": 10, "sigma": 1.0}),
    "approxndcg": (dict(fc_sizes=(96,), N=2, h=1, dff=384, p=0.1), "approxNDCGLoss", {"alpha": 1.0}),
    "ordinal_mlp": (dict(fc_sizes=(256, 512, 1024, 512, 256), fc_act="ReLU", p_fc=0.3, N=0, d_output=4,
                         out_act="Sigmoid"), "ordinal", {"n": 4}),
    "ordinal": (dict(fc_sizes=(144,), N=4, h=2, dff=512, p=0.4, d_output=4, out_act="Sigmoid"), "ordinal", {"n": 4}),
}


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_graphed_dropout_training_equals_eager_training(config, monkeypatch):
    from allrank_b200 import losses
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.optim import FlatAdam
    kw, loss_name, loss_kw = CONFIGS[config]
    loss_fn = getattr(losses, loss_name)
    batches = [_batch(16, 240, seed=20 + k) for k in range(2)] * 4
    s = 977

    eager = _model(**kw)
    opt = FlatAdam(eager, lr=1e-3, capturable=True)
    eager_losses = []
    for k, (x, y) in enumerate(batches, start=1):
        monkeypatch.setattr(eager, "_draw_seed", lambda k=k: s + k)
        loss = loss_fn(eager(x, y == -1, None), y, **loss_kw)
        opt.zero_grad()
        loss.backward()
        opt.step()
        eager_losses.append(loss.item())

    graphed = _model(**kw)
    gopt = FlatAdam(graphed, lr=1e-3, capturable=True)
    init = {k: v.clone() for k, v in graphed.state_dict().items()}
    monkeypatch.setattr(graphed, "_draw_seed", lambda: pytest.fail("the graphed step drew a host seed"))
    step = GraphedTrainStep(graphed, loss_fn, gopt, *batches[0], loss_kwargs=loss_kw, warmup=2, dropout_seed=s)
    assert step.dropout_seed.item() == s
    graphed.load_state_dict(init)          # rewind what the warm-up steps trained
    gopt.exp_avg.zero_(); gopt.exp_avg_sq.zero_(); gopt._dev_state.zero_()
    graph_losses = [step(x, y).item() for x, y in batches]
    assert step.dropout_seed.item() == s + len(batches)
    assert graph_losses == eager_losses
    assert torch.equal(graphed.flat_parameters, eager.flat_parameters)


def test_refusals():
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.losses import listNet
    from allrank_b200.optim import FlatAdam
    model = _model(fc_sizes=(64,), N=1, h=2, dff=128, p=0.2)
    for bad in (torch.tensor([3], dtype=torch.int64),                       # host memory
                torch.tensor([3], dtype=torch.int32, device="cuda"),
                torch.tensor([3.0], device="cuda"),
                torch.tensor([3, 4], dtype=torch.int64, device="cuda"),
                torch.tensor(3, dtype=torch.int64, device="cuda").expand(2),
                3):
        with pytest.raises(ValueError):
            with model.dropout_seed_from(bad):
                pass
    x, y = _batch(4, 32)
    for bad in (1.5, "7", True, _seed_tensor(7)):
        with pytest.raises(ValueError):
            GraphedTrainStep(model, listNet, FlatAdam(model, capturable=True), x, y, dropout_seed=bad)
