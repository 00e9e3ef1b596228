"""Every model configuration the reference ships -- reproducibility/configs/{contextaware,neuralndcg}_web30k/*.json
and scripts/local_config.json -- must build, score and train through the CUDA scorer with the config's own dropout:
single-layer FC + Transformer with head widths 32 / 64 / 72 / 96, the 5-layer ReLU MLPs (`*_mlp.json`, no
transformer), 4-output Sigmoid heads (ordinal), Tanh heads (neuralNDCG).

Golden vectors: tests/golden/scorer_shipped_configs.npz, written by oracle/make_golden.py from the UNMODIFIED
reference's make_model (/root/reference/allrank/models/model.py:131-151) at MSLR shape (136 features, slate length
240, eval mode).  The file stores the `model` section of each JSON, so nothing here reads /root/reference.
"""
import json

import numpy as np
import pytest
import torch

NAMES = ["ndcgloss2pp", "ndcgloss2pp_mlp", "ordinal", "ordinal_mlp", "approxndcg", "lambdarank_atmax",
         "neuralndcg_atmax", "local_config"]
F = 136


def build(golden, name, device=None):
    """make_model from the stored JSON under the seed the golden generator used, with the same perturbation of the
    1-D parameters (oracle/make_golden.py: gen_scorer_shipped / perturb_vectors)."""
    from allrank_b200.model import make_model
    g = golden("scorer_shipped_configs")
    m = json.loads(str(g[name + ":model"]))
    torch.manual_seed(77)
    model = make_model(fc_model=m["fc_model"], transformer=m["transformer"], post_model=m["post_model"], n_features=F)
    gen = torch.Generator().manual_seed(78)
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    return (model if device is None else model.to(device)), m, g


def grad_sample_index(numel, n=1024):
    return torch.arange(numel) if numel <= n else torch.linspace(0, numel - 1, n).long()


@pytest.mark.parametrize("name", NAMES)
def test_shipped_config_builds_with_the_reference_initialisation(golden, name):
    """Host side (no GPU): same state_dict keys as the reference and, under the same seed, the same parameter values
    (checksums of every tensor) -- multi-layer FC blocks and every head / encoder shape included."""
    model, m, g = build(golden, name)
    sd = model.state_dict()
    ref_keys = [k.split(":c:")[1] for k in g.files if k.startswith(name + ":c:")]
    assert list(sd.keys()) == ref_keys
    for k, v in sd.items():
        want = g[name + ":c:" + k]
        got = np.array([v.double().sum().item(), v.double().abs().sum().item()])
        assert np.array_equal(got, want), (k, got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_shipped_config_eval_matches_the_reference(golden, name, dense_rows):
    """Scores within the TF32 bound (5e-3 abs at unit scale, SURVEY.md 8c L2) of the reference's fp32 run and every
    parameter gradient (sampled positions + norm) within 5 %.  (Dense rows: the golden gradients weight the padded
    items too.)"""
    model, m, g = build(golden, name, "cuda")
    model.eval()
    x, y = torch.tensor(g["x"]).cuda(), torch.tensor(g["y"]).cuda()
    out = model(x, y == -1, None)
    ref = torch.tensor(g[name + ":scores"])
    assert tuple(out.shape) == tuple(ref.shape)
    valid = (y != -1).cpu()
    err = (out.detach().cpu() - ref)[valid].abs().max().item()
    assert err <= 5e-3 * max(1.0, ref[valid].abs().max().item()), err
    (out * torch.tensor(g[name + ":w"]).cuda()).sum().backward()
    worst = 0.0
    # gradients that are mathematically zero (the key-projection bias: softmax is invariant to a per-query shift of
    # the scores) are rounding noise on both sides: errors are measured against a floor tied to the largest
    # per-element gradient of the model, like the other scorer tests
    params = dict(model.named_parameters())
    rms_max = max(float(g[name + ":n:" + k]) / np.sqrt(p.numel()) for k, p in params.items())
    for k, p in params.items():
        gi = grad_sample_index(p.numel())
        got = p.grad.detach().flatten().cpu()[gi].double().numpy()
        want = g[name + ":g:" + k].astype(np.float64)
        floor = 1e-2 * rms_max * np.sqrt(len(gi))
        rel = np.linalg.norm(got - want) / max(np.linalg.norm(want), floor)
        worst = max(worst, rel)
        assert rel <= 5e-2, (k, rel)
        ref_norm = float(g[name + ":n:" + k])
        n_rel = abs(p.grad.norm().item() - ref_norm) / max(ref_norm, 1e-2 * rms_max * np.sqrt(p.numel()))
        assert n_rel <= 5e-2, (k, n_rel)
    print(name, "eval: score err", err, "worst sampled-gradient rel err", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_shipped_config_trains_with_its_dropout_like_the_reference_maths(golden, name):
    """train() mode with the config's dropout at B = 8, S = 240: the kernels' masks are regenerated on the host and fed
    to the eager functional scorer (oracle/tf32_emulation.py: the reference's maths with TF32-rounded matmuls); scores
    and every parameter gradient must agree.  Covers the unfused attention path under dropout (head widths 72 / 96),
    the fused forward + unfused backward pair (64) and the activated multi-layer FC block."""
    from allrank_b200.synth import make_slates
    from oracle.tf32_emulation import scorer_forward
    from tests.dropout_masks import scorer_masks
    model, m, g = build(golden, name, "cuda")
    model.train()
    B, S = 8, 240
    x, y, _ = make_slates(B, S, n_features=F, seed=43, mean_len=150, std_len=60)
    mask = y == -1
    tr = m["transformer"]
    N, h, dff, p = (tr["N"], tr["h"], tr["d_ff"], tr["dropout"]) if tr else (0, 1, 4, 0.0)
    p_fc = m["fc_model"]["dropout"] or 0.0
    sizes = m["fc_model"]["sizes"]
    torch.manual_seed(21)
    call_seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if (p > 0 or p_fc > 0) else 0   # LTRModel._draw_seed
    torch.manual_seed(21)
    out = model(x.cuda(), mask.cuda(), None)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(5))
    (out * w.cuda()).sum().backward()
    drop = scorer_masks(call_seed, B, S, sizes, N, h, dff, p, p_fc)
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    ref = scorer_forward(sd, x, mask, N, h, m["post_model"]["output_activation"], "rna", drop=drop,
                         fc_act=m["fc_model"]["activation"])
    (ref * w).sum().backward()
    valid = ~mask
    err = (ref.detach() - out.detach().cpu())[valid].abs().max().item()
    assert err <= 3e-3 * max(1.0, ref.detach()[valid].abs().max().item()), err
    floor = 1e-2 * max(v.grad.abs().max().item() for v in sd.values())
    worst = 0.0
    for k, q in model.named_parameters():
        a, r = q.grad.cpu().double().numpy(), sd[k].grad.double().numpy()
        fro = np.linalg.norm(a - r) / max(np.linalg.norm(r), floor * np.sqrt(r.size))
        worst = max(worst, fro)
        # Under identical dropout masks the CUDA path and the eager maths still differ by TF32-level rounding in the
        # forward (the fused attention rounds the un-normalised probabilities, the eager maths the normalised ones: scores
        # agree to 1e-3).  A hidden unit whose pre-activation lies within that noise of zero then has ReLU derivative 1 on
        # one side and 0 on the other; a fraction f of such units moves the gradients BELOW the first ReLU by ~sqrt(f)
        # (2-8 % on these small models, 0.03 % with the unfused attention path whose rounding matches the eager maths
        # exactly), while gradients above
        # it (w_2, final norm, head) agree to 1e-3.  Mask mismatches would show as O(1) errors everywhere.
        last = f"encoder.layers.{N - 1}.feed_forward.w_2" if N else "output_layer"
        tight = N == 0 or k.startswith(last) or k.startswith("encoder.norm") or k.startswith("output_layer")
        assert fro <= (3e-2 if tight else 1e-1), (k, fro)
    print(name, "train p =", p, "fc", p_fc, ": score err", err, "worst grad rel err", worst)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_shipped_config_runs_a_training_step_with_its_loss(golden, name):
    """loss_batch of the reference (train_utils.py:18-29) with the config's own loss and arguments: finite loss,
    finite gradients, parameters move."""
    from allrank_b200 import losses
    from allrank_b200.synth import make_slates
    model, m, g = build(golden, name, "cuda")
    model.train()
    cfg = json.loads(str(g[name + ":loss"]))
    loss_fn = getattr(losses, cfg["name"])
    x, y, _ = make_slates(16, 240, n_features=F, seed=44, mean_len=150, std_len=60)
    x, y = x.cuda(), y.cuda()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)       # what allrank/main.py:82 instantiates
    before = model.flat_parameters.clone() if model.flat_parameters is not None else None
    for _ in range(2):
        loss = loss_fn(model(x, y == -1, None), y, **cfg["args"])
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert np.isfinite(loss.item())
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())
    if before is not None:
        assert not torch.equal(before, model.flat_parameters)
