"""Layer widths that are not multiples of 4 on the GPU (FC sizes, d_model, d_ff): the scorer stores a layer of n columns
with round_up(n, 4) columns whose pads are exact zeros (DESIGN.md 4.16) and runs every product and row kernel at the
stored width, the LayerNorm statistics over the real columns; the dropout counters keep the real layout
(row * n + column).  Encoder shapes run at S = 240 and S = 1024.

Against oracle/scorer_ref.py (eval, fp32: scores, every parameter gradient, x.grad and prepare_for_output), the TF32
emulation under the regenerated dropout masks of the real widths (train mode), and the golden vectors of the unmodified
reference (tests/golden/scorer_odd_widths.npz, tools/make_golden_odd_widths.py).  The pads of the parameters and of
their gradients are +0 after FlatAdam steps with weight decay, repeated steps give the same bits, a graphed dropout
step equals the eager one, and the reference's rank_slates model ranks through allrank_b200.inference."""
import numpy as np
import pytest
import torch

from tests.test_gpu_fc_block import build_pair
from tests.test_host_odd_widths import golden_model

pytestmark = pytest.mark.gpu

CASES = [
    # F, sizes, act, input_norm, N, h, dff, positional, d_output, out_act
    (10, [10], None, False, 0, 1, 4, None, 1, None),          # the reference's rank_slates model
    (10, [10, 6], "ReLU", False, 0, 1, 4, None, 1, None),
    (46, [50, 30], "ReLU", False, 0, 1, 4, None, 1, None),
    (46, [50, 30], "Tanh", False, 0, 1, 4, None, 3, None),
    (46, [50, 30], "Sigmoid", False, 0, 1, 4, None, 1, "Sigmoid"),
    (46, [7, 1], None, False, 0, 1, 4, None, 2, None),
    (46, [46, 64], "ReLU", False, 1, 4, 128, None, 1, None),   # odd FC hidden width in front of an encoder
    (46, [30, 64], "Sigmoid", False, 1, 2, 128, ("learned", 250), 1, None),
    # encoders whose d_model and / or d_ff are not multiples of 4 (heads of 5, 23, 65, 127 and 2 columns, padded)
    (46, [10], None, False, 2, 2, 20, None, 1, None),
    (46, [46], "ReLU", False, 2, 2, 30, None, 1, None),
    (46, [130], None, False, 1, 2, 262, None, 1, None),
    (46, [254], None, False, 1, 2, 508, None, 1, None),
    (46, [6], None, False, 1, 3, 14, None, 3, None),
    (46, [64], None, False, 1, 4, 30, None, 1, None),
    (46, [10], None, False, 1, 2, 22, ("learned", 1100), 1, None),
    (46, [10], "Tanh", False, 1, 2, 20, ("fixed", 1100), 1, None),
]
ENC = [c for c in CASES if c[4] > 0 and (c[1][-1] % 4 or c[6] % 4)]
IDS = [f"F{c[0]}-{'x'.join(map(str, c[1]))}-{c[2]}-N{c[4]}h{c[5]}f{c[6]}-{c[7] and c[7][0]}-o{c[8]}" for c in CASES]


def _slates(B, S, F, seed):
    from allrank_b200.synth import make_slates
    x, y, idx = make_slates(B, S, n_features=F, seed=seed, mean_len=int(0.6 * S), std_len=S // 5)
    return x, y, idx


def _pads(model, flat):
    """The entries of a flat buffer outside every parameter's view (the pads and alignment gaps)."""
    n = flat.numel()
    covered = torch.zeros(n, dtype=torch.bool, device=flat.device)
    base = model.flat_parameters.data_ptr()
    for p in model.parameters():
        idx = torch.arange(n, device=flat.device).as_strided(p.shape, p.stride(), (p.data_ptr() - base) // 4)
        covered[idx.flatten()] = True
    return flat[~covered]


def _assert_pos_zero(t, what):
    t = t.contiguous()
    assert torch.equal(t.view(torch.int32), torch.zeros_like(t).view(torch.int32)), f"{what} are not +0"


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_eval_matches_the_oracle_with_input_gradient_and_hidden(case, dense_rows):
    # (dense rows: the gradient weights cover the padded items too, like the oracle's)
    ref, mine = build_pair(case)
    ref.eval(); mine.eval()
    B, S = 4, 240
    x, y, idx = _slates(B, S, case[0], seed=8)
    mask = y == -1
    xr = x.clone().requires_grad_(True)
    xm = x.cuda().requires_grad_(True)
    out_ref = ref(xr, mask, idx)
    out = mine(xm, mask.cuda(), idx.cuda())
    w = torch.randn(out_ref.shape, generator=torch.Generator().manual_seed(12))
    (out_ref * w).sum().backward()
    (out * w.cuda()).sum().backward()
    valid = ~mask
    err = (out.detach().cpu() - out_ref.detach())[valid].abs().max().item()
    assert err <= 5e-3 * max(1.0, out_ref.detach()[valid].abs().max().item()), err
    rp = dict(ref.named_parameters())
    gmax = max(q.grad.abs().max().item() for q in rp.values() if q.grad is not None)
    for k, q in mine.named_parameters():
        r = rp[k].grad
        rel = (q.grad.cpu() - r).norm().item() / max(r.norm().item(), 1e-2 * gmax * np.sqrt(r.numel()))
        assert rel <= 5e-2, (k, rel)
    gx, rx = xm.grad.cpu()[valid], xr.grad[valid]
    assert (gx - rx).norm().item() <= 5e-2 * max(rx.norm().item(), 1e-6), "x.grad"
    _assert_pos_zero(_pads(mine, mine.flat_gradients), "gradient pads")
    # prepare_for_output: [B, S, d] and its backward
    with torch.no_grad():
        hid = mine.prepare_for_output(x.cuda(), mask.cuda(), idx.cuda()).cpu()
        hid_ref = ref.prepare_for_output(x, mask, idx)
    assert hid.shape == hid_ref.shape == (B, S, case[1][-1])
    assert (hid - hid_ref)[valid].abs().max().item() <= 5e-3 * max(1.0, hid_ref[valid].abs().max().item())
    mine.zero_grad(set_to_none=True)
    for q in ref.parameters():
        q.grad = None
    wh = torch.randn(hid.shape, generator=torch.Generator().manual_seed(13))
    (ref.prepare_for_output(x, mask, idx) * wh).sum().backward()
    (mine.prepare_for_output(x.cuda(), mask.cuda(), idx.cuda()) * wh.cuda()).sum().backward()
    for k, q in mine.named_parameters():
        r = rp[k].grad
        if r is None or k.startswith("output_layer"):
            continue
        rel = (q.grad.cpu() - r).norm().item() / max(r.norm().item(), 1e-2 * gmax * np.sqrt(r.numel()))
        assert rel <= 5e-2, ("hidden", k, rel)


NO_PE = [c for c in CASES if c[7] is None]


@pytest.mark.parametrize("case", ENC, ids=[i for c, i in zip(CASES, IDS) if c in ENC])
def test_encoders_at_1024_items_match_the_oracle(case, dense_rows):
    """Eval scores and every parameter gradient at S = 1024 (the streaming attention kernels at the padded heads)."""
    ref, mine = build_pair(case)
    ref.eval(); mine.eval()
    B, S = 2, 1024
    x, y, idx = _slates(B, S, case[0], seed=18)
    mask = y == -1
    out_ref = ref(x, mask, idx)
    out = mine(x.cuda(), mask.cuda(), idx.cuda())
    w = torch.randn(out_ref.shape, generator=torch.Generator().manual_seed(14))
    (out_ref * w).sum().backward()
    (out * w.cuda()).sum().backward()
    valid = ~mask
    err = (out.detach().cpu() - out_ref.detach())[valid].abs().max().item()
    assert err <= 5e-3 * max(1.0, out_ref.detach()[valid].abs().max().item()), err
    rp = dict(ref.named_parameters())
    gmax = max(q.grad.abs().max().item() for q in rp.values() if q.grad is not None)
    for k, q in mine.named_parameters():
        r = rp[k].grad
        rel = (q.grad.cpu() - r).norm().item() / max(r.norm().item(), 1e-2 * gmax * np.sqrt(r.numel()))
        assert rel <= 5e-2, (k, rel)
    _assert_pos_zero(_pads(mine, mine.flat_gradients), "gradient pads")


@pytest.mark.parametrize("case", NO_PE, ids=[i for c, i in zip(CASES, IDS) if c[7] is None])
def test_train_mode_uses_the_real_width_masks(case):
    """FC dropout (+ encoder dropout) at padded widths: scores, every gradient and x.grad against the eager maths
    under the masks of tests/dropout_masks.scorer_masks over the REAL widths."""
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
    drop = scorer_masks(call_seed, B, S, sizes, N, h, dff, p, p_fc)
    ref = scorer_forward(sd, xe, mask, N, h, out_act, "rna", drop=drop, fc_act=act)
    (ref * w).sum().backward()
    valid = ~mask
    err = (ref.detach() - out.detach().cpu())[valid].abs().max().item()
    assert err <= 3e-3 * max(1.0, ref.detach()[valid].abs().max().item()), err
    floor = 1e-2 * max(v.grad.abs().max().item() for v in sd.values())
    for k, q in mine.named_parameters():
        a, r = q.grad.cpu().double().numpy(), sd[k].grad.double().numpy()
        rel = np.linalg.norm(a - r) / max(np.linalg.norm(r), floor * np.sqrt(r.size))
        assert rel <= (3e-2 if N == 0 else 1e-1), (k, rel)
    rel = (xm.grad.cpu() - xe.grad).norm().item() / max(xe.grad.norm().item(), 1e-6)
    assert rel <= (3e-2 if N == 0 else 1e-1), ("x.grad", rel)
    _assert_pos_zero(_pads(mine, mine.flat_gradients), "gradient pads")


@pytest.mark.parametrize("name", ["f10s10", "f46s10_6", "f46s50_30t", "f46s50_30s", "f46s46_64e", "d10h2", "d46h2f30",
                                  "d130h2", "d6h3o3"])
def test_eval_matches_the_reference_golden_vectors(golden, name):
    g = golden("scorer_odd_widths")
    model = golden_model(g, name).cuda().eval()
    F = int(g[name + ":F"])
    x, y = torch.tensor(g[f"x{F}"]).cuda(), torch.tensor(g[f"y{F}"]).cuda()
    out = model(x, y == -1, None)
    ref = torch.tensor(g[name + ":scores"])
    valid = (y != -1).cpu()
    err = (out.detach().cpu() - ref)[valid].abs().max().item()
    assert err <= 5e-3 * max(1.0, ref[valid].abs().max().item()), err
    (out * torch.tensor(g[name + ":w"]).cuda()).sum().backward()
    params = dict(model.named_parameters())
    rms_max = max(float(g[name + ":n:" + k]) / np.sqrt(p.numel()) for k, p in params.items())
    for k, p in params.items():
        n = p.numel()
        gi = torch.arange(n) if n <= 1024 else torch.linspace(0, n - 1, 1024).long()
        got = p.grad.detach().flatten().cpu()[gi].double().numpy()
        want = g[name + ":g:" + k].astype(np.float64)
        fro = np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-2 * rms_max * np.sqrt(len(gi)))
        nrm = abs(p.grad.norm().item() - float(g[name + ":n:" + k])) / max(float(g[name + ":n:" + k]),
                                                                           1e-2 * rms_max * np.sqrt(n))
        assert fro <= 5e-2 and nrm <= 5e-2, (k, fro, nrm)


def _train(case, steps, B=8, S=240, p_fc=0.25):
    from allrank_b200 import losses
    from allrank_b200.optim import FlatAdam
    _, mine = build_pair(case, p=0.1 if case[4] else 0.0, p_fc=p_fc)
    mine.train()
    opt = FlatAdam(mine, lr=1e-2, weight_decay=0.1)
    torch.manual_seed(5)
    for k in range(steps):
        x, y, idx = _slates(B, S, case[0], seed=40 + k)
        loss = losses.approxNDCGLoss(mine.score(x.cuda(), (y == -1).cuda(), idx.cuda() if case[7] else None), y.cuda())
        opt.zero_grad()
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    return mine


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_pads_stay_zero_through_flat_adam_and_steps_repeat_bit_for_bit(case):
    a = _train(case, 3)
    _assert_pos_zero(_pads(a, a.flat_parameters), "parameter pads")
    _assert_pos_zero(_pads(a, a.flat_gradients), "gradient pads")
    assert a.flat_parameters.isfinite().all()
    b = _train(case, 3)
    assert torch.equal(a.flat_parameters, b.flat_parameters)
    assert torch.equal(a.flat_gradients, b.flat_gradients)


@pytest.mark.parametrize("case", [CASES[2], CASES[4], CASES[6], CASES[8], CASES[10]],
                         ids=[IDS[2], IDS[4], IDS[6], IDS[8], IDS[10]])
def test_graphed_dropout_step_equals_the_eager_step(case, monkeypatch):
    from allrank_b200 import losses
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.optim import FlatAdam
    batches = [_slates(8, 240, case[0], seed=20 + k)[:2] for k in range(2)] * 2
    batches = [(x.cuda(), y.cuda()) for x, y in batches]
    s = 977
    p = 0.1 if case[4] else 0.0
    _, eager = build_pair(case, p=p, p_fc=0.25)
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
    _, graphed = build_pair(case, p=p, p_fc=0.25)
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


def test_the_reference_rank_slates_model_ranks():
    """The model of the reference's tests/test_rank_slates.py (F 10, sizes [10]) through rank_dataloader."""
    from torch.utils.data import DataLoader

    from allrank_b200.inference import rank_dataloader
    from allrank_b200.model import make_model
    rng = np.random.RandomState(42)
    X = [rng.rand(5, 10).astype(np.float32) for _ in range(2)]
    y_true = [rng.randint(0, 1, size=len(x)) for x in X]
    indices = [np.zeros(len(x)) for x in X]
    model = make_model({"sizes": [10], "input_norm": False, "activation": None, "dropout": None}, None,
                       {"d_output": 1}, 10).cuda()
    loader = DataLoader(list(zip(X, y_true, indices)), batch_size=2)
    slates_x, slates_y = rank_dataloader(loader, model)
    assert len(slates_x) == len(X) and len(slates_y) == len(y_true)
    with torch.no_grad():
        scores = model(torch.tensor(np.stack(X)).cuda(), torch.zeros(2, 5, dtype=torch.bool).cuda()).cpu()
    for b in range(2):
        order = torch.argsort(scores[b], descending=True)
        assert torch.equal(slates_x[b], torch.tensor(X[b])[order])
