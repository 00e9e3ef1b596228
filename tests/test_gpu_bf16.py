"""bf16 mode of the scorer (BASELINE config 3: Transformer(N=4, h=8, d=256) + lambdaLoss ndcgLoss2++, bf16):
every encoder linear is a tensor-core product of bfloat16 operands with fp32 accumulation; residual stream,
LayerNorm statistics, softmax, head, loss and parameter gradients stay fp32.
Bounds: SURVEY.md 8(c) L2 for bf16 -- score abs error <= 6e-2 at unit-scale scores, NDCG@10 within 5e-3, loss within
1e-2 relative of the fp32 oracle -- and an order tighter against the bf16-operand emulation of the same maths
(oracle/tf32_emulation.py, bf16=True)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def build(F, d, N, h, dff, seed=3, p=0.0):
    from allrank_b200.model import make_model
    from oracle.scorer_ref import make_ref_model
    ref = make_ref_model(F, [d], N, h, dff, dropout=0.0, seed=seed)
    gen = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for _, q in ref.named_parameters():
            if q.dim() == 1:
                q.add_(0.1 * torch.randn(q.shape, generator=gen))
    mine = make_model(fc_model={"sizes": [d], "input_norm": False, "activation": None, "dropout": 0.0},
                      transformer={"N": N, "d_ff": dff, "h": h, "positional_encoding": None, "dropout": p},
                      post_model={"d_output": 1, "output_activation": None}, n_features=F, compute_dtype="bf16")
    mine.load_state_dict(ref.state_dict())
    return ref, mine.cuda()


@pytest.mark.parametrize("shape", [(136, 256, 4, 8, 1024, 6, 240), (136, 128, 2, 4, 512, 5, 120), (20, 64, 1, 2, 128, 7, 37)])
def test_bf16_scores_loss_and_ndcg_within_the_contract_of_the_fp32_reference(shape):
    from allrank_b200 import losses, metrics
    from allrank_b200.synth import make_slates
    from oracle import losses_ref, metrics_ref
    F, d, N, h, dff, B, S = shape
    ref, mine = build(F, d, N, h, dff)
    ref.eval(); mine.eval()
    x, y, idx = make_slates(B, S, n_features=F, seed=8, mean_len=0.6 * S, std_len=0.25 * S)
    mask = y == -1
    with torch.no_grad():
        s_ref = ref(x, mask, idx)
        s = mine(x.cuda(), mask.cuda(), None).cpu()
    valid = ~mask
    scale = max(1.0, s_ref[valid].abs().max().item())
    err = (s - s_ref)[valid].abs().max().item()
    assert err <= 6e-2 * scale, err
    kw = {"weighing_scheme": "ndcgLoss2PP_scheme", "k": None, "mu": 10.0, "sigma": 1.0}
    l_ref = losses_ref.lambdaLoss(s_ref, y, **kw).item()
    l = losses.lambdaLoss(s.cuda(), y.cuda(), **kw).item()
    assert abs(l - l_ref) <= 1e-2 * abs(l_ref), (l, l_ref)
    nd_ref = metrics_ref.ndcg(s_ref, y, ats=[10]).mean().item()
    nd = metrics.ndcg(s.cuda(), y.cuda(), ats=[10]).mean().item()
    assert abs(nd - nd_ref) <= 5e-3, (nd, nd_ref)
    print("bf16 vs fp32:", shape, "score err", err, "loss", l, l_ref, "ndcg@10", nd, nd_ref)


@pytest.mark.parametrize("shape,p", [((136, 256, 2, 8, 1024, 4, 240), 0.0), ((136, 128, 2, 4, 512, 5, 120), 0.2),
                                     ((20, 64, 1, 2, 128, 7, 37), 0.1)])
def test_bf16_forward_and_backward_match_the_bf16_operand_emulation(shape, p):
    """Same weights, same dropout masks (regenerated on the host): scores and every parameter gradient against the
    eager maths with bfloat16-rounded operands -- an order tighter than the fp32 contract, so a kernel bug cannot hide
    behind the bf16 tolerance."""
    from allrank_b200.synth import make_slates
    from oracle.tf32_emulation import scorer_forward
    from tests.dropout_masks import scorer_masks
    F, d, N, h, dff, B, S = shape
    _, mine = build(F, d, N, h, dff, p=p)
    mine.train()
    x, y, _ = make_slates(B, S, n_features=F, seed=9, mean_len=0.6 * S, std_len=0.25 * S)
    mask = y == -1
    torch.manual_seed(31)
    call_seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if p > 0 else 0
    torch.manual_seed(31)
    out = mine(x.cuda(), mask.cuda(), None)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(6))
    w = torch.where(mask, torch.zeros_like(w), w)
    (out * w.cuda()).sum().backward()
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in mine.state_dict().items()}
    ref = scorer_forward(sd, x, mask, N, h, None, "rna", drop=scorer_masks(call_seed, B, S, [d], N, h, dff, p, 0.0),
                         bf16=True)
    (ref * w).sum().backward()
    valid = ~mask
    err = (ref.detach() - out.detach().cpu())[valid].abs().max().item()
    assert err <= 6e-3 * max(1.0, ref.detach()[valid].abs().max().item()), err
    floor = 1e-2 * max(v.grad.abs().max().item() for v in sd.values())
    worst = 0.0
    for k, q in mine.named_parameters():
        a, r = q.grad.cpu().double().numpy(), sd[k].grad.double().numpy()
        fro = np.linalg.norm(a - r) / max(np.linalg.norm(r), floor * np.sqrt(r.size))
        worst = max(worst, fro)
        # bfloat16 keeps 8 mantissa bits (tf32: 11): the emulation rounds the same operands but not in the same
        # order everywhere (e.g. delta = rowsum(dO * O) reads the bf16 context), so gradients agree to a few 2^-8 steps
        assert fro <= 1e-1, (k, fro)
    print("bf16 vs emulation:", shape, "p", p, "score err", err, "worst grad rel err", worst)


def test_bf16_training_reduces_the_loss_and_tracks_tf32():
    """A short training run in both arithmetic modes from the same initialisation: both converge, final losses close."""
    from allrank_b200 import losses
    from allrank_b200.model import make_model
    from allrank_b200.optim import FlatAdam
    from allrank_b200.synth import make_slates
    x, y, _ = make_slates(64, 120, 136, seed=9, mean_len=70, std_len=20)
    x, y = x.cuda(), y.cuda()
    final = {}
    for dtype in ("tf32", "bf16"):
        torch.manual_seed(6)
        model = make_model(fc_model={"sizes": [128], "input_norm": False, "activation": None, "dropout": 0.0},
                           transformer={"N": 2, "d_ff": 256, "h": 4, "positional_encoding": None, "dropout": 0.0},
                           post_model={"d_output": 1, "output_activation": None}, n_features=136,
                           compute_dtype=dtype).cuda().train()
        opt = FlatAdam(model, lr=1e-3)
        first = None
        for _ in range(40):
            loss = losses.approxNDCGLoss(model(x, y == -1, None), y)
            loss.backward(); opt.step(); opt.zero_grad()
            first = loss.item() if first is None else first
        final[dtype] = loss.item()
        assert np.isfinite(final[dtype]) and final[dtype] < first
    assert abs(final["bf16"] - final["tf32"]) <= 2e-2 * abs(final["tf32"]), final
