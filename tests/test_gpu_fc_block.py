"""General FCModel input block (allrank/models/model.py:16-44) in the CUDA scorer: any number of layers, ReLU / Tanh /
Sigmoid / identity activation, nn.LayerNorm on the features, per-layer dropout -- alone (transformer=None) and in
front of the encoder, with and without positional encodings.  Oracle: oracle/scorer_ref.py (eval, fp32) and
oracle/tf32_emulation.py (train mode under regenerated dropout masks)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = [
    # F, sizes, act, input_norm, N, h, dff, positional, d_output, out_act
    (20, [32, 48, 32], "ReLU", False, 0, 1, 4, None, 1, None),
    (20, [32, 48, 32], "Tanh", True, 0, 1, 4, None, 3, "Sigmoid"),
    (136, [64, 32], "Sigmoid", True, 1, 2, 64, None, 1, None),
    (20, [24, 32], "ReLU", False, 2, 2, 64, ("fixed", 15), 1, "Tanh"),
    (20, [40, 32], "Tanh", False, 1, 2, 64, ("learned", 15), 1, None),
    (20, [32, 32, 32, 32], None, True, 1, 4, 32, None, 1, None),
]


def build_pair(case, p=0.0, p_fc=0.0):
    from allrank_b200.model import make_model
    from oracle.scorer_ref import make_ref_model
    Fn, sizes, act, inorm, N, h, dff, pos, n_out, out_act = case
    ref = make_ref_model(Fn, list(sizes), N, h, dff, dropout=0.0, d_output=n_out, output_activation=out_act,
                         fc_activation=act, seed=3, positional=pos, input_norm=inorm)
    gen = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for _, q in ref.named_parameters():
            if q.dim() == 1:
                q.add_(0.1 * torch.randn(q.shape, generator=gen))
    tcfg = None
    if N > 0:
        pe = None if pos is None else {"strategy": pos[0], "max_indices": pos[1]}
        tcfg = {"N": N, "d_ff": dff, "h": h, "positional_encoding": pe, "dropout": p}
    mine = make_model(fc_model={"sizes": list(sizes), "input_norm": inorm, "activation": act, "dropout": p_fc},
                      transformer=tcfg, post_model={"d_output": n_out, "output_activation": out_act}, n_features=Fn)
    assert list(mine.state_dict().keys()) == list(ref.state_dict().keys())
    mine.load_state_dict(ref.state_dict())
    return ref, mine.cuda()


@pytest.mark.parametrize("case", CASES)
def test_fc_block_eval_forward_and_backward_match_the_oracle(case, dense_rows):
    # (dense rows: the gradient weights cover the padded items too, like the oracle's)
    from allrank_b200.synth import make_slates
    ref, mine = build_pair(case)
    ref.eval(); mine.eval()
    B, S = 5, 20
    x, y, idx = make_slates(B, S, n_features=case[0], seed=8, mean_len=14, std_len=4)
    gen = torch.Generator().manual_seed(12)
    idx = torch.where(idx >= 0, torch.stack([torch.randperm(S, generator=gen) for _ in range(B)]), idx)
    mask = y == -1
    out_ref = ref(x, mask, idx)
    out = mine(x.cuda(), mask.cuda(), idx.cuda())
    w = torch.randn(out_ref.shape, generator=gen)
    (out_ref * w).sum().backward()
    (out * w.cuda()).sum().backward()
    valid = ~mask
    err = (out.detach().cpu() - out_ref.detach())[valid].abs().max().item()
    assert err <= 5e-3 * max(1.0, out_ref.detach()[valid].abs().max().item()), err
    rp = dict(ref.named_parameters())
    gmax = max(q.grad.abs().max().item() for q in rp.values() if q.grad is not None)
    for k, q in mine.named_parameters():
        r = rp[k].grad
        if r is None:
            continue
        rel = (q.grad.cpu() - r).norm().item() / max(r.norm().item(), 1e-2 * gmax * np.sqrt(r.numel()))
        assert rel <= 5e-2, (k, rel)
    # score() of a multi-output head sums the outputs (model.py:119-128)
    with torch.no_grad():
        sc = mine.score(x.cuda(), mask.cuda(), idx.cuda()).cpu()
        assert torch.allclose(sc[valid], ref.score(x, mask, idx)[valid], atol=2e-2)


@pytest.mark.parametrize("case", [CASES[0], CASES[1], CASES[2], CASES[5]])
def test_fc_block_train_mode_uses_the_same_masks_forward_and_backward(case):
    """Per-layer FC dropout (+ encoder dropout): scores and all gradients against the eager maths under the kernels'
    regenerated masks."""
    from allrank_b200.synth import make_slates
    from oracle.tf32_emulation import scorer_forward
    from tests.dropout_masks import scorer_masks
    Fn, sizes, act, inorm, N, h, dff, pos, n_out, out_act = case
    p, p_fc = (0.2 if N else 0.0), 0.25
    _, mine = build_pair(case, p=p, p_fc=p_fc)
    mine.train()
    B, S = 6, 24
    x, y, _ = make_slates(B, S, n_features=Fn, seed=9, mean_len=16, std_len=5)
    mask = y == -1
    torch.manual_seed(31)
    call_seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    torch.manual_seed(31)
    out = mine(x.cuda(), mask.cuda(), None)
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(6))
    (out * w.cuda()).sum().backward()
    sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in mine.state_dict().items()}
    ref = scorer_forward(sd, x, mask, N, h, out_act, "rna",
                         drop=scorer_masks(call_seed, B, S, sizes, N, h, dff, p, p_fc), fc_act=act)
    (ref * w).sum().backward()
    valid = ~mask
    err = (ref.detach() - out.detach().cpu())[valid].abs().max().item()
    assert err <= 3e-3 * max(1.0, ref.detach()[valid].abs().max().item()), err
    floor = 1e-2 * max(v.grad.abs().max().item() for v in sd.values())
    errs = {}
    for k, q in mine.named_parameters():
        a, r = q.grad.cpu().double().numpy(), sd[k].grad.double().numpy()
        errs[k] = np.linalg.norm(a - r) / max(np.linalg.norm(r), floor * np.sqrt(r.size))
    print(case[:4], {k: round(float(v), 4) for k, v in errs.items()})
    above_relu = ("feed_forward.w_2", "encoder.norm", "output_layer")
    for k, v in errs.items():
        # Under identical dropout masks the CUDA path and the eager maths still differ by TF32-level rounding in the
        # forward (the fused attention rounds the un-normalised probabilities, the eager maths the normalised ones: scores
        # agree to 1e-3).  A hidden unit whose pre-activation lies within that noise of zero then has ReLU derivative 1 on
        # one side and 0 on the other; a fraction f of such units moves the gradients BELOW the first ReLU by ~sqrt(f)
        # (2-8 % on these small models, 0.03 % with the unfused attention path whose rounding matches the eager maths
        # exactly), while gradients above
        # it (w_2, final norm, head) agree to 1e-3.  Mask mismatches would show as O(1) errors everywhere.
        tight = N == 0 or any(t in k for t in above_relu)
        assert v <= (3e-2 if tight else 1e-1), (k, v)
