"""The fused attention forward (attn_fwd_kernel) computes every (slate, head) item on its own: a slate's scores and its
input gradient must be BIT-identical whatever batch it runs in -- alone, in reverse order, or embedded among many other
slates -- so that its items land in different CTAs, operand-pool slots and strip sequences.  The input gradient is
row-local and reads the forward's row statistics (max, sum) through the attention backward, so it pins those too.

Extents cover one item, both sides of every 16-row strip and 128-row boundary, full slates of 240 and 256 items and
(packed rows) empty slates; head widths 16, 32 and 64 (64 at S = 256: two items do not fit the operand pool side by
side), the bf16 context, and batches of several hundred slates (many items per CTA).  The values themselves are checked
element by element against an fp64 reference in tests/test_gpu_attention_kernels.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _model(d, h, dtype):
    from allrank_b200.model import make_model
    torch.manual_seed(5)
    m = make_model(fc_model={"sizes": [d], "input_norm": False, "activation": None, "dropout": 0.0},
                   transformer={"N": 1, "d_ff": 2 * d, "h": h, "positional_encoding": None, "dropout": 0.0},
                   post_model={"d_output": 1, "output_activation": None}, n_features=24, compute_dtype=dtype)
    gen = torch.Generator().manual_seed(6)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    return m.cuda().train()


def _slates(extents, S, F, seed):
    """One slate per extent: items below it real (but for one padded item inside longer slates), the rest padding."""
    g = torch.Generator().manual_seed(seed)
    B = len(extents)
    x = torch.randn(B, S, F, generator=g)
    y = torch.randint(0, 5, (B, S), generator=g).float()
    for b, e in enumerate(extents):
        y[b, e:] = -1.0
        x[b, e:] = 0.0
        if e > 20:
            y[b, e // 2] = -1.0
    w = torch.randn(B, S, generator=g)
    return x, y, torch.where(y == -1, torch.zeros_like(w), w)


def _run(model, x, y, w):
    xg = x.cuda().requires_grad_(True)
    model.zero_grad(set_to_none=True)
    s = model(xg, y.cuda() == -1, None)
    (s * w.cuda()).sum().backward()
    return s.detach().cpu(), xg.grad.detach().cpu()


def _bits(t):
    return t.contiguous().view(torch.int32)


CASES = [
    # (S, d_model, heads, compute dtype, extents; 0 = empty slate, packed rows only)
    (256, 128, 4, "tf32", [1, 15, 16, 17, 127, 128, 129, 240, 256, 0]),
    (37, 128, 4, "tf32", [1, 15, 16, 17, 36, 37, 0]),
    (256, 64, 4, "tf32", [1, 15, 16, 17, 127, 128, 129, 240, 256, 0]),
    (256, 128, 2, "tf32", [1, 15, 16, 17, 127, 128, 129, 240, 256]),
    (240, 128, 4, "bf16", [1, 15, 16, 17, 127, 128, 129, 240, 0]),
]


@pytest.mark.parametrize("S,d,h,dtype,extents", CASES, ids=["dk32-S256", "dk32-S37", "dk16-S256", "dk64-S256", "bf16-S240"])
def test_attention_forward_result_of_a_slate_does_not_depend_on_its_batch(S, d, h, dtype, extents):
    F = 24
    model = _model(d, h, dtype)
    x, y, w = _slates(extents, S, F, seed=11)
    n = len(extents)
    s0, g0 = _run(model, x, y, w)
    assert torch.isfinite(s0).all() and torch.isfinite(g0).all()

    rev = torch.arange(n - 1, -1, -1)
    s1, g1 = _run(model, x[rev], y[rev], w[rev])
    assert torch.equal(_bits(s1[rev]), _bits(s0))
    assert torch.equal(_bits(g1[rev]), _bits(g0))

    # embedded among 400 other slates of random lengths: several items per CTA on every SM
    from allrank_b200.synth import make_slates
    fx, fy, _ = make_slates(400, S, F, seed=12, mean_len=S / 2, std_len=S / 3)
    fw = torch.where(fy == -1, torch.zeros_like(fy), torch.randn(fy.shape, generator=torch.Generator().manual_seed(13)))
    at = 157
    ex = torch.cat([fx[:at], x, fx[at:]])
    ey = torch.cat([fy[:at], y, fy[at:]])
    ew = torch.cat([fw[:at], w, fw[at:]])
    s2, g2 = _run(model, ex, ey, ew)
    assert torch.equal(_bits(s2[at:at + n]), _bits(s0))
    assert torch.equal(_bits(g2[at:at + n]), _bits(g0))
