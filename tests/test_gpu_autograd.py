"""Gradients with respect to the input features and the encoder output (LTRModel.prepare_for_output) of the CUDA
scorer: arb_scorer_encode and arb_scorer_backward_ex (include/allrank_b200.h).

Parity with the unmodified reference comes from tests/golden/scorer_autograd.npz (tests/test_oracle_autograd_golden.py
pins the oracle to the same file); the other configurations compare with the TF32 / bf16 emulation of the same maths
(oracle/tf32_emulation.py), under dropout with the kernels' masks regenerated on the host."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scorer_autograd.npz")
CASES = ["dout4_sigmoid", "fc2_tanh_norm", "mlp", "pe_learned", "tf_noact"]


def _fro(a, r):
    a, r = np.asarray(a, np.float64), np.asarray(r, np.float64)
    return np.linalg.norm(a - r) / max(np.linalg.norm(r), 1e-30)


def _pack(on):
    from allrank_b200 import _lib
    _lib.lib().arb_set_pack_rows(on)


def _restore_pack():
    from allrank_b200 import _lib
    _lib.lib().arb_set_pack_rows(_lib.default_pack_rows())


def _launches():
    from allrank_b200 import _lib
    torch.cuda.synchronize()
    return int(_lib.lib().arb_launch_count())


def _golden_model(c):
    from allrank_b200.model import make_model
    F, N, h, dff, dout, B, S, norm, *sizes = (int(v) for v in c["meta"])
    act = None if str(c["act"]) == "None" else str(c["act"])
    out_act = None if str(c["out_act"]) == "None" else str(c["out_act"])
    pe = str(c["pe"])
    pcfg = {"strategy": pe.split(":")[0], "max_indices": int(pe.split(":")[1])} if pe else None
    tcfg = {"N": N, "d_ff": dff, "h": h, "positional_encoding": pcfg, "dropout": 0.0} if N else None
    m = make_model(fc_model={"sizes": sizes, "input_norm": bool(norm), "activation": act, "dropout": 0.0},
                   transformer=tcfg, post_model={"d_output": dout, "output_activation": out_act}, n_features=F)
    m.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in c.items() if k.startswith("p:")})
    return m.cuda().eval(), N, h, act, out_act


def _case(name):
    z = np.load(GOLDEN)
    return {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}


def _emulated(sd, x, mask, N, h, out_act, fc_act, hidden=False, **kw):
    """oracle.tf32_emulation.scorer_forward; hidden=True: the encoder output, read through an identity head (the
    emulation's head is an exact fp32 elementwise product and sum)."""
    from oracle.tf32_emulation import scorer_forward
    if hidden:
        d = sd["output_layer.w_1.weight"].shape[1]
        sd = dict(sd)
        sd["output_layer.w_1.weight"] = torch.eye(d)
        sd["output_layer.w_1.bias"] = torch.zeros(d)
        out_act = None
    return scorer_forward(sd, x, mask, N, h, out_act, "rna", fc_act=fc_act, **kw)


@pytest.mark.parametrize("pack", [0, 1])
@pytest.mark.parametrize("name", CASES)
def test_input_and_encoder_gradients_match_the_reference(name, pack):
    c = _case(name)
    model, N, h, act, out_act = _golden_model(c)
    x0 = torch.from_numpy(c["x"]).cuda()
    mask = torch.from_numpy(c["mask"]).cuda()
    idx = torch.from_numpy(c["idx"]).cuda() if str(c["pe"]) else None
    real = (~mask).float()
    w = torch.from_numpy(c["w"]).cuda()
    wh = torch.from_numpy(c["wh"]).cuda()
    sfx = "v" if pack else ""                     # packed rows: the sets with padded items' weights zeroed
    if pack:
        w = w * (real if w.dim() == 2 else real[..., None])
        wh = wh * real[..., None]
    _pack(pack)
    try:
        x = x0.clone().requires_grad_(True)
        (model(x, mask, idx) * w).sum().backward()
        assert _fro(x.grad.cpu(), c["xg" + sfx]) <= 5e-2, ("x.grad", _fro(x.grad.cpu(), c["xg" + sfx]))
        model.zero_grad(set_to_none=True)
        x = x0.clone().requires_grad_(True)
        hid = model.prepare_for_output(x, mask, idx)
        ref_h = torch.from_numpy(c["hidden"])
        sel = torch.ones_like(mask.cpu()) if not pack else ~mask.cpu()
        assert (hid.detach().cpu() - ref_h)[sel].abs().max().item() <= 5e-3
        (hid * wh).sum().backward()
        tag = "h" + sfx
        assert _fro(x.grad.cpu(), c[tag + "xg"]) <= 5e-2, ("hidden x.grad", _fro(x.grad.cpu(), c[tag + "xg"]))
        for k, p in model.named_parameters():
            if tag + "g:" + k in c:
                # (the FFN's W1 and b1: a unit whose TF32 pre-activation lands on the other side of its ReLU moves a whole
                # row of the gradient -- 6 % with the learned positional encoding, whose sqrt(d) scaling enlarges it)
                # (the key bias gradient is analytically zero -- softmax ignores a per-query constant: rounding only)
                e = _fro(p.grad.cpu(), c[tag + "g:" + k])
                tiny = np.linalg.norm(c[tag + "g:" + k]) < 1e-4
                assert tiny or e <= (1e-1 if ".feed_forward.w_1." in k else 5e-2), (k, e)
        if not str(c["pe"]):            # and within 1 % of the TF32 emulation of the same maths
            sd = {k: v.detach().cpu().clone().requires_grad_(True) for k, v in model.state_dict().items()}
            xe = x0.cpu().clone().requires_grad_(True)
            (_emulated(sd, xe, mask.cpu(), N, h, out_act, act, hidden=True).view_as(hid) * wh.cpu()).sum().backward()
            assert _fro(x.grad.cpu(), xe.grad) <= 1e-2, ("emulation", _fro(x.grad.cpu(), xe.grad))
    finally:
        _restore_pack()


@pytest.mark.parametrize("name", ["tf_noact", "fc2_tanh_norm"])
def test_packed_rows_equal_dense_rows_for_real_items(name):
    c = _case(name)
    model, *_ = _golden_model(c)
    x0 = torch.from_numpy(c["x"]).cuda()
    mask = torch.from_numpy(c["mask"]).cuda()
    real = ~mask
    w = torch.from_numpy(c["w"]).cuda() * real.float()
    wh = torch.from_numpy(c["wh"]).cuda() * real[..., None].float()
    out = {}
    for pack in (0, 1):
        _pack(pack)
        try:
            x = x0.clone().requires_grad_(True)
            (model(x, mask, None) * w).sum().backward()
            xs = x.grad.clone()
            x = x0.clone().requires_grad_(True)
            hid = model.prepare_for_output(x, mask, None)
            (hid * wh).sum().backward()
            out[pack] = (xs, hid.detach().clone(), x.grad.clone())
        finally:
            _restore_pack()
    for i, what in enumerate(("x.grad (scores)", "hidden", "x.grad (hidden)")):
        a, b = out[1][i][real], out[0][i][real]
        diff = (a - b).abs().max().item()
        print(name, what, "packed vs dense max |diff| on real items:", diff, "bit-identical:", torch.equal(a, b))
        assert diff <= 1e-6 * max(1.0, b.abs().max().item()), (what, diff)


def _model(F=136, sizes=(64,), N=2, h=2, dff=128, p=0.0, p_fc=0.0, act=None, norm=False, dtype="tf32", seed=3):
    from allrank_b200.model import make_model
    torch.manual_seed(seed)
    tcfg = {"N": N, "d_ff": dff, "h": h, "positional_encoding": None, "dropout": p} if N else None
    m = make_model(fc_model={"sizes": list(sizes), "input_norm": norm, "activation": act, "dropout": p_fc},
                   transformer=tcfg, post_model={"d_output": 1, "output_activation": None}, n_features=F,
                   compute_dtype=dtype)
    gen = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for q in m.parameters():
            if q.dim() == 1:
                q.add_(0.1 * torch.randn(q.shape, generator=gen))
    return m.cuda()


def _slates(B, S, F, seed=5):
    from allrank_b200.synth import make_slates
    x, y, _ = make_slates(B, S, n_features=F, seed=seed, mean_len=0.7 * S, std_len=0.2 * S)
    return x.cuda(), (y == -1).cuda()


def test_dropout_uses_the_forward_masks_for_x_and_hidden_gradients():
    from tests.dropout_masks import scorer_masks
    F, d, N, h, dff, B, S, p, p_fc = 136, 64, 2, 2, 128, 5, 48, 0.2, 0.1
    model = _model(F, (d,), N, h, dff, p=p, p_fc=p_fc).train()
    x0, mask = _slates(B, S, F)
    w, wh = torch.randn(B, S).cuda(), torch.randn(B, S, d).cuda()
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    for hidden in (False, True):
        torch.manual_seed(21)
        call_seed = int(torch.randint(0, 2 ** 62, (1,)).item())      # what LTRModel._draw_seed draws
        torch.manual_seed(21)
        x = x0.clone().requires_grad_(True)
        out = model.prepare_for_output(x, mask) if hidden else model(x, mask)
        (out * (wh if hidden else w)).sum().backward()
        drop = scorer_masks(call_seed, B, S, [d], N, h, dff, p, p_fc)
        xe = x0.cpu().clone().requires_grad_(True)
        ref = _emulated(sd, xe, mask.cpu(), N, h, None, None, hidden=hidden, drop=drop)
        (ref.view_as(out) * (wh if hidden else w).cpu()).sum().backward()
        e = _fro(x.grad.cpu(), xe.grad)
        print("dropout, hidden =", hidden, ": x.grad rel err", e)
        assert e <= 5e-2, (hidden, e)


def test_bf16_x_gradient_matches_the_bf16_emulation():
    F, d, N, h, dff, B, S = 136, 128, 2, 4, 256, 5, 120
    model = _model(F, (d,), N, h, dff, dtype="bf16").eval()
    x0, mask = _slates(B, S, F)
    w = torch.randn(B, S).cuda() * (~mask).float()
    wh = torch.randn(B, S, d).cuda() * (~mask)[..., None].float()
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    for hidden in (False, True):
        x = x0.clone().requires_grad_(True)
        out = model.prepare_for_output(x, mask) if hidden else model(x, mask)
        (out * (wh if hidden else w)).sum().backward()
        xe = x0.cpu().clone().requires_grad_(True)
        ref = _emulated(sd, xe, mask.cpu(), N, h, None, None, hidden=hidden, bf16=True)
        (ref.view_as(out) * (wh if hidden else w).cpu()).sum().backward()
        e = _fro(x.grad.cpu(), xe.grad)
        print("bf16, hidden =", hidden, ": x.grad rel err", e)
        assert e <= 3e-2, (hidden, e)


@pytest.mark.parametrize("shape", [(136, 128, 2, 256, 4, 48), (136, 64, 2, 128, 3, 300)])
def test_unfused_attention_shapes(shape):
    """Head width 64 (unfused attention backward) and a slate above 256 items (unfused attention), dense rows."""
    F, d, h, dff, B, S = shape
    model = _model(F, (d,), 2, h, dff).eval()
    x0, mask = _slates(B, S, F)
    wh = torch.randn(B, S, d).cuda()
    x = x0.clone().requires_grad_(True)
    (model.prepare_for_output(x, mask) * wh).sum().backward()
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    xe = x0.cpu().clone().requires_grad_(True)
    (_emulated(sd, xe, mask.cpu(), 2, h, None, None, hidden=True).view_as(wh) * wh.cpu()).sum().backward()
    e = _fro(x.grad.cpu(), xe.grad)
    print("unfused", shape, ": x.grad rel err", e)
    assert e <= 1e-2, e


def test_unpadded_feature_count_and_float64_non_contiguous_x():
    F, B, S = 22, 4, 40
    model = _model(F, (32, 64), 1, 2, 128, act="Tanh").eval()
    base, mask = _slates(B, S, F)
    x = base.double().transpose(1, 2).contiguous().transpose(1, 2).requires_grad_(True)   # [B,S,F], non-contiguous
    assert not x.is_contiguous()
    w = torch.randn(B, S).cuda() * (~mask).float()       # (packed rows: padded items' own scores are constant)
    (model(x, mask) * w).sum().backward()
    assert x.grad.shape == x.shape and x.grad.dtype == torch.float64
    x32 = base.clone().requires_grad_(True)              # the same values as contiguous fp32: the same launches
    (model(x32, mask) * w).sum().backward()
    assert torch.equal(x.grad, x32.grad.double())
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    xe = base.cpu().clone().requires_grad_(True)
    (_emulated(sd, xe, mask.cpu(), 1, 2, None, "Tanh") * w.cpu()).sum().backward()
    e = _fro(x.grad.cpu(), xe.grad)
    print("F = 22: x.grad rel err", e)
    assert e <= 1e-2, e


@pytest.mark.parametrize("pack,norm", [(1, False), (0, False), (1, True), (0, True)])
def test_no_interference_frozen_parameters_and_reproducibility(pack, norm):
    F, B, S = 136, 24, 120
    model = _model(F, (64,), 2, 2, 128, norm=norm).train()
    x0, mask = _slates(B, S, F)
    w = torch.randn(B, S).cuda() * (~mask).float()
    _pack(pack)
    try:
        def step(x_grad):
            model.zero_grad(set_to_none=True)
            x = x0.clone().requires_grad_(x_grad)
            s = model(x, mask)
            n0 = _launches()
            (s * w).sum().backward()
            return s.detach().clone(), model.flat_gradients.clone(), x.grad, _launches() - n0
        s1, g1, _, n1 = step(False)
        s2, g2, dx, n2 = step(True)
        assert torch.equal(s1, s2) and torch.equal(g1, g2)
        extra = (0 if norm else 1) + (1 if pack else 0)            # the dX product (input_norm: its LayerNorm already
        assert n2 - n1 == extra, (n1, n2)                           # computed it) and the scatter of packed rows
        _, _, dx2, _ = step(True)
        assert torch.equal(dx, dx2)                                 # reproducible
        # frozen parameters: x.grad alone; nothing touches the flat gradient buffer or any .grad
        model.requires_grad_(False)
        pattern = torch.arange(model.flat_gradients.numel(), dtype=torch.float32, device="cuda")
        model.flat_gradients.copy_(pattern)
        grads_before = {k: p.grad for k, p in model.named_parameters()}
        x = x0.clone().requires_grad_(True)
        s = model(x, mask)
        n0 = _launches()
        (s * w).sum().backward()
        n3 = _launches() - n0
        assert torch.equal(x.grad, dx)
        assert torch.equal(model.flat_gradients, pattern)
        assert all(p.grad is grads_before[k] for k, p in model.named_parameters())
        assert n3 < n1, (n3, n1)
        print("pack", pack, "norm", norm, "launches: full", n1, "with dX", n2, "frozen", n3)
    finally:
        model.requires_grad_(True)
        _restore_pack()


def test_encoder_output_feeds_the_head_and_follows_grad_mode():
    F, d, B, S = 136, 64, 6, 60
    model = _model(F, (d,), 2, 2, 128).eval()
    x0, mask = _slates(B, S, F)
    with torch.no_grad():
        hid = model.prepare_for_output(x0, mask)
        s = model(x0, mask)
    assert hid.grad_fn is None and not hid.requires_grad
    head = model.output_layer.w_1
    s_torch = torch.nn.functional.linear(hid, head.weight, head.bias).squeeze(-1)
    real = ~mask
    assert torch.allclose(s_torch[real], s[real], rtol=1e-3, atol=1e-3)
    x = x0.clone().requires_grad_(True)
    hid = model.prepare_for_output(x, mask)
    (g,) = torch.autograd.grad((hid * hid).sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()
