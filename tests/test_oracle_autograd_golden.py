"""The oracle scorer (oracle/scorer_ref.py, eager autograd) against the unmodified reference's gradients with respect to
the input features and its encoder output (tests/golden/scorer_autograd.npz, tools/make_golden_autograd.py): this
anchors the oracle that the GPU tests of x.grad and prepare_for_output compare with."""
import os

import numpy as np
import pytest
import torch

from tests.test_oracle_golden import zero_by_symmetry

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scorer_autograd.npz")


def _cases(z):
    return sorted({k.split("/")[0] for k in z.files})


def load_case(z, name):
    """(oracle model loaded with the case's parameters, x, mask, indices, blob of the case)."""
    from oracle.scorer_ref import make_ref_model
    c = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
    F, N, h, dff, dout, B, S, norm, *sizes = (int(v) for v in c["meta"])
    act = None if str(c["act"]) == "None" else str(c["act"])
    out_act = None if str(c["out_act"]) == "None" else str(c["out_act"])
    pe = str(c["pe"])
    positional = (pe.split(":")[0], int(pe.split(":")[1])) if pe else None
    model = make_ref_model(F, sizes, N, h, dff, d_output=dout, output_activation=out_act, fc_activation=act,
                           positional=positional, input_norm=bool(norm))
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in c.items() if k.startswith("p:")})
    return model.eval(), torch.from_numpy(c["x"]), torch.from_numpy(c["mask"]), torch.from_numpy(c["idx"]), c


def _close(a, b, name):
    scale = max(1e-6, float(np.abs(b).max()))
    err = float(np.abs(a - b).max())
    assert err <= 1e-5 * scale + 1e-7, (name, err, scale)


@pytest.mark.parametrize("name", _cases(np.load(GOLDEN)))
def test_oracle_reproduces_the_reference_input_and_encoder_gradients(name):
    model, x, mask, idx, c = load_case(np.load(GOLDEN), name)
    real = (~mask).float()
    w = torch.from_numpy(c["w"])
    wv = w * (real if w.dim() == 2 else real[..., None])
    for tag, weights in (("xg", w), ("xgv", wv)):
        xr = x.clone().requires_grad_(True)
        (model(xr, mask, idx) * weights).sum().backward()
        _close(xr.grad.numpy(), c[tag], tag)
    wh = torch.from_numpy(c["wh"])
    xr = x.clone().requires_grad_(True)
    hidden = model.prepare_for_output(xr, mask, idx)
    _close(hidden.detach().numpy(), c["hidden"], "hidden")
    for tag, weights in (("h", wh), ("hv", wh * real[..., None])):
        model.zero_grad()
        xr = x.clone().requires_grad_(True)
        (model.prepare_for_output(xr, mask, idx) * weights).sum().backward()
        _close(xr.grad.numpy(), c[tag + "xg"], tag + "xg")
        for k, p in model.named_parameters():
            if tag + "g:" + k in c and zero_by_symmetry(k):
                level = 1e-5 * np.abs(c[tag + "g:" + k[:-len("bias")] + "weight"]).max()
                assert np.abs(p.grad.numpy()).max() <= level and np.abs(c[tag + "g:" + k]).max() <= level, k
            elif tag + "g:" + k in c:
                _close(p.grad.numpy(), c[tag + "g:" + k], tag + "g:" + k)
            else:
                assert p.grad is None, k           # the head takes no part in the encoder output
