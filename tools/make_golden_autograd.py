"""Generate tests/golden/scorer_autograd.npz from the UNMODIFIED reference (run where an allRank source tree is
available; same set-up as oracle/make_golden.py, whose import hides CUDA and puts the reference on the path).

    PYTHONDONTWRITEBYTECODE=1 python tools/make_golden_autograd.py

Per case: x, mask and the reference's gradients with respect to x and the parameters through both public outputs --
the scores (`model(x, mask, indices)`) and the encoder output (`model.prepare_for_output(x, mask, indices)`) -- each
once with random weights on every item and once with the weights of padded items zeroed ("v" sets: what a loss that
masks padded items sends back, and what the packed-row layout of allrank_b200 reproduces).
"""
import os
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import make_golden as mg  # noqa: E402  (CUDA hidden, reference importable)

import numpy as np  # noqa: E402
import torch  # noqa: E402

# name: (F, fc sizes, fc activation, input_norm, N, h, d_ff, d_output, output activation, positional, B, S)
CASES = {
    "tf_noact": (20, [32], None, False, 2, 2, 64, 1, None, None, 3, 24),
    "fc2_tanh_norm": (16, [48, 32], "Tanh", True, 1, 2, 64, 1, None, None, 3, 20),
    "mlp": (20, [48, 32], "ReLU", False, 0, 1, 4, 1, None, None, 3, 20),
    "dout4_sigmoid": (20, [32], None, False, 1, 2, 64, 4, "Sigmoid", None, 3, 20),
    "pe_learned": (20, [32], None, False, 2, 2, 64, 1, None, ("learned", 15), 3, 20),
}


def _grads(model, x, out, w):
    model.zero_grad()
    x.grad = None
    (out * w).sum().backward()
    return x.grad.numpy().copy(), {k: p.grad.numpy().copy() for k, p in model.named_parameters() if p.grad is not None}


def gen_scorer_autograd():
    blob = {}
    for name, (F, sizes, act, norm, N, h, dff, dout, out_act, pe, B, S) in CASES.items():
        torch.manual_seed(13)
        tcfg = None
        if N > 0:
            pcfg = None if pe is None else mg.PositionalEncoding(strategy=pe[0], max_indices=pe[1])
            tcfg = mg.TransformerConfig(N=N, d_ff=dff, h=h, positional_encoding=pcfg, dropout=0.0)
        model = mg.ref_make_model(
            fc_model={"sizes": list(sizes), "input_norm": norm, "activation": act, "dropout": 0.0},
            transformer=tcfg, post_model={"d_output": dout, "output_activation": out_act}, n_features=F)
        g = torch.Generator().manual_seed(17)
        with torch.no_grad():                         # perturb gains / biases so that the gradients exercise them
            for p in model.parameters():
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.eval()
        x, y, idx = mg.make_slates(B, S, n_features=F, seed=41, mean_len=0.6 * S, std_len=0.3 * S)
        if pe is not None:
            idx = torch.where(idx >= 0, torch.stack([torch.randperm(S, generator=g) for _ in range(B)]), idx)
        mask = y == -1
        real = (~mask).float()
        x = x.clone().requires_grad_(True)
        pre = f"{name}/"
        blob[pre + "x"] = x.detach().numpy()
        blob[pre + "mask"] = mask.numpy()
        blob[pre + "idx"] = idx.numpy()
        blob[pre + "meta"] = np.array([F, N, h, dff, dout, B, S, 1 if norm else 0] + list(sizes))
        blob[pre + "act"] = np.array(str(act))
        blob[pre + "out_act"] = np.array(str(out_act))
        blob[pre + "pe"] = np.array("" if pe is None else f"{pe[0]}:{pe[1]}")
        for k, v in model.state_dict().items():
            blob[pre + "p:" + k] = v.numpy()
        scores = model(x, mask, idx)
        w = torch.randn(scores.shape, generator=g)
        wv = w * (real if dout == 1 else real[..., None])
        blob[pre + "scores"] = scores.detach().numpy()
        blob[pre + "w"] = w.numpy()
        blob[pre + "xg"], _ = _grads(model, x, model(x, mask, idx), w)
        blob[pre + "xgv"], _ = _grads(model, x, model(x, mask, idx), wv)
        hidden = model.prepare_for_output(x, mask, idx)
        wh = torch.randn(hidden.shape, generator=g)
        blob[pre + "hidden"] = hidden.detach().numpy()
        blob[pre + "wh"] = wh.numpy()
        for tag, weights in (("h", wh), ("hv", wh * real[..., None])):
            xg, pg = _grads(model, x, model.prepare_for_output(x, mask, idx), weights)
            blob[pre + tag + "xg"] = xg
            for k, v in pg.items():
                blob[pre + tag + "g:" + k] = v
        print("scorer_autograd", name, "hidden", tuple(hidden.shape))
    np.savez_compressed(os.path.join(mg.OUT, "scorer_autograd.npz"), **blob)


if __name__ == "__main__":
    torch.set_num_threads(4)
    gen_scorer_autograd()
