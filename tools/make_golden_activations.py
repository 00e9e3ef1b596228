"""Golden vectors of models whose FC activation or output activation is one of the twelve classes beyond None / ReLU /
Tanh / Sigmoid, built by the UNMODIFIED reference's make_model (allrank/models/model.py, which instantiates
torch.nn.modules.activation classes by name) -> tests/golden/scorer_activations.npz.  Run where an allRank source tree
is available ($ALLRANK_REFERENCE):

    PYTHONDONTWRITEBYTECODE=1 python tools/make_golden_activations.py

Each case: seeded initialisation (torch.manual_seed before make_model), every 1-D parameter shifted by 0.1 N(0, 1)
from a second seed, eval mode, seeded slates (allrank_b200.synth).  Stored: the model section and feature count,
checksums of every parameter (they pin the initialisation the tests rebuild), the inputs (once per feature count), the scores, the weight of
the score sum that is differentiated, and every parameter gradient at up to 1024 sampled positions plus its norm.  The
tests read only the committed file.
"""
import json
import os
import sys

os.environ["CUDA_VISIBLE_DEVICES"] = ""       # the reference's get_torch_device() would pick cuda:0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle", "_stubs"), os.environ["ALLRANK_REFERENCE"], ROOT]
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402
import torch  # noqa: E402

from allrank.config import TransformerConfig  # noqa: E402
from allrank.models.model import make_model as ref_make_model  # noqa: E402
from allrank_b200.synth import make_slates  # noqa: E402

B, S = 3, 120
ACTS = ["LeakyReLU", "ELU", "CELU", "SELU", "Softplus", "Softsign", "Hardtanh", "ReLU6", "Hardsigmoid", "LogSigmoid",
        "Hardshrink", "Softshrink"]
# name: (n_features, sizes, activation, d_output, output_activation, transformer (N, h, d_ff) or None)
CASES = {}
for a in ACTS:
    CASES["fc_" + a] = (46, [50, 30], a, 1, None, None)       # the FC activation of an MLP with odd widths
for a in ACTS:
    CASES["out_" + a] = (46, [50, 30], "ReLU", 1, a, None)    # the output activation
for a in ["Softplus", "SELU", "Hardtanh"]:
    CASES["enc_" + a] = (46, [64], a, 1, None, (2, 4, 128))   # in front of a 2-layer encoder
CASES["d4_Hardsigmoid"] = (46, [64], "ELU", 4, "Hardsigmoid", (1, 4, 128))
GRAD_SAMPLES = 256


def grad_sample_index(numel):
    if numel <= GRAD_SAMPLES:
        return torch.arange(numel)
    return torch.linspace(0, numel - 1, GRAD_SAMPLES).long()


def model_section(sizes, act, d_output, out_act, enc):
    tr = None if enc is None else {"N": enc[0], "d_ff": enc[2], "h": enc[1], "positional_encoding": None,
                                   "dropout": 0.1}
    return {"fc_model": {"sizes": list(sizes), "input_norm": False, "activation": act, "dropout": 0.1},
            "transformer": tr, "post_model": {"d_output": d_output, "output_activation": out_act}}


def main():
    blob = {}
    for name, (F, sizes, act, d_output, out_act, enc) in CASES.items():
        m = model_section(sizes, act, d_output, out_act, enc)
        x, y, _ = make_slates(B, S, n_features=F, seed=51, mean_len=75, std_len=30)
        mask = y == -1
        tr = m["transformer"]
        torch.manual_seed(87)
        # (copies: the reference's FCModel inserts the input width into the list it is given)
        model = ref_make_model(fc_model=dict(m["fc_model"], sizes=list(sizes)), post_model=dict(m["post_model"]),
                               n_features=F,
                               transformer=None if tr is None else TransformerConfig(
                                   N=tr["N"], d_ff=tr["d_ff"], h=tr["h"], dropout=tr["dropout"],
                                   positional_encoding=None))
        g = torch.Generator().manual_seed(88)
        with torch.no_grad():
            for _, p in model.named_parameters():
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.eval()
        for k, v in model.state_dict().items():
            blob[name + ":c:" + k] = np.array([v.double().sum().item(), v.double().abs().sum().item()])
        out = model(x, mask, None)
        w = torch.randn(out.shape, generator=torch.Generator().manual_seed(89))
        w = w * (~mask).float().reshape(mask.shape + (1,) * (out.dim() - 2))
        (out * w).sum().backward()
        blob[name + ":model"] = np.array(json.dumps(m))
        blob[name + ":F"] = np.array(F)
        blob[f"x{F}"], blob[f"y{F}"] = x.numpy(), y.numpy()
        blob[name + ":scores"] = out.detach().numpy()
        blob[name + ":w"] = w.numpy()
        for k, p in model.named_parameters():
            blob[name + ":g:" + k] = p.grad.flatten()[grad_sample_index(p.numel())].numpy()
            blob[name + ":n:" + k] = np.array(p.grad.norm().item())
        print(name, tuple(out.shape), sum(p.numel() for p in model.parameters()), "parameters")
    blob["names"] = np.array(list(CASES))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "scorer_activations.npz"), **blob)


if __name__ == "__main__":
    main()
