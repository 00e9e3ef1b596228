"""Golden vectors of models whose head width d_model / h is not a multiple of 4, from the UNMODIFIED reference's
make_model (allrank/models/model.py) -> tests/golden/scorer_odd_heads.npz.  Run where an allRank source tree is
available ($ALLRANK_REFERENCE, default /root/reference):

    PYTHONDONTWRITEBYTECODE=1 python tools/make_golden_odd_heads.py

Each case: seeded initialisation (torch.manual_seed before make_model), every 1-D parameter shifted by 0.1 N(0, 1)
from a second seed, eval mode, seeded slates (allrank_b200.synth).  Stored: the model section, checksums of every
parameter (they pin the initialisation the tests rebuild), the inputs, the scores, the weight of the score sum that is
differentiated, and every parameter gradient at up to 1024 sampled positions plus its norm.  The tests read only the
committed file.
"""
import json
import os
import sys

os.environ["CUDA_VISIBLE_DEVICES"] = ""       # the reference's get_torch_device() would pick cuda:0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle", "_stubs"), os.environ.get("ALLRANK_REFERENCE", "/root/reference"), ROOT]
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402
import torch  # noqa: E402

from allrank.config import TransformerConfig  # noqa: E402
from allrank.models.model import make_model as ref_make_model  # noqa: E402
from allrank_b200.synth import make_slates  # noqa: E402

F, B, S = 136, 3, 240
# name: (d_model, h, N, d_ff): heads of 18 columns (the shipped ordinal model's width with eight heads) and of 3
CASES = {"d144h8": (144, 8, 2, 576), "d96h32": (96, 32, 2, 384)}
GRAD_SAMPLES = 1024


def grad_sample_index(numel):
    if numel <= GRAD_SAMPLES:
        return torch.arange(numel)
    return torch.linspace(0, numel - 1, GRAD_SAMPLES).long()


def model_section(d, h, N, dff):
    return {"fc_model": {"sizes": [d], "input_norm": False, "activation": None, "dropout": 0.0},
            "transformer": {"N": N, "d_ff": dff, "h": h, "positional_encoding": None, "dropout": 0.1},
            "post_model": {"d_output": 1, "output_activation": None}}


def main():
    blob = {}
    x, y, _ = make_slates(B, S, n_features=F, seed=51, mean_len=150, std_len=60)
    mask = y == -1
    blob["x"], blob["y"] = x.numpy(), y.numpy()
    for name, (d, h, N, dff) in CASES.items():
        m = model_section(d, h, N, dff)
        tr = m["transformer"]
        torch.manual_seed(87)
        # (copies: the reference's FCModel inserts the input width into the list it is given)
        model = ref_make_model(fc_model=dict(m["fc_model"], sizes=list(m["fc_model"]["sizes"])),
                               post_model=dict(m["post_model"]), n_features=F,
                               transformer=TransformerConfig(N=tr["N"], d_ff=tr["d_ff"], h=tr["h"],
                                                             dropout=tr["dropout"], positional_encoding=None))
        g = torch.Generator().manual_seed(88)
        with torch.no_grad():
            for _, p in model.named_parameters():
                if p.dim() == 1:
                    p.add_(0.1 * torch.randn(p.shape, generator=g))
        model.eval()
        for k, v in model.state_dict().items():
            blob[name + ":c:" + k] = np.array([v.double().sum().item(), v.double().abs().sum().item()])
        out = model(x, mask, None)
        w = torch.randn(out.shape, generator=torch.Generator().manual_seed(89)) * (~mask).float()
        (out * w).sum().backward()
        blob[name + ":model"] = np.array(json.dumps(m))
        blob[name + ":scores"] = out.detach().numpy()
        blob[name + ":w"] = w.numpy()
        for k, p in model.named_parameters():
            blob[name + ":g:" + k] = p.grad.flatten()[grad_sample_index(p.numel())].numpy()
            blob[name + ":n:" + k] = np.array(p.grad.norm().item())
        print(name, tuple(out.shape), sum(p.numel() for p in model.parameters()), "parameters")
    blob["names"] = np.array(list(CASES))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "scorer_odd_heads.npz"), **blob)


if __name__ == "__main__":
    main()
