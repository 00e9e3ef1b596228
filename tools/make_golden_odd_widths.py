"""Golden vectors of models whose FC layer widths, d_model or d_ff are not multiples of 4, from the UNMODIFIED
reference's make_model (allrank/models/model.py) -> tests/golden/scorer_odd_widths.npz.  Run where an allRank source tree is available
($ALLRANK_REFERENCE, default /root/reference):

    PYTHONDONTWRITEBYTECODE=1 python tools/make_golden_odd_widths.py

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
sys.path[:0] = [os.path.join(ROOT, "oracle", "_stubs"), os.environ.get("ALLRANK_REFERENCE", "/root/reference"), ROOT]
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402
import torch  # noqa: E402

from allrank.config import TransformerConfig  # noqa: E402
from allrank.models.model import make_model as ref_make_model  # noqa: E402
from allrank_b200.synth import make_slates  # noqa: E402

B, S = 3, 240
# name: (n_features, sizes, activation, d_output, transformer (N, h, d_ff) or None)
CASES = {
    "f10s10": (10, [10], None, 1, None),                  # the model of the reference's tests/test_rank_slates.py
    "f46s10_6": (46, [10, 6], "ReLU", 1, None),
    "f46s50_30t": (46, [50, 30], "Tanh", 3, None),
    "f46s50_30s": (46, [50, 30], "Sigmoid", 1, None),
    "f46s46_64e": (46, [46, 64], "ReLU", 1, (1, 4, 128)),   # an FC hidden width of 46 in front of an encoder
    # encoders whose d_model / d_ff are not multiples of 4 (their heads are padded too)
    "d10h2": (46, [10], None, 1, (1, 2, 20)),
    "d46h2f30": (46, [46], "ReLU", 1, (2, 2, 30)),
    "d130h2": (46, [130], None, 1, (1, 2, 262)),
    "d6h3o3": (46, [6], None, 3, (1, 3, 14)),
}
GRAD_SAMPLES = 1024


def grad_sample_index(numel):
    if numel <= GRAD_SAMPLES:
        return torch.arange(numel)
    return torch.linspace(0, numel - 1, GRAD_SAMPLES).long()


def model_section(sizes, act, d_output, enc):
    tr = None if enc is None else {"N": enc[0], "d_ff": enc[2], "h": enc[1], "positional_encoding": None,
                                   "dropout": 0.1}
    return {"fc_model": {"sizes": list(sizes), "input_norm": False, "activation": act, "dropout": 0.1},
            "transformer": tr, "post_model": {"d_output": d_output, "output_activation": None}}


def main():
    blob = {}
    for name, (F, sizes, act, d_output, enc) in CASES.items():
        m = model_section(sizes, act, d_output, enc)
        x, y, _ = make_slates(B, S, n_features=F, seed=51, mean_len=150, std_len=60)
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
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "scorer_odd_widths.npz"), **blob)


if __name__ == "__main__":
    main()
