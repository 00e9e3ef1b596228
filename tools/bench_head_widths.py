"""Training steps of Transformer configurations whose heads are not 16 or 32 columns wide -- local_config (d 64, h 1:
width 64), contextaware ordinal (d 144, h 2: width 72, four outputs), neuralNDCG-paper approxNDCG (d 96, h 1: width
96) -- of a d = 256, h = 4 model (width 64), of two width-128 models (d 128, h 1 and d 256, h 2), of the
neuralNDCG-paper model widened to one head of 136, 192 or 256 columns, and of the neuralNDCG-paper model at d 64, 96
and 192 with eight heads (widths 8, 12 and 24), and models whose head width is not a multiple of 4 (padded heads,
DESIGN.md 4.15: d 144 / h 8, width 18; d 96 / h 32, width 3; d 200 / h 8, width 25) beside the nearest multiple-of-4
width at the same d_model (d 144 / h 9, width 16; d 96 / h 24, width 4; d 200 / h 10, width 20), each with its own
dropout and loss: the fused attention kernels
(attention mode 2) against the unfused sequence
(arb_set_attention_mode(0): [B, h, S, S] probabilities in HBM) where the latter exists (S <= 1536).

    python tools/bench_head_widths.py [--steps 5] [--warmup 2] [--runs 3] [--models a,b] [--json out.json]

Shapes: every model at B = 64 and B = 1024 slates of S = 240 items, and the models of width 96 and above and the
eight-head models at S = 1024, 2048, 4096 (B = 245760 / S slates, fewer where the unfused path would not fit in
memory), and the padded-head models and their comparisons at S = 1024 (B = 240).  --fused-only skips the unfused
arm.  Slate lengths ~ N(S/2, S/4) clamped to [1, S].  Step time is the host clock around `steps` training steps
that end in a device synchronise, per run; the modes alternate run by run.  Peak memory is torch.cuda.max_memory_allocated over a run.  The attention kernels' times
come from torch.profiler in a separate run per shape.  The GPU's name and power limit are printed with the numbers."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_long_slates import gpu_info, kernel_times, set_mode, timed  # noqa: E402

# the `model` and `loss` sections of the shipped configurations (d_256_h4: a wider model at the same width as local_config)
MODELS = {
    "local_config": (dict(fc_model={"sizes": [64], "input_norm": False, "activation": None, "dropout": 0.0},
                          transformer={"N": 1, "d_ff": 64, "h": 1, "positional_encoding": None, "dropout": 0.0},
                          post_model={"output_activation": "Sigmoid", "d_output": 4}), ("ordinal", {"n": 4})),
    "ordinal": (dict(fc_model={"sizes": [144], "input_norm": False, "activation": None, "dropout": 0.0},
                     transformer={"N": 4, "d_ff": 512, "h": 2, "positional_encoding": None, "dropout": 0.4},
                     post_model={"output_activation": "Sigmoid", "d_output": 4}), ("ordinal", {"n": 4})),
    "approxndcg": (dict(fc_model={"sizes": [96], "input_norm": False, "activation": None, "dropout": 0.0},
                        transformer={"N": 2, "d_ff": 384, "h": 1, "positional_encoding": None, "dropout": 0.1},
                        post_model={"output_activation": None, "d_output": 1}), ("approxNDCGLoss", {"alpha": 1.0})),
    "d256_h4": (dict(fc_model={"sizes": [256], "input_norm": False, "activation": None, "dropout": 0.0},
                     transformer={"N": 2, "d_ff": 1024, "h": 4, "positional_encoding": None, "dropout": 0.1},
                     post_model={"output_activation": None, "d_output": 1}), ("approxNDCGLoss", {"alpha": 1.0})),
    "d128_h1": (dict(fc_model={"sizes": [128], "input_norm": False, "activation": None, "dropout": 0.0},
                     transformer={"N": 2, "d_ff": 512, "h": 1, "positional_encoding": None, "dropout": 0.1},
                     post_model={"output_activation": None, "d_output": 1}), ("approxNDCGLoss", {"alpha": 1.0})),
    "d256_h2": (dict(fc_model={"sizes": [256], "input_norm": False, "activation": None, "dropout": 0.0},
                     transformer={"N": 2, "d_ff": 1024, "h": 2, "positional_encoding": None, "dropout": 0.1},
                     post_model={"output_activation": None, "d_output": 1}), ("approxNDCGLoss", {"alpha": 1.0})),
}
# the neuralNDCG-paper model (approxndcg) widened to one head of 136 (the MSLR feature count), 192 and 256 columns
for _w in (136, 192, 256):
    MODELS[f"d{_w}_h1"] = (dict(fc_model={"sizes": [_w], "input_norm": False, "activation": None, "dropout": 0.0},
                                transformer={"N": 2, "d_ff": 384, "h": 1, "positional_encoding": None, "dropout": 0.1},
                                post_model={"output_activation": None, "d_output": 1}), ("approxNDCGLoss", {"alpha": 1.0}))
# ... and with eight heads of 8 (d 64, the local_config width), 12 (d 96, the paper's width) and 24 (d 192) columns
for _d in (64, 96, 192):
    MODELS[f"d{_d}_h8"] = (dict(fc_model={"sizes": [_d], "input_norm": False, "activation": None, "dropout": 0.0},
                                transformer={"N": 2, "d_ff": 384, "h": 8, "positional_encoding": None, "dropout": 0.1},
                                post_model={"output_activation": None, "d_output": 1}), ("approxNDCGLoss", {"alpha": 1.0}))
# ... and padded heads (widths 18, 3, 25) next to the nearest multiple-of-4 width at the same d_model (16, 4, 20)
for _d, _h in ((144, 8), (144, 9), (96, 32), (96, 24), (200, 8), (200, 10)):
    MODELS[f"d{_d}_h{_h}"] = (dict(fc_model={"sizes": [_d], "input_norm": False, "activation": None, "dropout": 0.0},
                                   transformer={"N": 2, "d_ff": 384, "h": _h, "positional_encoding": None,
                                                "dropout": 0.1},
                                   post_model={"output_activation": None, "d_output": 1}),
                              ("approxNDCGLoss", {"alpha": 1.0}))
ODD = ("d144_h8", "d144_h9", "d96_h32", "d96_h24", "d200_h8", "d200_h10")
SHAPES = [(name, B, 240) for name in MODELS for B in (64, 1024)] + [
    (name, 245760 // S, S) for name in ("approxndcg", "d128_h1", "d256_h2", "d136_h1", "d192_h1", "d256_h1",
                                        "d64_h8", "d96_h8", "d192_h8")
    for S in (1024, 2048, 4096)] + [(name, 240, 1024) for name in ODD]


def make_batch(B, S, seed=7):
    from allrank_b200.synth import make_slates
    x, y, _ = make_slates(B, S, n_features=136, seed=seed, mean_len=S / 2, std_len=S / 4)
    return x.cuda(), y.cuda()


def make_step(name):
    from allrank_b200 import losses
    from allrank_b200.model import make_model
    from allrank_b200.optim import FlatAdam
    cfg, (loss_name, loss_args) = MODELS[name]
    torch.manual_seed(0)
    model = make_model(**cfg, n_features=136).cuda().train()
    opt = FlatAdam(model, lr=1e-3)
    loss_fn = getattr(losses, loss_name)

    def step(x, y):
        loss = loss_fn(model(x, y == -1, None), y, **loss_args)
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss
    return step


def fits_unfused(name, B, S):
    """The unfused path's [B, h, S, S] buffers: one per layer in the workspace plus two in the backward scratch."""
    t = MODELS[name][0]["transformer"]
    return S <= 1536 and (t["N"] + 2) * B * t["h"] * S * S * 4 < 0.7 * torch.cuda.get_device_properties(0).total_memory


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--models", default=None, help="comma-separated subset of the models (default: all)")
    ap.add_argument("--json", default=None)
    ap.add_argument("--fused-only", action="store_true", help="skip the unfused arm")
    args = ap.parse_args()
    only = set(args.models.split(",")) if args.models else set(MODELS)
    assert only <= set(MODELS), f"unknown model in {sorted(only - set(MODELS))}"
    assert torch.cuda.is_available(), "needs a CUDA device"
    name_gpu, power = gpu_info()
    print(f"GPU: {name_gpu}; power limit, max SM clock: {power}", flush=True)
    rows = []
    for name, B, S in SHAPES:
        if name not in only:
            continue
        step = make_step(name)
        modes = (2, 0) if fits_unfused(name, B, S) and not args.fused_only else (2,)
        x, y = make_batch(B, S)
        res = {m: [] for m in modes}
        for _ in range(args.runs):
            for m in modes:
                set_mode(m)
                res[m].append(timed(step, x, y, args.steps, args.warmup))
        kt = {}
        for m in modes:
            set_mode(m)
            kt[m] = kernel_times(step, x, y)
        set_mode(2)
        for m in modes:
            ms = [r[0] for r in res[m]]
            mem = max(r[1] for r in res[m])
            row = dict(model=name, B=B, S=S, path="fused" if m == 2 else "unfused", step_ms=ms, peak_gib=mem,
                       attention_kernel_ms=kt[m])
            rows.append(row)
            print(f"{name:12s} B={B:5d} S={S:5d} {row['path']:7s} step ms " + " / ".join(f"{v:8.2f}" for v in ms) +
                  f"   peak {mem:6.2f} GiB   kernels " + ", ".join(f"{k} {v:.2f}" for k, v in sorted(kt[m].items())),
                  flush=True)
        del x, y, step
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(gpu=name_gpu, power=power, steps=args.steps, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
