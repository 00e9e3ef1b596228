"""What padding a layer to a multiple of 4 columns costs (DESIGN.md 4.16): a training step (forward, approxNDCG loss,
backward, FlatAdam) of a model with widths that are not multiples of 4 against the same model at the next multiples of
4, at B = 1024 slates of S = 240 items and 136 features, alternating the two models round by round.  FC-only pairs
(fc_model.sizes) and encoder pairs (N = 2, h = 2, d_ff = 2 d: d_model 130 against 128).

    python tools/bench_fc_widths.py [--rounds 7] [--steps 20] [--out DIR]

Prints one JSON line per pair (median and spread of the per-round step times) and the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PAIRS = [([50, 30], [52, 32]), ([10], [12]), ([100, 50], [100, 52])]
ENC_PAIRS = [(130, 128)]      # d_model with h = 2: heads of 65 (padded to 68) against 64


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or "unknown"


def make(sizes, F, enc=False):
    from allrank_b200.model import make_model
    torch.manual_seed(0)
    tr = {"N": 2, "d_ff": 2 * sizes[-1], "h": 2, "positional_encoding": None, "dropout": 0.0} if enc else None
    return make_model({"sizes": sizes, "input_norm": False, "activation": "ReLU", "dropout": 0.0}, tr,
                      {"d_output": 1, "output_activation": None}, F).cuda().train()


def step_time(model, opt, x, y, steps):
    from allrank_b200 import losses
    mask = y == -1
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        loss = losses.approxNDCGLoss(model(x, mask, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--slate", type=int, default=240)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fc_widths: no GPU")
    from allrank_b200.optim import FlatAdam
    from allrank_b200.synth import make_slates
    F = 136
    x, y, _ = make_slates(a.batch, a.slate, n_features=F, seed=3, mean_len=int(0.75 * a.slate), std_len=a.slate // 5)
    x, y = x.cuda(), y.cuda()
    info = gpu_info()
    rows = []
    pairs = [(odd, even, False) for odd, even in PAIRS] + [([a], [b], True) for a, b in ENC_PAIRS]
    for odd, even, enc in pairs:
        models = {tuple(odd): make(odd, F, enc), tuple(even): make(even, F, enc)}
        opts = {k: FlatAdam(m, lr=1e-4) for k, m in models.items()}
        for k, m in models.items():
            step_time(m, opts[k], x, y, 3)            # warm-up
        times = {k: [] for k in models}
        for _ in range(a.rounds):
            for k, m in models.items():
                times[k].append(step_time(m, opts[k], x, y, a.steps))
        row = {"gpu": info, "B": a.batch, "S": a.slate, "F": F, "encoder": "N 2, h 2, d_ff 2d" if enc else None}
        for k, t in times.items():
            t = sorted(t)
            row["x".join(map(str, k))] = {"median_ms": round(t[len(t) // 2], 4), "min_ms": round(t[0], 4),
                                          "max_ms": round(t[-1], 4)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_fc_widths.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
