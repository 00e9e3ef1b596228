"""What each FC activation costs: a training step (forward, approxNDCG loss, backward, FlatAdam) of an FC-only MLP at
the MSLR shape (136 features, sizes [256, 128], FC dropout 0.1) for each of the sixteen activations, B = 4096 slates of
S = 240 items, the models taking turns round by round; and the summed GPU time of the activation kernels
(act_fwd_kernel, act_bwd_kernel) in one step, from torch.profiler.  ReLU and None run inside the GEMM epilogues, so their
activation-kernel time is that of the dropout passes alone.

    python tools/bench_activations.py [--rounds 5] [--steps 10] [--out DIR]

Prints one JSON line per activation (median and spread of the per-round step times, activation-kernel time) and the
GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

ACTS = [None, "ReLU", "Tanh", "Sigmoid", "LeakyReLU", "ELU", "CELU", "SELU", "Softplus", "Softsign", "Hardtanh",
        "ReLU6", "Hardsigmoid", "LogSigmoid", "Hardshrink", "Softshrink"]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or "unknown"


def make(act, F):
    from allrank_b200.model import make_model
    torch.manual_seed(0)
    return make_model({"sizes": [256, 128], "input_norm": False, "activation": act, "dropout": 0.1}, None,
                      {"d_output": 1, "output_activation": None}, F).cuda().train()


def run(model, opt, x, y, steps):
    from allrank_b200 import losses
    mask = y == -1
    for _ in range(steps):
        loss = losses.approxNDCGLoss(model(x, mask, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()


def step_time(model, opt, x, y, steps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    run(model, opt, x, y, steps)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def act_kernel_ms(model, opt, x, y):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(model, opt, x, y, 1)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if e.key.startswith(("arb::act_fwd", "arb::act_bwd",
                                                                                    "act_fwd", "act_bwd")))
    return us / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--slate", type=int, default=240)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_activations: no GPU")
    from allrank_b200.optim import FlatAdam
    from allrank_b200.synth import make_slates
    F = 136
    x, y, _ = make_slates(a.batch, a.slate, n_features=F, seed=3, mean_len=int(0.75 * a.slate), std_len=a.slate // 5)
    x, y = x.cuda(), y.cuda()
    info = gpu_info()
    models = {str(k): make(k, F) for k in ACTS}
    opts = {k: FlatAdam(m, lr=1e-4) for k, m in models.items()}
    for k, m in models.items():
        step_time(m, opts[k], x, y, 2)                  # warm-up
    times = {k: [] for k in models}
    for r in range(a.rounds):
        order = list(models) if r % 2 == 0 else list(models)[::-1]
        for k in order:
            times[k].append(step_time(models[k], opts[k], x, y, a.steps))
    rows = []
    for k, t in times.items():
        t = sorted(t)
        row = {"gpu": info, "B": a.batch, "S": a.slate, "F": F, "sizes": [256, 128], "activation": k,
               "step_median_ms": round(t[len(t) // 2], 3), "step_min_ms": round(t[0], 3), "step_max_ms": round(t[-1], 3),
               "activation_kernels_ms": round(act_kernel_ms(models[k], opts[k], x, y), 3)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_activations.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
