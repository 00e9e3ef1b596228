"""Training-step time with dropout at allRank's batch size: eager steps (host-drawn dropout seed, one launch sequence per
step) against CUDA-graph replays of the same step (GraphedTrainStep(dropout_seed=...): the seed is read from device
memory).  The models and losses are those of the shipped configurations that train with dropout, at B = 64, S = 240,
F = 136, with FlatAdam(capturable=True) in both arms.  The two arms alternate within each round; the median over the
rounds is reported, with the card's name and power limit.

    python tools/bench_graph_dropout.py [--steps 100] [--warmup 10] [--rounds 5] [--eager-only] [--out FILE.json]

--eager-only times the eager host-seeded step alone (the path a device-read seed must not slow down).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {   # contextaware_web30k/{ndcgloss2pp,ordinal,ordinal_mlp}.json, neuralndcg_web30k/approxndcg.json
    "ndcgloss2pp": ({"sizes": [128], "activation": None, "dropout": 0.0},
                    {"N": 4, "d_ff": 512, "h": 4, "dropout": 0.3}, {"d_output": 1, "output_activation": None},
                    "lambdaLoss", {"weighing_scheme": "ndcgLoss2PP_scheme", "k": None, "mu": 10, "sigma": 1.0}),
    "ordinal": ({"sizes": [144], "activation": None, "dropout": 0.0},
                {"N": 4, "d_ff": 512, "h": 2, "dropout": 0.4}, {"d_output": 4, "output_activation": "Sigmoid"},
                "ordinal", {"n": 4}),
    "approxndcg": ({"sizes": [96], "activation": None, "dropout": 0.0},
                   {"N": 2, "d_ff": 384, "h": 1, "dropout": 0.1}, {"d_output": 1, "output_activation": None},
                   "approxNDCGLoss", {"alpha": 1.0}),
    "ordinal_mlp": ({"sizes": [256, 512, 1024, 512, 256], "activation": "ReLU", "dropout": 0.3}, None,
                    {"d_output": 4, "output_activation": "Sigmoid"}, "ordinal", {"n": 4}),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def setup(name, B, S, F):
    from allrank_b200 import losses
    from allrank_b200.model import make_model
    from allrank_b200.optim import FlatAdam
    from allrank_b200.synth import make_slates
    fc, tr, post, loss_name, loss_kw = CONFIGS[name]
    torch.manual_seed(0)
    if tr is not None:
        tr = dict(tr, positional_encoding=None)
    model = make_model(fc_model=dict(fc, input_norm=False), transformer=tr, post_model=post,
                       n_features=F).cuda().train()
    opt = FlatAdam(model, lr=1e-3, capturable=True)
    x, y, _ = make_slates(B, S, F, seed=1, mean_len=120.0, std_len=60.0)
    return model, opt, getattr(losses, loss_name), loss_kw, x.cuda(), y.cuda()


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--eager-only", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_dropout.py needs a CUDA device")
    B, S, F = a.batch, 240, 136
    name, power = card()
    result = {"gpu": name, "power_limit": power, "batch": B, "slate_length": S, "n_features": F, "steps": a.steps,
              "rounds": a.rounds, "configs": {}}
    for cfg in a.configs.split(","):
        model, opt, loss_fn, loss_kw, x, y = setup(cfg, B, S, F)
        mask = y == -1

        def eager():
            loss = loss_fn(model(x, mask, None), y, **loss_kw)
            opt.zero_grad()
            loss.backward()
            opt.step()

        arms = {"eager_ms": eager}
        if not a.eager_only:
            from allrank_b200.graph import GraphedTrainStep
            step = GraphedTrainStep(model, loss_fn, opt, x, y, loss_kwargs=loss_kw, dropout_seed=1)
            arms["graph_ms"] = step.replay
        for fn in arms.values():
            timed(fn, a.warmup)
        times = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, fn in arms.items():
                times[k].append(timed(fn, a.steps))
        row = {k: round(statistics.median(v), 4) for k, v in times.items()}
        row.update({k.replace("_ms", "_all_ms"): [round(t, 4) for t in v] for k, v in times.items()})
        if "graph_ms" in row:
            row["speedup"] = round(row["eager_ms"] / row["graph_ms"], 3)
        result["configs"][cfg] = row
        print(cfg, json.dumps(row), flush=True)
        del model, opt, arms
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
