"""Training steps of a cfg2-shaped Transformer scorer (N = 2, h = 4, d = 128, d_ff = 512, approxNDCGLoss) on slates
longer than 256 items: the fused long-slate attention kernels (csrc/attention_long.cu, attention mode 2) against the
unfused sequence (arb_set_attention_mode(0): [B, h, S, S] probabilities in HBM) where the latter exists (S <= 1536).

    python tools/bench_long_slates.py [--steps 5] [--warmup 2] [--runs 3] [--items 245760] [--json out.json]

Batches hold B = items / S slates (fewer where the unfused path would not fit in memory), with two length profiles:
full slates and extents ~ N(S/2, S/4) clamped to [1, S].  Step time is the host clock around `steps` training steps
that end in a device synchronise, per run; the modes alternate run by run.  Peak memory is
torch.cuda.max_memory_allocated over a run.  The attention kernels' times come from torch.profiler in a separate run
per shape.  The GPU's name and power limit are printed with the numbers."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHORT = (512, 1024, 1536)      # both paths
LONG = (2048, 4096)            # beyond the unfused softmax: fused kernels only


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def set_mode(mode):
    from allrank_b200 import _lib
    L = _lib.lib()
    L.arb_set_attention_mode.argtypes = [ctypes.c_int32]
    L.arb_set_attention_mode(mode)


def make_batch(B, S, profile, seed=7):
    from allrank_b200.synth import make_slates
    x, y, _ = make_slates(B, S, n_features=136, seed=seed, mean_len=S / 2, std_len=S / 4, full=profile == "full")
    return x.cuda(), y.cuda()


def make_step():
    from allrank_b200 import losses
    from allrank_b200.model import make_model
    from allrank_b200.optim import FlatAdam
    torch.manual_seed(0)
    model = make_model(fc_model={"sizes": [128], "input_norm": False, "activation": None, "dropout": 0.0},
                       transformer={"N": 2, "d_ff": 512, "h": 4, "positional_encoding": None, "dropout": 0.0},
                       post_model={"d_output": 1, "output_activation": None}, n_features=136).cuda().train()
    opt = FlatAdam(model, lr=1e-3)

    def step(x, y):
        loss = losses.approxNDCGLoss(model(x, y == -1, None), y, alpha=1.0)
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss
    return step


def timed(step, x, y, steps, warmup):
    for _ in range(warmup):
        step(x, y)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    for _ in range(steps):
        step(x, y)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3, torch.cuda.max_memory_allocated() / 2 ** 30


def kernel_times(step, x, y):
    """ms per step of every attention kernel (profiler run of one step after one warm-up step)."""
    from torch.profiler import ProfilerActivity, profile
    step(x, y)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(x, y)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "attn" in e.key or "softmax" in e.key:
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            key = e.key.split("(")[0].split("<")[0].replace("void ", "").replace("arb::", "")
            out[key] = out.get(key, 0.0) + t / 1e3
    return out


def fits_unfused(B, S):
    """The unfused path's [B, h, S, S] buffers: one per layer in the workspace plus two in the backward scratch."""
    return (2 + 2) * B * 4 * S * S * 4 < 0.7 * torch.cuda.get_device_properties(0).total_memory


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--items", type=int, default=245760)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    name, power = gpu_info()
    print(f"GPU: {name}; power limit, max SM clock: {power}", flush=True)
    step = make_step()
    rows = []
    for S in SHORT + LONG:
        B = max(1, args.items // S)
        modes = (2,)
        if S in SHORT:
            while not fits_unfused(B, S):
                B //= 2
            modes = (2, 0)
        for profile in ("full", "half"):
            x, y = make_batch(B, S, profile)
            res = {m: [] for m in modes}
            for _ in range(args.runs):
                for m in modes:
                    set_mode(m)
                    res[m].append(timed(step, x, y, args.steps, args.warmup))
            set_mode(2)
            kt = {m: None for m in modes}
            for m in modes:
                set_mode(m)
                kt[m] = kernel_times(step, x, y)
            set_mode(2)
            for m in modes:
                ms = [r[0] for r in res[m]]
                mem = max(r[1] for r in res[m])
                row = dict(S=S, B=B, profile=profile, path="fused" if m == 2 else "unfused", step_ms=ms,
                           peak_gib=mem, attention_kernel_ms=kt[m])
                rows.append(row)
                print(f"S={S:5d} B={B:4d} {profile:4s} {row['path']:7s} step ms " +
                      " / ".join(f"{v:8.2f}" for v in ms) + f"   peak {mem:6.2f} GiB   kernels " +
                      ", ".join(f"{k} {v:.2f}" for k, v in sorted(kt[m].items())), flush=True)
            del x, y
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(gpu=name, power=power, steps=args.steps, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
