"""Throughput of the device click models: slates/s of `click_on_slates` (host lists in and out, as rank_and_click.py
uses it) and of the device `click()` (tensors already on the GPU, CUDA events), per model kind, on N synthetic
MSLR-shaped ranked slates (S = 240, F = 136, 20-240 real items, labels 0-4); next to the unmodified reference's
click_on_slates on a host sample when oracle/_ref is present.

    python tools/bench_clicks.py [--slates 20000] [--ref-slates 500] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KINDS = {
    "OnlyRelevant(1)": {"name": "OnlyRelevantClickModel", "args": {"relevancy_threshold": 1}},
    "BaseCascade(1,1)": {"name": "BaseCascadeModel", "args": {"eta": 1, "threshold": 1}},
    "Random(3)": {"name": "RandomClickModel", "args": {"n_clicks": 3}},
    "Fixed([0,2,-1])": {"name": "FixedClickModel", "args": {"click_positions": [0, 2, -1]}},
    "Multiple": {"name": "MultipleClickModel", "args": {"inner_click_models": [
        {"name": "OnlyRelevantClickModel", "args": {"relevancy_threshold": 2}},
        {"name": "BaseCascadeModel", "args": {"eta": 0.5, "threshold": 1}}], "probabilities": [0.5, 0.5]}},
    "Conditioned(any)": {"name": "ConditionedClickModel", "args": {"inner_click_models": [
        {"name": "OnlyRelevantClickModel", "args": {"relevancy_threshold": 3}},
        {"name": "FixedClickModel", "args": {"click_positions": [0]}}], "combiner": "np.any"}},
    "MaxClicks(Cascade,2)": {"name": "MaxClicksModel", "args": {"inner_click_model": {
        "name": "BaseCascadeModel", "args": {"eta": 1, "threshold": 1}}, "max_clicks": 2}},
    "Duplicates(euclidean)": {"name": "EverythingButDuplicatesClickModel",
                              "args": {"duplicate_margin": 12.0, "metric": "euclidean"}},
    "Diverse(OnlyRelevant(1))": {"name": "DiverseClicksModel", "args": {"inner_click_model": {
        "name": "OnlyRelevantClickModel", "args": {"relevancy_threshold": 1}}, "q_percentile": 0.5}},
    "Diverse(Cascade(0.5,2))": {"name": "DiverseClicksModel", "args": {"inner_click_model": {
        "name": "BaseCascadeModel", "args": {"eta": 0.5, "threshold": 2}}, "q_percentile": 0.5}},
}


def slates(N, S=240, F=136, seed=0):
    rng = np.random.RandomState(seed)
    x = rng.randn(N, S, F).astype(np.float32)
    y = rng.randint(0, 5, (N, S)).astype(np.float32)
    n = rng.randint(20, S + 1, N)
    y[np.arange(S)[None, :] >= n[:, None]] = -1.0
    x[y == -1] = 0.0
    return torch.from_numpy(x), torch.from_numpy(y)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slates", type=int, default=20000)
    ap.add_argument("--ref-slates", type=int, default=500)
    ap.add_argument("--out")
    a = ap.parse_args()
    from allrank_b200 import click_models as cmod
    from oracle.clicks_ref import build_model
    from oracle.install_reference import import_path, installed
    assert torch.cuda.is_available(), "bench_clicks measures the GPU path and needs a CUDA device"
    dev = torch.device("cuda:0")
    x, y = slates(a.slates)
    xd, yd = x.to(dev), y.to(dev)
    ref_cu = ref_classes = None
    if installed() and a.ref_slates > 0:
        sys.path[:0] = import_path()
        import allrank.click_models.click_utils as ref_cu
        from tools.make_golden_clicks import reference_classes
        ref_classes = reference_classes()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip()
    rows = []
    for label, spec in KINDS.items():
        model = build_model(spec, cmod)
        cmod.click(model, xd[:64], yd[:64], seed=1)                       # warm-up (module load, tables)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 3
        e0.record()
        for r in range(reps):
            cmod.click(model, xd, yd, seed=r, check=False)
        e1.record()
        torch.cuda.synchronize()
        dev_s = e0.elapsed_time(e1) / 1e3 / reps
        np.random.seed(0)
        t0 = time.perf_counter()
        cmod.click_on_slates((x, y), model, include_empty=True)
        host_s = time.perf_counter() - t0
        row = {"model": label, "slates": a.slates, "device_click_slates_per_s": a.slates / dev_s,
               "click_on_slates_slates_per_s": a.slates / host_s}
        if ref_cu is not None:
            k = a.ref_slates
            np.random.seed(0)
            t0 = time.perf_counter()
            ref_cu.click_on_slates((x[:k], y[:k]), build_model(spec, ref_classes), include_empty=True)
            row["reference_host_slates_per_s"] = k / (time.perf_counter() - t0)
            row["reference_slates"] = k
        row["gpu"] = gpu
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
