"""File -> SlateStore wall time of the two LibSVM parsers on an MSLR-shaped file (tests/libsvm_cases.mslr_text).

    python tools/bench_libsvm.py [--rows 2270000] [--seed 0] [--rounds 2] [--out DIR]

The file is generated from the seed into a temporary directory (MSLR-WEB30K's train fold has 2.27 M rows).  Rounds
alternate the parsers (sklearn, device, sklearn, device, ...).  For the device parser the time is split into the
file read + upload, pass 1 (line index and validation, to its summary read-back) and pass 2 + store (dense rows,
group offsets, upload of the offsets).  Prints the GPU name and power limit of the same run, then one JSON line.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from allrank_b200.data import LibSVMPlan, SlateStore, group_offsets, read_svm_to_device  # noqa: E402
from tests.libsvm_cases import mslr_text  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def device_split(path, dev):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    text = read_svm_to_device(path, dev)
    t1 = time.perf_counter()
    plan = LibSVMPlan(text)
    t2 = time.perf_counter()
    x = torch.empty((plan.n_rows, plan.n_features), device=dev)
    y = torch.empty((plan.n_rows,), device=dev)
    q = torch.empty((plan.n_rows,), dtype=torch.int64, device=dev)
    plan.write(x, y, q)
    offsets = torch.from_numpy(group_offsets(q.cpu().numpy())).to(dev)
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    return {"read_upload_s": t1 - t0, "pass1_s": t2 - t1, "pass2_store_s": t3 - t2, "total_s": t3 - t0,
            "n_rows": plan.n_rows, "offsets": int(offsets.numel())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_270_000)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None, help="directory for the JSON result (optional)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_libsvm.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    print("gpu:", gpu_info(), flush=True)
    res = {"rows": args.rows, "seed": args.seed, "gpu": gpu_info(), "sklearn_s": [], "device_s": [], "device_split": []}
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "train.txt")
        t = time.perf_counter()
        with open(path, "wb") as fh:
            fh.write(mslr_text(args.rows, seed=args.seed))
        res["bytes"] = os.path.getsize(path)
        print("generated {} bytes in {:.1f} s".format(res["bytes"], time.perf_counter() - t), flush=True)
        device_split(path, dev)                      # warm-up: module load, allocator
        for r in range(args.rounds):
            torch.cuda.synchronize()
            t = time.perf_counter()
            SlateStore.from_svm_file(path, device=dev, parser="sklearn")
            torch.cuda.synchronize()
            res["sklearn_s"].append(time.perf_counter() - t)
            torch.cuda.synchronize()
            t = time.perf_counter()
            SlateStore.from_svm_file(path, device=dev, parser="device")
            torch.cuda.synchronize()
            res["device_s"].append(time.perf_counter() - t)
            res["device_split"].append(device_split(path, dev))
            print("round {}: sklearn {:.2f} s, device {:.3f} s, split {}".format(
                r, res["sklearn_s"][-1], res["device_s"][-1], res["device_split"][-1]), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_libsvm.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
