"""Times `allrank_b200.normalize.normalize_features` on an MSLR-shaped fold (tests/normalize_cases.mslr_fold: 136
features, train of --rows rows, test and vali a third of that each) and the script's algorithm on the host
(oracle/normalize_ref.py with np.log) on --reference-rows, scaled linearly to the full fold.

    python tools/bench_normalize.py --rows 300000 --reference-rows 3000

Prints one JSON line: the card and power limit from the same run, the device path end to end after one warm-up, split
into read + parse, the transforms + statistics, and format + write, and the reference arm.
"""
import argparse
import contextlib
import io
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from allrank_b200 import normalize as N  # noqa: E402
from tests import normalize_cases as C  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def device_run(fold, fwl, fneg, dev):
    """(read + parse, transforms + statistics, format + write) seconds, each ending in a synchronise."""
    t0 = time.perf_counter()
    loaded = [N._load_role(os.path.join(fold, r + ".txt"), dev) for r in C.ROLES]
    torch.cuda.synchronize(dev)
    t1 = time.perf_counter()
    roles = [x for x, _, _, _ in loaded]
    N.normalize_roles(roles[0], roles[1:], fwl, fneg)
    torch.cuda.synchronize(dev)
    t2 = time.perf_counter()
    out_dir = fold + "_normalized"
    os.makedirs(out_dir, exist_ok=True)
    for r, (x, y, q, _) in zip(C.ROLES, loaded):
        rows = N.DeviceRows(x, y, zero_based=True, query_id=q, device=dev)
        with open(os.path.join(out_dir, r + ".txt"), "wb") as f:
            rows.write_to(f)
    torch.cuda.synchronize(dev)
    return t1 - t0, t2 - t1, time.perf_counter() - t2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=300_000)
    ap.add_argument("--reference-rows", type=int, default=3000)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    tmp = tempfile.mkdtemp()
    try:
        texts, fwl, fneg = C.mslr_fold(a.rows, seed=1)
        fold = os.path.join(tmp, "fold")
        C.write_fold(texts, fold)
        in_bytes = sum(len(t) for t in texts.values())
        with contextlib.redirect_stdout(io.StringIO()):
            N.normalize_features(fold, fwl, fneg, device=dev)          # warm-up, and the end-to-end entry point
            t = time.perf_counter()
            N.normalize_features(fold, fwl, fneg, device=dev)
            torch.cuda.synchronize(dev)
            end_to_end = time.perf_counter() - t
            parts = [device_run(fold, fwl, fneg, dev) for _ in range(a.repeats)]
        out_bytes = sum(os.path.getsize(os.path.join(fold + "_normalized", r + ".txt")) for r in C.ROLES)
        best = np.min(np.array(parts), axis=0)
        from oracle import normalize_ref as R
        rtexts, _, _ = C.mslr_fold(a.reference_rows, seed=1)
        rfold = os.path.join(tmp, "ref")
        C.write_fold(rtexts, rfold)
        t = time.perf_counter()
        R.normalize(rfold, fwl, fneg, log=np.log)
        ref = (time.perf_counter() - t) * a.rows / a.reference_rows
        print(json.dumps({"card": card(), "rows_train": a.rows, "input_bytes": in_bytes, "output_bytes": out_bytes,
                          "device_end_to_end_s": round(end_to_end, 3), "read_parse_s": round(best[0], 3),
                          "transform_stats_s": round(best[1], 3), "format_write_s": round(best[2], 3),
                          "reference_rows": a.reference_rows, "reference_scaled_s": round(ref, 1),
                          "speedup": round(ref / end_to_end, 1)}))
    finally:
        shutil.rmtree(tmp)


if __name__ == "__main__":
    main()
