"""Times allRank's write_to_libsvm_without_masked (sklearn's dump_svmlight_file) against the device writer
(allrank_b200.writer) on an MSLR-WEB30K-shaped click-through role: 136 float32 features, ~40 % zeros, 0/1 labels,
slates of 1 to 240 rows.  Prints one JSON line: seconds and MB/s of the file for both, and the device time split into
upload, format (the kernels alone) and download + file write.

    python tools/bench_libsvm_write.py [--rows 2270000] [--sklearn-rows 200000] [--out DIR]

sklearn's time is measured on --sklearn-rows rows and scaled to --rows (its per-row loop has no fixed cost worth the
name); both files are compared byte for byte on the rows both wrote.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from allrank_b200 import writer  # noqa: E402
from tests import libsvm_write_cases as C  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception:                       # noqa: BLE001
        return "unknown"


def slates(X, y, qid):
    """The role as the list of clicked slates write_to_libsvm_without_masked receives (no padding left)."""
    cuts = np.flatnonzero(np.diff(qid)) + 1
    return np.split(X, cuts), np.split(y, cuts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_270_000)
    ap.add_argument("--sklearn-rows", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    X, y, qid = C.mslr_block(n_rows=a.rows, seed=3)
    out_dir = a.out or tempfile.mkdtemp()
    os.makedirs(out_dir, exist_ok=True)
    dev_path, ref_path = os.path.join(out_dir, "device.txt"), os.path.join(out_dir, "sklearn.txt")
    torch.cuda.init()
    torch.empty(1, device="cuda").sum().item()

    # device arm, end to end through the allRank entry point
    Xs, ys = slates(X, y, qid)
    writer.write_to_libsvm_without_masked(dev_path + ".warm", Xs[:100], ys[:100])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    writer.write_to_libsvm_without_masked(dev_path, Xs, ys)
    t_dev = time.perf_counter() - t0
    size = os.path.getsize(dev_path)

    # the device time split: upload, format (kernels only), download + file write
    t0 = time.perf_counter()
    rows = writer.DeviceRows(X, y, query_id=qid)
    torch.cuda.synchronize()
    t_up = time.perf_counter() - t0
    t0 = time.perf_counter()
    for _ in rows.chunks():
        pass
    torch.cuda.synchronize()
    t_fmt = time.perf_counter() - t0
    t0 = time.perf_counter()
    with open(dev_path + ".split", "wb") as fh:
        rows.write_to(fh)
    t_write = time.perf_counter() - t0 - t_fmt

    # sklearn arm on the first slates covering --sklearn-rows rows
    sys.path[:0] = [os.path.join(ROOT, "oracle", "_stubs")]
    from sklearn.datasets import dump_svmlight_file
    n_ref = min(a.sklearn_rows, a.rows)
    k = int(np.searchsorted(np.cumsum([len(v) for v in ys]), n_ref, side="right"))
    n_ref = int(sum(len(v) for v in ys[:k]))

    def reference_write(path, Xl, yl):       # allrank/data/dataset_saving.py:9-32 as it stands
        Xv, yv, qv = [], [], []
        for q, (xs, yq) in enumerate(zip(Xl, yl)):
            mask = yq != -1
            Xv.append(xs[mask]), yv.append(yq[mask]), qv.append(np.repeat(q, len(yq[mask])))
        dump_svmlight_file(np.vstack(Xv), np.concatenate(yv), path, query_id=np.concatenate(qv))

    t0 = time.perf_counter()
    reference_write(ref_path, Xs[:k], ys[:k])
    t_ref = time.perf_counter() - t0
    ref_size = os.path.getsize(ref_path)
    with open(ref_path, "rb") as r, open(dev_path, "rb") as d:
        same = r.read() == d.read(ref_size)
    mb = size / 1e6
    print(json.dumps({
        "gpu": gpu_info(), "rows": a.rows, "features": X.shape[1], "file_MB": round(mb, 1),
        "sklearn": {"rows": n_ref, "s": round(t_ref, 3), "MB_per_s": round(ref_size / 1e6 / t_ref, 2),
                    "s_scaled_to_rows": round(t_ref * a.rows / n_ref, 1)},
        "device": {"s": round(t_dev, 3), "MB_per_s": round(mb / t_dev, 1), "upload_s": round(t_up, 3),
                   "format_s": round(t_fmt, 3), "download_and_write_s": round(t_write, 3)},
        "speedup": round(t_ref * a.rows / n_ref / t_dev, 1), "identical_prefix": same}))
    for p in (dev_path, dev_path + ".warm", dev_path + ".split", ref_path):
        os.remove(p)


if __name__ == "__main__":
    main()
