"""Edge cases of the ranking metrics from the UNMODIFIED reference (allrank/models/metrics.py) ->
tests/golden/metrics_edges.npz.  Run where an allRank source tree is available ($ALLRANK_REFERENCE, default
/root/reference):

    PYTHONDONTWRITEBYTECODE=1 python tools/make_golden_metrics_edges.py

Cases: cut-offs <= 0, above the slate and empty lists; padding indicators 0 and -5 (0 also a real label); fillers 0
and 0.25 with slates whose ideal DCG is 0; the identity gain with negative labels; fractional labels; NaN, +-inf and
+-0 scores (a real -inf item among padded ones) at S <= 16.  For each case the file holds the inputs, the call (JSON)
and either the reference's output or the name of the exception it raised.  The reference sorts with torch's default
(unstable) sort; the score cases are kept only where that sort agrees with the stable one, the order the CUDA kernel
documents.  The tests read only the committed file.
"""
import json
import os
import sys

os.environ["CUDA_VISIBLE_DEVICES"] = ""
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle", "_stubs"), os.environ.get("ALLRANK_REFERENCE", "/root/reference"), ROOT]
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402
import torch  # noqa: E402

from allrank.models import metrics as ref  # noqa: E402

NAN, INF = float("nan"), float("inf")


def cases():
    g = torch.Generator().manual_seed(4242)
    out = {}

    def add(name, fn, yp, yt, ats, gain="pow2", pad=-1.0, filler=1.0, frac=False):
        out[name] = dict(fn=fn, yp=torch.as_tensor(yp, dtype=torch.float32),
                         yt=torch.as_tensor(yt, dtype=torch.float32), ats=ats, gain=gain, pad=pad, filler=filler,
                         frac=frac)

    # cut-offs: the reference reads cum_dcg[:, at - 1] of max(clipped ats) columns
    yp = [[0.9, 0.1, 0.5, 0.3, 0.7], [0.2, 0.4, 0.6, 0.8, 1.0]]
    yt = [[1.0, 3.0, 0.0, 2.0, 1.0], [0.0, 2.0, -1.0, 1.0, 4.0]]
    for fn, ats in [("dcg", [0, 2]), ("ndcg", [0, 3]), ("dcg", [-1, 4]), ("ndcg", [-2, 5]), ("dcg", [3, -3]),
                    ("dcg", []), ("ndcg", []), ("mrr", []), ("mrr", [0, -1, 7, 2]), ("dcg", [7, 0]), ("dcg", [-2]),
                    ("dcg", [0]), ("dcg", [-5]), ("ndcg", [9, -1, 9, 1]), ("dcg", None), ("mrr", None)]:
        add(f"ats_{fn}_{'none' if ats is None else '_'.join(map(str, ats))}", fn, yp, yt, ats)

    # padding indicators and fillers, with all-zero and all-padded slates
    yp = torch.randn(4, 8, generator=g)
    for pad in (0.0, -5.0):
        yt = torch.randint(0, 4, (4, 8), generator=g).float()
        yt[0, 5:] = pad
        yt[1] = 0.0
        yt[1, 6:] = pad
        yt[2] = pad
        yt[3, 2] = pad
        for fn in ("dcg", "ndcg", "mrr"):
            add(f"pad{int(pad)}_{fn}", fn, yp, yt, [1, 3, 8], pad=pad)
        for filler in (0.0, 0.25):
            add(f"pad{int(pad)}_fill{filler}", "ndcg", yp, yt, [2, 8], pad=pad, filler=filler)

    # identity gain with negative labels (and a -0.0 label)
    yp = torch.randn(3, 10, generator=g)
    yt = torch.randint(-3, 4, (3, 10), generator=g).float()
    yt[0, 7:] = -1.0
    yt[1] = -2.0
    yt[2, 0] = -0.0
    for fn in ("dcg", "ndcg"):
        add(f"identity_neg_{fn}", fn, yp, yt, [1, 4, 10], gain="identity", pad=-7.0)

    # fractional labels in [0, 5) and (-1, 0)
    yp = torch.randn(4, 12, generator=g)
    pos = torch.rand(4, 12, generator=g) * 5.0
    neg = -torch.rand(4, 12, generator=g)
    for lab_name, yt in (("pos", pos), ("neg", torch.where(neg == 0.0, torch.tensor(-0.5), neg))):
        yt = yt.clone()
        yt[0, 9:] = -1.0
        for gain in ("pow2", "identity"):
            for fn in ("dcg", "ndcg"):
                add(f"frac_{lab_name}_{gain}_{fn}", fn, yp, yt, [1, 5, 12], gain=gain, frac=True)
        add(f"frac_{lab_name}_mrr", "mrr", yp, yt, [1, 5, 12], frac=True)

    # NaN / +-inf / +-0 scores and ties among the real items, a real -inf item before and after padded ones
    yp = [[NAN, 1.0, INF, -INF, 0.0, -0.0, 1.0, NAN, 2.0, -INF, 0.0, INF, -0.0, 2.0, -1.0, NAN],
          [-INF, 0.5, -0.0, 0.0, -INF, 0.5, NAN, 3.0, -INF, 0.0, 0.5, -0.0, INF, -INF, 1.0, 0.0],
          [0.0, -0.0, 0.0, -0.0, 1.0, 1.0, -INF, -INF, NAN, NAN, INF, INF, 0.0, -0.0, 0.0, -0.0]]
    yt = [[2.0, 0.0, 1.0, 3.0, 4.0, 1.0, 2.0, 0.0, 1.0, -1.0, 2.0, -1.0, 3.0, 0.0, 1.0, -1.0],
          [3.0, -1.0, 1.0, 2.0, -1.0, 0.0, 1.0, -1.0, 4.0, 1.0, -1.0, 2.0, 0.0, 1.0, 2.0, -1.0],
          [1.0, 2.0, 3.0, 4.0, 0.0, 1.0, 2.0, -1.0, 3.0, 0.0, 1.0, 2.0, -1.0, 4.0, 0.0, 1.0]]
    for S in (5, 16):
        for fn in ("dcg", "ndcg", "mrr"):
            add(f"scores_S{S}_{fn}", fn, [r[:S] for r in yp], [r[:S] for r in yt], [1, 2, 4, S])
        add(f"scores_S{S}_identity_dcg", "dcg", [r[:S] for r in yp], [r[:S] for r in yt], [1, 3, S], gain="identity")
    return out


def stable_agrees(yp, yt, pad):
    for key in (yp.masked_fill(yt == pad, -INF), yt.masked_fill(yt == pad, -INF)):
        if not torch.equal(key.sort(descending=True, dim=-1).indices,
                           key.sort(descending=True, stable=True, dim=-1).indices):
            return False
    return True


def main():
    blob = {}
    names = []
    for name, c in cases().items():
        if name.startswith("scores_"):
            assert stable_agrees(c["yp"], c["yt"], c["pad"]), name
        kw = {"padding_indicator": c["pad"]}
        if c["fn"] != "mrr":
            kw["gain_function"] = (lambda x: x) if c["gain"] == "identity" else (lambda x: torch.pow(2, x) - 1)
        if c["fn"] == "ndcg":
            kw["filler_value"] = c["filler"]
        call = {k: c[k] for k in ("fn", "ats", "gain", "pad", "filler", "frac")}
        try:
            res = getattr(ref, c["fn"])(c["yp"].clone(), c["yt"].clone(), ats=c["ats"], **kw)
            blob[name + ":out"] = res.numpy()
            call["raises"] = None
        except Exception as exc:  # the exception type is part of the reference's behaviour
            call["raises"] = type(exc).__name__
        blob[name + ":pred"], blob[name + ":true"] = c["yp"].numpy(), c["yt"].numpy()
        blob[name + ":call"] = np.array(json.dumps(call))
        names.append(name)
        print(name, call["raises"] or tuple(blob[name + ":out"].shape))
    blob["names"] = np.array(names)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "metrics_edges.npz"), **blob)


if __name__ == "__main__":
    main()
