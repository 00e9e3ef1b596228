"""The redraw and append rules of the UNMODIFIED reference's FixLength._sample (allrank/data/dataset_loading.py:61-79)
-> tests/golden/slates_rules.npz.  Run where an allRank source tree is available ($ALLRANK_REFERENCE, default
/root/reference):

    PYTHONDONTWRITEBYTECODE=1 python tools/make_golden_slates_rules.py

np.random.choice is replaced by a scripted chooser: the k-th call choice(n, S) returns the k-th scripted draw (the
last one again once the script runs out) and choice(indices, m) returns indices[sub[:m]] for a scripted position
list `sub`.  Each case records the labels, the script and what FixLength returned -- the kept, redrawn or appended
indices and the number of draws -- or the name of the exception it raised.  Every label sum is exact in fp32, so the
rules read the same on the fp32 labels the CUDA kernel sums.  The tests read only the committed file.
"""
import json
import os
import sys

os.environ["CUDA_VISIBLE_DEVICES"] = ""
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "oracle", "_stubs"), os.environ.get("ALLRANK_REFERENCE", "/root/reference"), ROOT]
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402

from allrank.data.dataset_loading import FixLength  # noqa: E402

NAN = float("nan")

# name: (labels, S, draws of choice(n, S) in call order, positions for choice(indices, S - 1))
CASES = {
    "zero_labels_keep": ([0, 0, 0, 0, 0, 0], 3, [[3, 1, 4]], [2, 1, 0]),
    "single_one_hit": ([0, 0, 1, 0, 0, 0], 3, [[2, 4, 1]], [2, 1, 0]),
    "single_one_append": ([0, 0, 1, 0, 0, 0], 3, [[5, 0, 3]], [2, 0, 1]),
    "single_one_append_first": ([0, 0, 0, 0, 1, 0, 0], 4, [[6, 0, 3, 1]], [0, 1, 2, 3]),
    "sum2_two_ones_redraw": ([1, 0, 0, 0, 1, 0], 3, [[1, 2, 3], [5, 2, 0]], [2, 1, 0]),
    "sum2_one_two_redraw_twice": ([0, 2, 0, 0, 0], 2, [[0, 3], [4, 2], [3, 1]], [1, 0]),
    "sum2_hit": ([0, 2, 0, 0, 0], 2, [[1, 3]], [1, 0]),
    "sum_minus1_keep": ([-1, 0, 0, 0, 0], 2, [[1, 2]], [1, 0]),
    "sum_minus1_mixed_keep": ([1, -2, 0, 0, 0], 2, [[2, 3]], [1, 0]),
    "sum_zero_mixed_keep": ([1, -1, 0, 0, 0], 2, [[3, 4]], [1, 0]),
    "nan_keep": ([NAN, 0, 0, 0, 0], 2, [[1, 2]], [1, 0]),
    "nan_with_one_keep": ([NAN, 1, 0, 0, 0], 2, [[2, 3]], [1, 0]),
    "nan_drawn_keep": ([NAN, 1, 0, 0, 0], 2, [[0, 3]], [1, 0]),
    "frac_quarter_append_argmax": ([0.25, 0.75, 0, 0, 0], 2, [[2, 3]], [1, 0]),
    "frac_half_append_argmax": ([0.5, 1.5, -1, 0, 0], 2, [[3, 4]], [1, 0]),
    "frac_half_hit_negative": ([0.5, 1.5, -1, 0, 0], 2, [[2, 4]], [1, 0]),
    "ones_minus_one_append_first_max": ([1, 1, -1, 0, 0], 2, [[3, 4]], [1, 0]),
    "ones_minus_one_sample_sums_zero": ([1, -1, 1, 0, 0], 2, [[0, 1]], [1, 0]),
    "ties_first_max_late": ([0, 0, 0.5, 0, 0.5, 0, 0], 3, [[0, 1, 6]], [2, 0, 1]),
    "neg_zero_keep": ([-0.0, 0, -0.0, 0], 2, [[0, 2]], [1, 0]),
    "neg_zero_append": ([-0.0, 0, 1, -0.0], 2, [[0, 3]], [1, 0]),
    "s1_append": ([0, 0, 1, 0], 1, [[0]], [0]),
    "s1_redraw": ([0, 1, 1, 0], 1, [[0], [3], [2]], [0]),
    "s1_keep_zero": ([0, 0, 0], 1, [[2]], [0]),
    "n_eq_s_single": ([0, 1, 0], 3, [[2, 0, 1]], [2, 1, 0]),
    "n_eq_s_negative": ([0, -1, 0], 3, [[1, 2, 0]], [2, 1, 0]),
    "n_eq_s_nan": ([0, NAN, 0, 2], 4, [[3, 1, 0, 2]], [3, 2, 1, 0]),
    "never_relevant_recurses": ([0, 0, 1, 1, 0], 2, [[0, 1]], [1, 0]),
}


class Script:
    def __init__(self, draws, sub):
        self.draws, self.sub, self.calls = [np.asarray(d, dtype=np.int64) for d in draws], np.asarray(sub), 0

    def __call__(self, a, size=None, replace=True, p=None):
        assert replace is False and p is None
        if np.isscalar(a):
            d = self.draws[min(self.calls, len(self.draws) - 1)]
            self.calls += 1
            assert len(d) == size and d.max() < a and len(np.unique(d)) == size
            return d.copy()
        return np.asarray(a)[self.sub[:size]]


def main():
    blob, names = {}, []
    real_choice = np.random.choice
    for name, (labels, S, draws, sub) in CASES.items():
        y = np.asarray(labels, dtype=np.float64)
        assert np.isnan(y.sum()) or float(np.float32(y).sum()) == y.sum(), name
        x = np.arange(len(y), dtype=np.float64)[:, None] * np.ones((1, 2))
        script = Script(draws, sub)
        np.random.choice = script
        try:
            fx, fy, idx = FixLength(S)((x, y, np.arange(len(y))))
            raises = None
            assert np.array_equal(fx[:, 0], idx) and np.array_equal(fy, y[idx], equal_nan=True)
            blob[name + ":idx"] = np.asarray(idx, dtype=np.int64)
        except RecursionError as exc:   # the exception type is part of the reference's behaviour
            raises = type(exc).__name__
        finally:
            np.random.choice = real_choice
        width = max(len(d) for d in draws)
        blob[name + ":y"] = y
        blob[name + ":draws"] = np.array([list(d) + [-1] * (width - len(d)) for d in draws], dtype=np.int64)
        blob[name + ":sub"] = np.asarray(sub, dtype=np.int64)
        blob[name + ":call"] = np.array(json.dumps({"slate_length": S, "raises": raises,
                                                    "draws_made": None if raises else script.calls}))
        names.append(name)
        print(name, raises or (blob[name + ":idx"].tolist(), script.calls))
    blob["names"] = np.array(names)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "slates_rules.npz"), **blob)


if __name__ == "__main__":
    main()
