"""Writes tests/golden/libsvm_small.npz and tests/golden/libsvm_mslr.npz: what sklearn's load_svmlight_file +
SlateStore store for the texts of tests/libsvm_cases.py, so that the GPU tests of the device parser need no sklearn.

    python tools/make_golden_libsvm.py

libsvm_small.npz: per case <name>, the text (<name>.text, uint8), docs_x / docs_y as their float32 bit patterns,
offsets, n_features and longest_query_length.  libsvm_mslr.npz: the seed and row count of the MSLR-shaped text and a
sha256 of each array's bytes instead of the arrays.
"""
import hashlib
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import libsvm_cases as C  # noqa: E402

MSLR_ROWS, MSLR_SEED = 100_000, 1


def small_cases():
    cases = dict(C.LAYOUT_CASES)
    cases["hard_numerals"] = C.hard_text(seed=0)
    return cases


def main():
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)     # float32 overflow of 1e400-like values is the point
        for name, text in small_cases().items():
            r = C.reference_arrays(text)
            out[name + ".text"] = np.frombuffer(text, np.uint8)
            out[name + ".docs_x"] = r["docs_x"].view(np.uint32)
            out[name + ".docs_y"] = r["docs_y"].view(np.uint32)
            out[name + ".offsets"] = r["offsets"]
            out[name + ".meta"] = np.array([r["n_features"], r["longest_query_length"]], np.int64)
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", "libsvm_small.npz"), **out)
        r = C.reference_arrays(C.mslr_text(MSLR_ROWS, seed=MSLR_SEED))
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "libsvm_mslr.npz"),
                        meta=np.array([MSLR_ROWS, MSLR_SEED, r["n_features"], r["longest_query_length"]], np.int64),
                        docs_x_sha=sha(r["docs_x"]), docs_y_sha=sha(r["docs_y"]), offsets_sha=sha(r["offsets"]))


if __name__ == "__main__":
    main()
