"""Writes tests/golden/libsvm_write.npz: the bytes sklearn's dump_svmlight_file writes for the cases of
tests/libsvm_write_cases.py, and the bytes the unmodified reference's write_to_libsvm_without_masked writes for its
ragged slates, so that the GPU tests of the device writer need no sklearn.

    python tools/make_golden_libsvm_write.py    # reference source from $ALLRANK_REFERENCE (default /root/reference)

Per small case <name>: <name>.bytes (uint8, the whole file).  The MSLR-shaped block (20 000 rows) keeps its sha256
and length only.  "rules" records each rule of the output format as sklearn applies it here, checked as it runs.
"""
import hashlib
import io
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import libsvm_write_cases as C  # noqa: E402


def dump(X, y, qid=None, zero_based=True):
    from sklearn.datasets import dump_svmlight_file
    f = io.BytesIO()
    dump_svmlight_file(X, y, f, zero_based=zero_based, query_id=qid)
    return f.getvalue()


def raises(fn):
    try:
        fn()
    except Exception as e:                  # noqa: BLE001  (the type is what is recorded)
        return type(e).__name__
    return None


def rules():
    """What the contract says, as sklearn does it; each assertion is a rule the device writer follows."""
    X = np.array([[0, 0.1, -0.0], [0, 0, 0]], np.float32)
    r = {}
    r["float_label_neg_zero"] = dump(X, np.array([-0.0, 1.0])).decode()
    assert r["float_label_neg_zero"] == "-0 1:0.1000000014901161\n1 \n"
    r["int_label"] = dump(X, np.array([3, -2])).decode()
    assert r["int_label"] == "3 1:0.1000000014901161\n-2 \n"
    r["qid_empty_row"] = dump(X, np.array([1.0, 0.0]), qid=np.array([5, -6])).decode()
    assert r["qid_empty_row"] == "1 qid:5 1:0.1000000014901161\n0 qid:-6 \n"
    r["one_based"] = dump(X, np.array([1.0, 0.0]), zero_based=False).decode()
    assert r["one_based"] == "1 2:0.1000000014901161\n0 \n"
    r["int_x"] = dump(np.array([[0, 7, -(2 ** 63)]]), np.array([1.5])).decode()
    assert r["int_x"] == "1.5 1:7 2:-9223372036854775808\n"
    for v, s in ((9.99994610111476e-41, "9.99994610111476e-41"), (3.000000005497756e+38, "3.000000005497756e+38"),
                 (1.000000011686097e-07, "1.000000011686097e-07"), (2.0, "2"), (1.5, "1.5"),
                 (float(np.float32(999.99993896484375)), "999.9999389648438")):
        assert dump(np.array([[v]]), np.array([0])).decode() == "0 0:%s\n" % s, v
    refusals = {
        "nan_x": raises(lambda: dump(np.array([[np.nan]]), np.array([1.0]))),
        "inf_x": raises(lambda: dump(np.array([[np.inf]]), np.array([1.0]))),
        "nan_y": raises(lambda: dump(np.array([[1.0]]), np.array([np.nan]))),
        "inf_y": raises(lambda: dump(np.array([[1.0]]), np.array([-np.inf]))),
        "y_length": raises(lambda: dump(np.ones((2, 1)), np.array([1.0]))),
        "qid_length": raises(lambda: dump(np.ones((2, 1)), np.ones(2), qid=np.array([1]))),
        "no_rows": raises(lambda: dump(np.ones((0, 1)), np.ones(0))),
    }
    assert all(v == "ValueError" for v in refusals.values()), refusals
    r["refusals"] = refusals
    return r


def reference_ragged():
    """The unmodified reference's write_to_libsvm_without_masked on tests/libsvm_write_cases.ragged_slates()."""
    import tempfile
    sys.path[:0] = [os.path.join(ROOT, "oracle", "_stubs"), os.environ.get("ALLRANK_REFERENCE", "/root/reference")]
    from allrank.data.dataset_saving import write_to_libsvm_without_masked
    Xs, ys = C.ragged_slates()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "ragged.txt")
        write_to_libsvm_without_masked(path, Xs, ys)
        with open(path, "rb") as fh:
            return fh.read()


def main():
    import sklearn
    out = {}
    cases = C.small_cases()
    for name, c in cases.items():
        out[name + ".bytes"] = np.frombuffer(dump(c["X"], c["y"], c["qid"], c["zero_based"]), np.uint8)
    X, y, qid = C.mslr_block()
    text = dump(X, y, qid)
    out["mslr.sha256"] = np.array(hashlib.sha256(text).hexdigest())
    out["mslr.length"] = np.array(len(text), np.int64)
    out["ragged.bytes"] = np.frombuffer(reference_ragged(), np.uint8)
    out["rules"] = np.array(json.dumps(rules()))
    out["sklearn_version"] = np.array(sklearn.__version__)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "libsvm_write.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
