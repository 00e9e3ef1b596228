"""Writes tests/golden/normalize.npz for the feature-normalisation tests, asserting two things as it goes:

  1. oracle/normalize_ref.py with np.log writes the unmodified reproducibility/normalize_features.py's bytes (run from
     $ALLRANK_REFERENCE, default /root/reference) on every fold of tests/normalize_cases.py, prints its lines and
     raises its exception type on every refusal, so the restatement is the script;
  2. every byte that differs between the oracle with np.log and with a correctly rounded log lies in a logged
     column holding a value whose np.log is not correctly rounded on this host.

    python tools/make_golden_normalize.py

Keys per fold <f>: <f>/<role> (uint8: the correctly rounded bytes), <f>/stdout (the script's lines, with "{dir}" for
the fold path), <f>/mean and <f>/std (int64 bit patterns), <f>/nolog/<role> (the script's bytes with every column in
--features_without_logarithm).  The large MSLR-shaped fold keeps sha256 and length only: large/<role>/sha256 and
large/<role>/len.  Float64 parser arrays: parse/<case>/x, /y (int64 bits of load_svmlight_file(...).toarray() and y)
and /text for the hard and layout texts of tests/libsvm_cases.py.
"""
import hashlib
import io
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import normalize_ref as R  # noqa: E402
from tests import libsvm_cases as LC  # noqa: E402
from tests import normalize_cases as C  # noqa: E402

SCRIPT = os.path.join(os.environ.get("ALLRANK_REFERENCE", "/root/reference"), "reproducibility",
                      "normalize_features.py")


def run_script(fold, fwl, fneg):
    """(files {role: bytes} or None, stdout lines, exception type name or None) of the unmodified script."""
    args = [sys.executable, SCRIPT, "--ds_path", fold, "--features_without_logarithm", *map(str, fwl),
            "--features_negative", *map(str, fneg)]
    r = subprocess.run(args, capture_output=True, text=True)
    err = None
    if r.returncode:
        err = r.stderr.strip().splitlines()[-1].split(":")[0]
    files = None
    out_dir = fold + "_normalized"
    if not r.returncode:
        files = {role: open(os.path.join(out_dir, role + ".txt"), "rb").read() for role in C.ROLES}
    shutil.rmtree(out_dir, ignore_errors=True)
    return files, r.stdout.splitlines(), err


def check_differences(a, b):
    """Assertion 2: columns whose normalised bytes differ are logged, with an input np.log rounds wrongly."""
    from sklearn.datasets import load_svmlight_file
    for role in C.ROLES:
        if a["files"][role] == b["files"][role]:
            continue
        xa = load_svmlight_file(io.BytesIO(a["files"][role]), zero_based=True)[0].toarray()
        xb = load_svmlight_file(io.BytesIO(b["files"][role]), zero_based=True)[0].toarray()
        assert xa.shape == xb.shape
        for col in np.nonzero((xa != xb).any(axis=0))[0]:
            assert col in a["logged"], (role, col)
            vals = np.concatenate([a["inputs"][r][col] for r in C.ROLES if col < a["inputs"][r].shape[0]]) + 1e-2
            assert (np.log(vals).view(np.int64) != R.log_cr(vals).view(np.int64)).any(), (role, col)


def main():
    out = {}
    tmp = tempfile.mkdtemp()
    folds = dict(C.FOLDS)
    folds["large"] = C.mslr_fold(C.LARGE_ROWS, seed=11)
    for name, (texts, fwl, fneg) in folds.items():
        fold = os.path.join(tmp, name)
        C.write_fold(texts, fold)
        files, stdout, err = run_script(fold, fwl, fneg)
        assert err is None, (name, err)
        a = R.normalize(fold, fwl, fneg, log=np.log)
        assert a["files"] == files, name                                          # assertion 1
        assert a["stdout"] == stdout, name
        b = R.normalize(fold, fwl, fneg, log=R.log_cr)
        check_differences(a, b)                                                   # assertion 2
        stdout_t = "\n".join(stdout).replace(fold, "{dir}").encode()
        if name == "large":
            for role in C.ROLES:
                out["large/{}/sha256".format(role)] = np.frombuffer(
                    hashlib.sha256(b["files"][role]).digest(), np.uint8)
                out["large/{}/len".format(role)] = np.array(len(b["files"][role]), np.int64)
            out["large/stdout"] = np.frombuffer(stdout_t, np.uint8)
            continue
        for role in C.ROLES:
            out["{}/{}".format(name, role)] = np.frombuffer(b["files"][role], np.uint8)
        out[name + "/stdout"] = np.frombuffer(stdout_t, np.uint8)
        out[name + "/mean"] = b["mean"].view(np.int64)
        out[name + "/std"] = b["std"].view(np.int64)
        every = list(range(200))
        nolog, _, err = run_script(fold, every, fneg)
        assert err is None and nolog == R.normalize(fold, every, fneg)["files"], name
        for role in C.ROLES:
            out["{}/nolog/{}".format(name, role)] = np.frombuffer(nolog[role], np.uint8)
    for name, (texts, exc) in C.REFUSALS.items():
        fold = os.path.join(tmp, "refusal_" + name)
        C.write_fold(texts, fold)
        _, _, err = run_script(fold, [], [])
        assert err == exc.__name__, (name, err, exc)
        try:
            R.normalize(fold, [], [])
            raise AssertionError(name)
        except exc:
            pass
    from sklearn.datasets import load_svmlight_file
    parse_cases = dict(("layout_" + k, v) for k, v in LC.LAYOUT_CASES.items())
    parse_cases["hard"] = LC.hard_text()
    for name, text in parse_cases.items():
        X, y, _ = load_svmlight_file(io.BytesIO(text), query_id=True)
        out["parse/{}/text".format(name)] = np.frombuffer(text, np.uint8)
        out["parse/{}/x".format(name)] = X.toarray().view(np.int64)
        out["parse/{}/y".format(name)] = np.asarray(y, np.float64).view(np.int64)
    shutil.rmtree(tmp)
    path = os.path.join(ROOT, "tests", "golden", "normalize.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
