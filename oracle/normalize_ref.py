"""A restatement of allRank's reproducibility/normalize_features.py for tests and fixtures: the same sklearn and numpy
calls in the same order, with the logarithm as a parameter.

    normalize(ds_path, features_without_logarithm, features_negative, log=np.log)
        -> {"files": {role: bytes}, "stdout": [lines], "mean": [F] float64, "std": [F] float64,
            "inputs": {role: [F_role, rows] float64, after negation}, "logged": [column numbers]}

log=np.log gives the script's bytes on this host; log=log_cr gives the bytes of a correctly rounded logarithm
(mpmath at 256 bits over the column's distinct values), which is what allrank_b200.normalize computes.  Nothing is
written to disk; the output directory is named in stdout as the script names it.
"""
import io
import os

import numpy as np

ROLES = ("train", "test", "vali")


def log_cr(a):
    """log of every element of a float64 array, correctly rounded (round to nearest even) via mpmath."""
    import mpmath
    a = np.asarray(a, np.float64)
    u, inv = np.unique(a, return_inverse=True)
    out = np.empty_like(u)
    with mpmath.workprec(256):
        for k, v in enumerate(u):
            if np.isnan(v) or v < 0:
                out[k] = np.nan
            elif v == 0:
                out[k] = -np.inf
            elif np.isinf(v):
                out[k] = np.inf
            else:
                out[k] = float(mpmath.log(mpmath.mpf(float(v))))   # mpf -> float rounds to nearest even
    return out[inv].reshape(a.shape)


def normalize(ds_path, features_without_logarithm, features_negative, log=np.log):
    from sklearn.datasets import dump_svmlight_file, load_svmlight_file
    loaded = [load_svmlight_file(os.path.join(ds_path, "{}.txt".format(r)), query_id=True) for r in ROLES]
    cols = [x.toarray().T for x, _, _ in loaded]                 # [F_role, rows]: row i is column i
    normalized = [np.zeros(c.shape) for c in cols]
    stdout, means, stds, logged = [], [], [], []
    inputs = [c.copy() for c in cols]
    for i in range(cols[0].shape[0]):
        vecs = [c[i, ] for c in cols]                            # IndexError where a role has fewer columns
        if i in features_negative:
            vecs = [(-1) * v for v in vecs]
            for inp, v in zip(inputs, vecs):
                inp[i, ] = v
        if i not in features_without_logarithm:
            if all(np.all(v >= 0) for v in vecs):
                vecs = [log(v + 1e-2) for v in vecs]
                logged.append(i)
            else:
                stdout.append("Some values of feature no. {} are still < 0 which is why the feature won't be "
                              "normalized".format(i))
        mean, std = np.mean(vecs[0]), np.std(vecs[0])
        means.append(mean)
        stds.append(std)
        for out, v in zip(normalized, vecs):
            out[i, ] = (v - mean) / (std + 1e-6)
    out_dir = "{}_normalized".format(ds_path)
    files = {}
    for r, out, (_, y, qid) in zip(ROLES, normalized, loaded):
        f = io.BytesIO()
        dump_svmlight_file(out.T, y, f, query_id=qid)
        files[r] = f.getvalue()
    stdout.append("Dataset with normalized features saved here: {}.".format(out_dir))
    return {"files": files, "stdout": stdout, "mean": np.array(means, np.float64), "std": np.array(stds, np.float64),
            "inputs": dict(zip(ROLES, inputs)), "logged": logged}
