"""LibSVM folds (train / test / vali texts) for the feature-normalisation tests and tools/make_golden_normalize.py.

FOLDS: name -> (texts {role: bytes}, features_without_logarithm, features_negative).  REFUSALS: name -> (texts, with
a role missing where its text is None, the exception type the script raises first).  mslr_fold(rows) is the
MSLR-shaped generator (136 features) of the large golden fold and of tools/bench_normalize.py.
"""
import numpy as np

ROLES = ("train", "test", "vali")
FEATURES_WITHOUT_LOGARITHM = [5, 6, 7, 8, 9, 15, 19, 57, 58, 62, 75, 79, 85, 95, 96, 97, 98, 99, 100, 101, 102, 103,
                              104, 121, 122, 127, 129, 130]
FEATURES_NEGATIVE = [110, 111, 112, 113, 114, 115, 116, 117, 118, 119, 120, 123, 124]


def _text(X, y, qid, one_based=True):
    """Rows "label qid:Q j:v ..." with the non-zero values of X (and explicit zeros where X holds -0.0)."""
    lines = []
    for row, lab, q in zip(X, y, qid):
        toks = ["{:g}".format(lab), "qid:{}".format(int(q))]
        for j, v in enumerate(row):
            if v != 0 or np.signbit(v):
                toks.append("{}:{}".format(j + one_based, "-0" if v == 0 else repr(float(v))))
        lines.append(" ".join(toks))
    return ("\n".join(lines) + "\n").encode()


def _mslr_matrix(rng, rows):
    """136 MSLR-like columns: counts, 6-digit decimals, the FEATURES_NEGATIVE columns mostly negative (a few
    positive values, so some stay < 0 after negation), column 3 of mixed sign, column 4 constant."""
    X = np.zeros((rows, 136))
    for j in range(136):
        kind = j % 3
        if kind == 0:
            X[:, j] = rng.poisson(3.0, rows) * (rng.random(rows) < 0.7)
        elif kind == 1:
            X[:, j] = np.round(rng.random(rows) * 10 ** rng.integers(0, 4), 6)
        else:
            X[:, j] = np.round(rng.exponential(50.0, rows), 6)
    for j in FEATURES_NEGATIVE:
        X[:, j] = -np.round(rng.random(rows) * 30, 6)
        if j % 2:
            X[rng.integers(0, rows, 2), j] = 1.5
    X[:, 3] = np.round(rng.standard_normal(rows), 6)
    X[:, 4] = 7.0
    return X


def mslr_fold(rows, seed=0):
    """(texts, features_without_logarithm, features_negative): train of `rows` rows, test and vali a third each."""
    rng = np.random.default_rng(seed)
    texts = {}
    for k, role in enumerate(ROLES):
        n = rows if role == "train" else max(1, rows // 3)
        X = _mslr_matrix(rng, n)
        y = rng.integers(0, 5, n).astype(float)
        qid = np.repeat(np.arange(n // 20 + 1) + 1000 * k, 20)[:n]
        texts[role] = _text(X, y, qid)
    return texts, FEATURES_WITHOUT_LOGARITHM, FEATURES_NEGATIVE


def near_one_values():
    """Values v whose fl(v + 0.01) is 1 + k 2^-52, 1 - k 2^-52 or 1 - k 2^-53 for small k: logarithms within a tiny
    fraction of an ulp of a rounding midpoint, which need the accurate phase."""
    out = []
    for k in range(1, 40):
        for target in (1 + k * 2.0 ** -52, 1 - k * 2.0 ** -52, 1 - k * 2.0 ** -53):
            v = target - 0.01
            for _ in range(8):
                s = v + 0.01
                if s == target:
                    out.append(v)
                    break
                v = np.nextafter(v, np.inf if s < target else -np.inf)
    return np.array(out)


def _small(seed, rows=(40, 15, 12), F=(8, 8, 8), one_based=(True, True, True)):
    rng = np.random.default_rng(seed)
    texts, mats = {}, []
    for k, role in enumerate(ROLES):
        X = np.round(rng.random((rows[k], F[k])) * 20, 6)
        X[rng.random(X.shape) < 0.3] = 0.0
        mats.append(X)
    return rng, mats, one_based


def _emit(rng, mats, one_based):
    texts = {}
    for k, (role, X) in enumerate(zip(ROLES, mats)):
        n = X.shape[0]
        y = rng.integers(0, 5, n).astype(float)
        texts[role] = _text(X, y, np.repeat(np.arange(n // 4 + 1), 4)[:n], one_based=one_based[k])
    return texts


def _folds():
    folds = {}
    rng, mats, ob = _small(1)
    mats[0][:, 2] = -mats[0][:, 2]                        # negated back to >= 0
    mats[1][:, 2] = -mats[1][:, 2]
    mats[2][:, 2] = -mats[2][:, 2]
    mats[0][3, 5] = -1.0                                  # mixed sign: message, not logged
    mats[0][:, 6] = 2.5                                   # constant: std 0
    folds["basic"] = (_emit(rng, mats, ob), [0], [2])

    rng, mats, ob = _small(2, rows=(30, 10, 10), F=(4, 4, 4))
    near = near_one_values()
    for X in mats:
        X[:, 1] = near[rng.integers(0, len(near), X.shape[0])]
        X[:, 3] = near[rng.integers(0, len(near), X.shape[0])]
    folds["near_one"] = (_emit(rng, mats, ob), [], [])

    rng, mats, ob = _small(3, F=(6, 6, 6), one_based=(True, False, True))   # test alone has "0:" tokens
    folds["per_file_shift"] = (_emit(rng, mats, ob), [], [])

    rng, mats, ob = _small(4, F=(5, 9, 7))
    folds["wider_test_vali"] = (_emit(rng, mats, ob), [1], [])

    rng, mats, ob = _small(5, F=(5, 5, 5))
    for X in mats:
        X[::3, 1] = -0.0
        X[::4, 2] = -0.0
    folds["negative_zero"] = (_emit(rng, mats, ob), [], [2])

    texts, fwl, fneg = mslr_fold(120, seed=6)
    folds["mslr_small"] = (texts, fwl, fneg)
    return folds


FOLDS = _folds()
LARGE_ROWS = 20000          # the MSLR-shaped fold whose bytes are kept as sha256 and length


def _refusals():
    good = FOLDS["basic"][0]
    r = {}
    r["missing_vali"] = (dict(good, vali=None), FileNotFoundError)
    r["bad_test_value"] = (dict(good, test=b"1 qid:1 1:abc\n"), ValueError)
    r["test_index_overflow"] = (dict(good, test=b"1 qid:1 99999999999:1\n"), OverflowError)
    r["narrow_vali"] = (dict(good, vali=b"1 qid:1 1:0.5 3:1\n"), IndexError)
    r["nan_train"] = (dict(good, train=good["train"] + b"1 qid:77 1:nan\n"), ValueError)
    r["inf_test"] = (dict(good, test=good["test"] + b"1 qid:77 2:inf\n"), ValueError)
    r["empty_test"] = (dict(good, test=b""), IndexError)                 # shape (0, 1): narrower than train
    r["empty_train"] = (dict(good, train=b""), ValueError)
    r["missing_qid_vali"] = (dict(good, vali=good["vali"] + b"1 1:0.5\n"), ValueError)
    return r


REFUSALS = _refusals()


def write_fold(texts, path):
    import os
    os.makedirs(path, exist_ok=True)
    for role in ROLES:
        if texts.get(role) is not None:
            with open(os.path.join(path, "{}.txt".format(role)), "wb") as f:
                f.write(texts[role])
