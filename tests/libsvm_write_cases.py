"""Inputs of the device LibSVM writer's tests (allrank_b200/writer.py): dense X / y / qid cases built from fixed
seeds, so that tools/make_golden_libsvm_write.py (run with sklearn) and the GPU tests (run without it) build the same
arrays, and the values whose "%.16g" is hard to get right."""
from fractions import Fraction

import numpy as np

F32_MAX = float(np.finfo(np.float32).max)
F32_TINY = float(np.finfo(np.float32).tiny)
F32_SUB = float(np.float32(1e-45))
DBL_MAX = float(np.finfo(np.float64).max)


def f32_ties(k_values=range(0, 25), per_k=12, seed=0):
    """float32 m * 2^-k (m odd) whose m * 5^k has 17 digits: exact ties at 16 digits, e.g. 999.99993896484375."""
    rng = np.random.default_rng(seed)
    out = [999.99993896484375]
    for k in k_values:
        lo, hi = -(-10 ** 16 // 5 ** k), (10 ** 17 - 1) // 5 ** k
        lo, hi = max(lo, 1 << 23), min(hi, (1 << 24) - 1)
        if lo > hi:
            continue
        for m in rng.integers(lo, hi + 1, per_k).tolist():
            m |= 1
            if m <= hi:
                out.append(float(np.float32(m * 2.0 ** -k)))
    return out


def f64_ties(k_values=range(0, 25), per_k=12, seed=1):
    """float64 m * 2^-k (m odd, m < 2^53) whose m * 5^k has 17 digits: exact 16-digit ties."""
    rng = np.random.default_rng(seed)
    out = []
    for k in k_values:
        lo, hi = -(-10 ** 16 // 5 ** k), min((10 ** 17 - 1) // 5 ** k, (1 << 53) - 1)
        if lo > hi:
            continue
        for m in rng.integers(lo, hi + 1, per_k).tolist():
            m |= 1
            if m <= hi:
                out.append(m * 2.0 ** -k)
    return out


def near_ties(qs=range(-30, -23), tol_bits=50):
    """Doubles v >= 1e16 whose v * 10^q lies within 2^-tol_bits of a half-integer (q = 15 - the decimal exponent):
    m * 2^j = delta (mod 5^-q), j = e + q + 1, |delta| < 5^-q * 2^(1 - tol_bits).  Those within 2^-56 reach the
    formatter's exact path."""
    out = []
    for q in qs:
        M = 5 ** -q
        E = 15 - q
        lim = max(1, M >> (tol_bits - 1))
        e0 = int(E * 3.321928) - 54
        for e in range(e0 - 2, e0 + 8):
            j = e + q + 1
            if j < 1:
                continue
            inv = pow(2 ** j, -1, M)
            for d in range(-lim, lim + 1, 2):
                m = ((d | 1) * inv) % M
                if (1 << 52) <= m < (1 << 53):
                    v = m * Fraction(2) ** e
                    if 10 ** E <= v < 10 ** (E + 1):
                        out.append(float(v))
    return out


def boundary_values():
    """Doubles and float32s either side of 1e-5, 1e-4, 1e15 and 1e16 (where the notation and E change), of every
    power of ten, and the extremes."""
    out = [0.0, -0.0, 1.0, -1.0, 2.0, 1.5, 0.1, float(np.float32(0.1)), 5e-324, -5e-324, DBL_MAX, -DBL_MAX, F32_MAX,
           F32_TINY, F32_SUB, 2.2250738585072014e-308, 2.225073858507201e-308, 9.99994610111476e-41,
           3.000000005497756e+38, 1.000000011686097e-07]
    for p in range(-324, 309):
        try:
            v = float("1e%d" % p)
        except OverflowError:
            continue
        if v == 0.0:
            continue
        out += [v, np.nextafter(v, 0.0), np.nextafter(v, np.inf)]
        for c in ("9.9999999999999995e%d", "9.99999999999999949e%d", "9.99999999999999951e%d"):
            w = float(c % p)
            if np.isfinite(w):
                out += [w, np.nextafter(w, 0.0), np.nextafter(w, np.inf)]
    for p in (-5, -4, 15, 16, 38, -38):
        bits = int(np.array([float("1e%d" % p)], np.float32).view(np.int32)[0])
        for k in range(-8, 9):
            out.append(float(np.array([bits + k], np.int32).view(np.float32)[0]))
    return [float(x) for x in out if np.isfinite(x)]


def mslr_block(n_rows=20_000, seed=5, n_features=136):
    """An MSLR-WEB30K-shaped click-through role: float32 features, ~40 % zeros, MSLR-like magnitudes; 0/1 float32
    labels; qids in runs of 1 to 240 rows."""
    rng = np.random.default_rng(seed)
    X = np.empty((n_rows, n_features), np.float32)
    kinds = rng.integers(0, 4, n_features)
    for j in range(n_features):
        if kinds[j] == 0:
            col = rng.integers(0, 40, n_rows).astype(np.float32)
        elif kinds[j] == 1:
            col = rng.random(n_rows).astype(np.float32)
        elif kinds[j] == 2:
            col = (rng.standard_normal(n_rows) * 1e3).astype(np.float32)
        else:
            col = rng.integers(0, 65536, n_rows).astype(np.float32) * np.float32(2.0 ** -int(rng.integers(0, 20)))
        col[rng.random(n_rows) < 0.4] = 0
        X[:, j] = col
    y = (rng.random(n_rows) < 0.1).astype(np.float32)
    runs = rng.integers(1, 241, n_rows)
    qid = np.repeat(np.arange(n_rows), runs)[:n_rows].astype(np.int64)
    return X, y, qid


def small_cases():
    """name -> dict(X, y, qid or None, zero_based): every rule of the output format."""
    rng = np.random.default_rng(11)
    c = {}
    Xf = np.array([[0, 1.5, -0.0, 0.1], [0, 0, 0, 0], [-0.0, 0, 0, 0], [1e-5, 9.9999e-5, 1e15, 1e16]], np.float32)
    c["f32_basic"] = dict(X=Xf, y=np.array([-0.0, 1.0, 2.5, 0.0]), qid=None, zero_based=True)
    c["f32_qid"] = dict(X=Xf, y=np.array([-0.0, 1.0, 2.5, 0.0], np.float32), qid=np.array([3, 3, -4, 2 ** 62]),
                        zero_based=True)
    c["f32_one_based"] = dict(X=Xf, y=np.array([1, 2, 3, 4]), qid=np.array([1, 1, 2, 2], np.int32), zero_based=False)
    c["f64_basic"] = dict(X=Xf.astype(np.float64) * np.pi, y=np.array([1, 0, -3, 2 ** 62]), qid=None, zero_based=True)
    Xi = rng.integers(-5, 6, (9, 7)).astype(np.int64)
    Xi[0, 0], Xi[1, 1], Xi[2] = 2 ** 63 - 1, -2 ** 63, 0
    c["i64_int_y"] = dict(X=Xi, y=rng.integers(-3, 5, 9), qid=np.arange(9), zero_based=True)
    c["i64_float_y"] = dict(X=Xi, y=rng.standard_normal(9), qid=None, zero_based=False)
    c["i32_x"] = dict(X=Xi.astype(np.int32) // 3, y=np.arange(9, dtype=np.float32) / 3, qid=None, zero_based=True)
    ext = np.array(boundary_values())
    pad = (-len(ext)) % 8
    Xe = np.concatenate([ext, np.zeros(pad)]).reshape(-1, 8)
    c["f64_boundaries"] = dict(X=Xe, y=Xe[:, 0].copy(), qid=np.arange(len(Xe)) // 3, zero_based=True)
    e32 = ext[(np.abs(ext) <= F32_MAX) & ((np.abs(ext) >= F32_SUB) | (ext == 0))].astype(np.float32)
    pad = (-len(e32)) % 8
    X32 = np.concatenate([e32, np.zeros(pad, np.float32)]).reshape(-1, 8)
    c["f32_boundaries"] = dict(X=X32, y=X32[:, 1].copy(), qid=None, zero_based=True)
    sub = np.array([np.float32(k * 2.0 ** -149) for k in (1, 2, 3, 7, 1000, 2 ** 22, 2 ** 23 - 1)] +
                   [np.float32(F32_TINY), np.float32(F32_MAX), np.float32(-F32_MAX)], np.float32)
    c["f32_extremes"] = dict(X=sub.reshape(2, 5), y=np.array([F32_MAX, -F32_SUB], np.float32), qid=None,
                             zero_based=True)
    t32 = np.array(f32_ties(), np.float32)
    pad = (-len(t32)) % 10
    T32 = np.concatenate([t32, np.zeros(pad, np.float32)]).reshape(-1, 10)
    c["f32_ties"] = dict(X=T32, y=T32[:, 2].copy(), qid=None, zero_based=True)
    t64 = np.array(f64_ties() + near_ties())
    pad = (-len(t64)) % 10
    T64 = np.concatenate([t64, np.zeros(pad)]).reshape(-1, 10)
    c["f64_ties"] = dict(X=T64, y=T64[:, 3].copy(), qid=np.arange(len(T64)), zero_based=False)
    return c


def ragged_slates(seed=7, n_features=5):
    """(X, y) lists of padded slates for write_to_libsvm_without_masked: ragged lengths, -1 padding in the middle and
    at the end, an all-padding slate and a one-item slate."""
    rng = np.random.default_rng(seed)
    Xs, ys = [], []
    for n in (4, 7, 3, 1, 6, 5):
        x = (rng.standard_normal((n, n_features)) * rng.choice([1e-3, 1, 1e6], (n, n_features))).astype(np.float32)
        x[rng.random((n, n_features)) < 0.3] = 0
        y = rng.integers(0, 2, n).astype(np.float32)
        Xs.append(x)
        ys.append(y)
    ys[1][[2, 5, 6]] = -1
    ys[2][:] = -1                        # all padding: its qid is still counted
    ys[4][-2:] = -1
    return Xs, ys
