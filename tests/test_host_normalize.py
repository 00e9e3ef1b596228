"""The feature normalisation's host-side pieces without a GPU: the correctly rounded log (csrc/log_cr.cuh, the same
code the kernels run) against mpmath, the pairwise summation against np.add.reduce, the command line against the
script's, and refusals made before any device work."""
import os

import mpmath
import numpy as np
import pytest

from allrank_b200 import normalize as N
from tests import normalize_cases as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "normalize.npz"))


def _mp_log(values, prec=200):
    out = np.empty(len(values))
    with mpmath.workprec(prec):
        for k, v in enumerate(values):
            out[k] = float(mpmath.log(mpmath.mpf(float(v))))
    return out


def _values(seed=0):
    """~10^6 positive finite doubles: random bit patterns over the whole range (subnormals included), v + 0.01 of
    6-digit decimals, near-1 families and powers of two."""
    rng = np.random.default_rng(seed)
    bits = rng.integers(1, 0x7ff0000000000000, 700_000, dtype=np.int64).view(np.float64)
    sub = rng.integers(1, 1 << 52, 20_000, dtype=np.int64).view(np.float64)
    dec = np.round(rng.random(400_000) * 10.0 ** rng.integers(-3, 6, 400_000), 6) + 0.01
    k = np.arange(1, 2000, dtype=np.float64)
    near = np.concatenate([1 + k * 2.0 ** -52, 1 - k * 2.0 ** -53, 1 - k * 2.0 ** -52, C.near_one_values() + 0.01])
    pow2 = 2.0 ** np.arange(-1074, 1024, dtype=np.float64)
    return np.unique(np.concatenate([bits, sub, dec, near, pow2, [np.finfo(float).max, 0.01]]))


@pytest.fixture(scope="module")
def values_and_reference():
    v = _values()
    return v, _mp_log(v)


@pytest.mark.parametrize("force_accurate", [False, True])
def test_log_cr_host_against_mpmath(values_and_reference, force_accurate):
    v, ref = values_and_reference
    assert v.size >= 10 ** 6
    y, n_accurate = N.log_cr(v, force_accurate)
    bad = np.nonzero(y.view(np.int64) != ref.view(np.int64))[0]
    assert bad.size == 0, [(float(v[i]), float(y[i]), float(ref[i])) for i in bad[:5]]
    if force_accurate:
        assert n_accurate == v.size - int((v == 1.0).sum())      # log(1) = +0 needs neither phase
    else:
        assert 0 < n_accurate < v.size // 1000


def _midpoint_distance_ulps(x):
    """Distance of log(x) from the nearest rounding midpoint beside its rounding, in ulps of the result."""
    with mpmath.workprec(300):
        t = mpmath.log(mpmath.mpf(float(x)))
        r = float(t)
        half = mpmath.mpf(float(np.spacing(abs(r)))) / 2
        return float(min(abs(t - (r + half)), abs(t - (r - half))) / (2 * half))


def test_near_one_takes_the_accurate_phase():
    """1 - 2 * 2^-53 and its neighbours lie ~1e-16 ulp from a midpoint: no double-double result can decide them."""
    k = np.arange(1, 20, dtype=np.float64)
    xs = np.concatenate([1 - k * 2.0 ** -53, 1 + k * 2.0 ** -52, 1 - k * 2.0 ** -52])
    hard = np.array([x for x in xs if _midpoint_distance_ulps(x) < 2.0 ** -40])
    assert 1 - 2 * 2.0 ** -53 in hard
    for x in hard:
        y, n_accurate = N.log_cr(np.array([x]))
        assert n_accurate == 1, x
        assert y[0] == _mp_log([x])[0]


def test_log_cr_special_values():
    x = np.array([0.0, -0.0, -1.0, -np.inf, np.nan, np.inf, 1.0, 5e-324])
    y, _ = N.log_cr(x)
    assert y[0] == -np.inf and y[1] == -np.inf
    assert np.isnan(y[2]) and np.isnan(y[3]) and np.isnan(y[4])
    assert y[5] == np.inf and y[6] == 0.0 and not np.signbit(y[6])
    assert y[7] == _mp_log([5e-324])[0]


def test_pairwise_sum_small_n_signed_zero_and_start():
    rng = np.random.default_rng(1)
    for n in range(0, 301):
        for a in (np.full(n, -0.0), rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n),
                  np.where(rng.random(n) < 0.5, -0.0, 0.0)):
            got, ref = N.pairwise_sum_host(a), np.add.reduce(a)
            assert got.tobytes() == ref.tobytes(), (n, got, ref)


@pytest.mark.parametrize("n", [1000, 9000, 50_000, 100_001])
def test_pairwise_sum_large_strided_and_contiguous(n):
    rng = np.random.default_rng(n)
    m = rng.standard_normal((n, 7)) * 10.0 ** rng.integers(-6, 6, (n, 7))
    for a in (m[:, 3], np.ascontiguousarray(m[:, 3]), m.reshape(-1)[:n]):
        assert N.pairwise_sum_host(a).tobytes() == np.add.reduce(a).tobytes()
        assert (N.pairwise_sum_host(a) / n).tobytes() == np.mean(a).tobytes()


def test_pairwise_plan_covers_numpys_tree():
    for n in (1, 7, 8, 128, 129, 1000, 100_001):
        leaf_start, children, levels = N.pairwise_plan(n)
        lens = np.diff(leaf_start)
        assert leaf_start[0] == 0 and leaf_start[-1] == n and (lens > 0).all() and (lens <= 128).all()
        assert n < 8 or (lens >= 8).all()
        assert children.shape[0] == len(lens) - 1 == levels.sum()


def test_command_line_matches_the_script():
    p = N.parser()
    a = p.parse_args(["--ds_path", "x"])
    assert a.ds_path == "x"
    assert a.features_without_logarithm == C.FEATURES_WITHOUT_LOGARITHM == N.FEATURES_WITHOUT_LOGARITHM
    assert a.features_negative == C.FEATURES_NEGATIVE == N.FEATURES_NEGATIVE
    a = p.parse_args(["--ds_path", "y/", "--features_without_logarithm", "--features_negative", "1", "2"])
    assert a.features_without_logarithm == [] and a.features_negative == [1, 2]
    assert p.prog == "Normalize features script"
    with pytest.raises(SystemExit):
        p.parse_args([])
    with pytest.raises(SystemExit):
        p.parse_args(["--ds_path", "x", "--features_negative", "a"])


def test_missing_file_refused_before_device_work(tmp_path):
    texts, exc = C.REFUSALS["missing_vali"]
    C.write_fold(dict(texts, train=None), str(tmp_path / "fold"))
    with pytest.raises(FileNotFoundError):
        N.normalize_features(str(tmp_path / "fold"), device="cuda:0")
    assert not os.path.exists(str(tmp_path / "fold") + "_normalized")


def test_fixture_stdout_names_the_script_lines():
    out = bytes(GOLD["basic/stdout"]).decode().splitlines()
    assert out[0] == N.unlogged_message(5)
    assert out[-1] == "Dataset with normalized features saved here: {dir}_normalized."
