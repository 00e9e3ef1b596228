"""The sampling rules of oracle/slates_ref.py against the unmodified reference's FixLength (tests/golden/slates_rules.npz,
tools/make_golden_slates_rules.py): `_sample`, driven by the draws the reference was given, keeps, redraws and appends
exactly as the reference did -- labels summing to 0, below 0 or NaN, fractional sums of 1, -0.0, S = 1 and n == S.
Also pins the host restatement of the kernel's counter hash (HashSource) against a scalar one."""
import builtins
import json
import sys

import numpy as np
import pytest

from oracle import slates_ref


class ScriptedSource:
    """The draws tools/make_golden_slates_rules.py scripted into np.random.choice."""

    def __init__(self, draws, sub, max_attempts=None):
        self.draws = [d[d >= 0] for d in draws]
        self.sub, self.max_attempts, self.calls = sub, max_attempts, 0

    def choice_n(self, n, k, attempt):
        assert attempt == self.calls
        if self.max_attempts is None and attempt >= sys.getrecursionlimit():   # where the reference's recursion ends
            raise RecursionError("maximum recursion depth exceeded")
        self.calls += 1
        d = self.draws[min(attempt, len(self.draws) - 1)]
        assert len(d) == k and d.max() < n
        return d.copy()

    def choice_sub(self, idx, k):
        return np.asarray(idx)[self.sub[:k]]


def cases(golden):
    g = golden("slates_rules")
    for name in g["names"]:
        yield str(name), g, json.loads(str(g[f"{name}:call"]))


def test_the_golden_covers_every_rule(golden):
    names = {n for n, _, _ in cases(golden)}
    assert len(names) >= 25
    for part in ("zero", "single_one_append", "redraw", "minus1", "nan", "frac", "neg_zero", "s1_", "n_eq_s",
                 "recurses"):
        assert any(part in n for n in names), part


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_sample_reproduces_the_reference_under_scripted_draws(golden, dtype):
    for name, g, call in cases(golden):
        y = g[f"{name}:y"].astype(dtype)
        n, S = len(y), call["slate_length"]
        x = np.arange(n, dtype=np.float32)[:, None] * np.ones((1, 3), dtype=np.float32)
        src = ScriptedSource(g[f"{name}:draws"], g[f"{name}:sub"])
        if call["raises"]:
            with pytest.raises(getattr(builtins, call["raises"])):
                slates_ref.fix_length(x, y, S, src)
            continue
        fx, fy, idx = slates_ref.fix_length(x, y, S, src)
        want = g[f"{name}:idx"]
        assert idx.dtype == np.int64 and np.array_equal(idx, want), (name, idx, want)
        assert src.calls == call["draws_made"], name
        assert np.array_equal(fx, x[want]) and np.array_equal(fy, y[want], equal_nan=True), name


def test_the_attempt_cap_keeps_the_last_draw(golden):
    g = golden("slates_rules")
    name = "never_relevant_recurses"
    y = g[f"{name}:y"].astype(np.float32)
    src = ScriptedSource([np.array([0, 4]), np.array([0, 1])], g[f"{name}:sub"], max_attempts=slates_ref.MAX_ATTEMPTS)
    _, fy, idx = slates_ref.fix_length(np.zeros((len(y), 1), np.float32), y, 2, src)
    assert src.calls == slates_ref.MAX_ATTEMPTS == 1024
    assert idx.tolist() == [0, 1] and fy.sum() == 0


def _mix32(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    return h ^ (h >> 16)


def _hash(seed, slate, attempt, item):
    # csrc/slates.cu sample_hash, one item at a time in Python integers
    h = _mix32((seed & 0xFFFFFFFF) ^ ((slate * 0x9E3779B1) & 0xFFFFFFFF))
    h = _mix32(h ^ (seed >> 32) ^ ((attempt * 0x85EBCA6B + 0x7F4A7C15) & 0xFFFFFFFF))
    return _mix32(h ^ ((item * 0xC2B2AE35 + 0x165667B1) & 0xFFFFFFFF))


@pytest.mark.parametrize("seed", [0, 1, 2 ** 32 - 1, 2 ** 32, 0xDEADBEEF12345678, 2 ** 63, 2 ** 64 - 1])
def test_hash_source_restates_the_kernel_hash(seed):
    items = [0, 1, 2, 255, 256, 1250, 16383, 2 ** 31 - 1]
    for slate, attempt in ((0, 0), (1, 0), (69999, 3), (5, 1023)):
        got = slates_ref.sample_hash(seed, slate, attempt, items)
        assert got.tolist() == [_hash(seed, slate, attempt, i) for i in items]
    src = slates_ref.HashSource(seed, 7)
    idx = src.choice_n(300, 40, 2)
    keys = sorted((_hash(seed, 7, 2, i) << 32) | i for i in range(300))
    assert idx.tolist() == [k & 0xFFFFFFFF for k in keys[:40]]
    assert src.choice_sub(idx, 39).tolist() == idx[:39].tolist()


@pytest.mark.parametrize("seed", [0, 12345, 2 ** 64 - 1])
def test_hash_keys_never_tie(seed):
    """For a fixed (seed, slate, attempt) the hash is a bijection of the 32-bit item (mix32 is invertible), so the
    sort keys of one draw are distinct in their high half and the sampled order does not depend on the index in the
    low half: the kernel's sort has no tie to break."""
    for slate, attempt in ((0, 0), (3, 1), (70000, 1023)):
        h = slates_ref.sample_hash(seed, slate, attempt, np.arange(16384))
        assert len(np.unique(h)) == 16384
        idx = slates_ref.HashSource(seed, slate).choice_n(16384, 16384, attempt)
        assert sorted(idx.tolist()) == list(range(16384))
        assert (np.diff(h[idx].astype(np.int64)) > 0).all()
