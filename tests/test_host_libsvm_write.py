"""The device LibSVM writer without a GPU: its "%.16g" formatter (the same __host__ __device__ code the kernels run,
called through arb_format_g16_host) against Python's '%.16g' % v, the refusals the Python layer makes before it
touches a device, the fixtures' recorded rules, and the patch_write bindings."""
import io
import json
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from allrank_b200 import writer
from tests import libsvm_write_cases as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "libsvm_write.npz"))
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "allrank", "rank_and_click.py"))


def _expect(values):
    return [("%.16g" % v).encode() for v in values]


def _mismatches(values):
    got = writer.format_g16(np.asarray(values, np.float64))
    return [(v, g, e) for v, g, e in zip(values, got, _expect(values)) if g != e]


def test_format_matches_python_on_random_bit_patterns():
    rng = np.random.default_rng(20261019)
    f64 = rng.integers(0, 0x7ff0000000000000, 1_000_000, dtype=np.uint64).view(np.float64)
    f32 = rng.integers(0, 0x7f800000, 1_000_000, dtype=np.uint32).view(np.float32).astype(np.float64)
    values = np.concatenate([f64, -f64[:1000], f32, -f32[:1000]]).tolist()
    assert _mismatches(values) == []


def test_format_matches_python_on_hard_values():
    values = C.boundary_values() + C.f32_ties() + C.f64_ties() + C.near_ties()
    values += [-v for v in values] + [float("inf"), float("-inf"), float("nan"), -float("nan")]
    assert _mismatches(values) == []


def test_near_ties_reach_the_exact_path():
    """At least one constructed value lies within 2^-56 of a 16-digit half, where the formatter compares big
    integers; every f32 tie is an exact half."""
    from fractions import Fraction

    def frac(v):
        E = int(("%.20e" % v).split("e")[1])
        x = Fraction(v) * Fraction(10) ** (15 - E)
        return x - x.numerator // x.denominator

    assert any(abs(frac(v) - Fraction(1, 2)) <= Fraction(1, 2 ** 56) for v in C.near_ties())
    assert all(frac(v) == Fraction(1, 2) for v in C.f32_ties())


def test_every_binade_of_float32_around_the_notation_switches():
    """Every float32 of the binades holding 1e-5 and 1e16, on the CPU build of the formatter."""
    values = []
    for p in (-5, 16):
        lo = int(np.array([float("1e%d" % p)], np.float32).view(np.uint32)[0]) & 0xFF800000
        bits = np.arange(lo, lo + (1 << 23), dtype=np.uint32)
        values.append(bits.view(np.float32).astype(np.float64))
    values = np.concatenate(values)
    for k in range(0, len(values), 1 << 20):
        assert _mismatches(values[k:k + (1 << 20)].tolist()) == []


def test_fixture_rules_hold_in_python():
    rules = json.loads(str(GOLD["rules"]))
    assert rules["float_label_neg_zero"] == "-0 1:0.1000000014901161\n1 \n"
    assert rules["qid_empty_row"].endswith("0 qid:-6 \n")
    assert set(rules["refusals"].values()) == {"ValueError"}
    assert str(GOLD["sklearn_version"]).startswith("1.")


@pytest.mark.parametrize("kw, exc", [
    (dict(multilabel=True), NotImplementedError),
    (dict(comment="x"), NotImplementedError),
    (dict(query_id=[1]), ValueError),
    (dict(query_id=[1.5, 2.5]), TypeError),
])
def test_refusals_before_any_device_work(tmp_path, kw, exc):
    path = tmp_path / "out.txt"
    path.write_bytes(b"old")
    with pytest.raises(exc):
        writer.write_svm_file(np.ones((2, 3), np.float32), np.ones(2), str(path), **kw)
    assert path.read_bytes() == b"old"


@pytest.mark.parametrize("X, y, exc", [
    (sp.csr_matrix(np.ones((2, 3))), np.ones(2), NotImplementedError),
    (np.ones((2, 3)), np.ones(3), ValueError),
    (np.ones((2, 3)), np.ones((2, 1)), ValueError),
    (np.ones(3), np.ones(3), ValueError),
    (np.ones((0, 3)), np.ones(0), ValueError),
    (np.ones((2, 0)), np.ones(2), ValueError),
    (np.ones((2, 3), np.uint8), np.ones(2), TypeError),
    (np.ones((2, 3), np.float16), np.ones(2), TypeError),
])
def test_shape_and_dtype_refusals(tmp_path, X, y, exc):
    with pytest.raises(exc):
        writer.write_svm_file(X, y, io.BytesIO())


def test_worst_row_bound_covers_the_longest_tokens():
    longest = max(len(("%.16g" % v).encode()) for v in C.boundary_values() + [-2.2250738585072014e-308])
    assert longest <= writer.FMT_SLOT - 1 and len(str(-2 ** 63)) <= writer.FMT_SLOT
    F = 136
    line = "-1.234567890123457e-308 qid:-9223372036854775808" + "".join(
        " %d:%s" % (j, "-1.234567890123457e-308") for j in range(F)) + "\n"
    assert len(line) <= writer.worst_row_bytes(F, 0)


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
@pytest.mark.parametrize("patch_write", [False, True])
def test_patch_write_bindings(patch_write):
    from oracle.install_reference import import_path
    paths = import_path()
    sys.path[:0] = paths
    try:
        import allrank.data.dataset_saving as ref_ds
        import allrank.rank_and_click as rac
        from allrank_b200 import integration
        before_ds, before_rac = ref_ds.write_to_libsvm_without_masked, rac.write_to_libsvm_without_masked
        saved = integration.patch_allrank(patch_write=patch_write)
        try:
            if patch_write:
                assert ref_ds.write_to_libsvm_without_masked is writer.write_to_libsvm_without_masked
                assert rac.write_to_libsvm_without_masked is writer.write_to_libsvm_without_masked
            else:
                assert ref_ds.write_to_libsvm_without_masked is before_ds
                assert rac.write_to_libsvm_without_masked is before_rac
        finally:
            integration.unpatch_allrank(saved)
        assert ref_ds.write_to_libsvm_without_masked is before_ds
        assert rac.write_to_libsvm_without_masked is before_rac
    finally:
        for p in paths:
            if p in sys.path:
                sys.path.remove(p)
