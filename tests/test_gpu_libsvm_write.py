"""The device LibSVM writer (allrank_b200/writer.py, csrc/libsvm_write.cu) on the GPU: the "%.16g" kernel against
Python byte for byte, files against the sklearn fixtures of tests/golden/libsvm_write.npz (built by
tools/make_golden_libsvm_write.py) at several chunk sizes, refusals, a round trip through the device parser, and
`rank_and_click.run()` with the writer patched in."""
import hashlib
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from allrank_b200 import _lib, data, writer
from tests import libsvm_write_cases as C

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "libsvm_write.npz"))
CASES = C.small_cases()
DEV = torch.device("cuda:0")
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "allrank", "rank_and_click.py"))


def _check_format(values):
    """arb_format_g16 on the device against '%.16g' % v, for a float64 array."""
    values = np.ascontiguousarray(values, np.float64)
    for k in range(0, len(values), 1 << 22):
        part = values[k:k + (1 << 22)]
        got = np.array(writer.format_g16(torch.from_numpy(part).to(DEV)), dtype="S24")
        want = np.array([("%.16g" % v).encode() for v in part.tolist()], dtype="S24")
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, [(part[i], got[i], want[i]) for i in bad[:5]]


def _binade(p):
    lo = int(np.array([p], np.float32).view(np.uint32)[0]) & 0xFF800000
    return np.arange(lo, lo + (1 << 23), dtype=np.uint32).view(np.float32).astype(np.float64)


@pytest.mark.parametrize("where", ["1e-5", "1e-4", "1", "1e15", "1e16", "1e38", "subnormal", "largest"])
def test_format_every_float32_of_a_binade(where):
    if where == "subnormal":
        values = np.arange(1, 1 << 23, dtype=np.uint32).view(np.float32).astype(np.float64)
    elif where == "largest":
        values = np.arange(0x7F000000, 0x7F800000, dtype=np.uint32).view(np.float32).astype(np.float64)
    else:
        values = _binade(float(where))
    _check_format(values)


def test_format_random_bit_patterns():
    rng = np.random.default_rng(7)
    f32 = rng.integers(0, 0xFF800000, 20_000_000, dtype=np.uint32)
    f32 = f32[(f32 & 0x7F800000) != 0x7F800000].view(np.float32).astype(np.float64)
    _check_format(f32)
    f64 = rng.integers(0, 2 ** 64, 20_000_000, dtype=np.uint64)
    f64 = f64[(f64 & 0x7FF0000000000000) != 0x7FF0000000000000].view(np.float64)
    _check_format(f64)


def test_format_constructed_ties_and_boundaries():
    values = C.boundary_values() + C.f32_ties() + C.f64_ties() + C.near_ties()
    values += [-v for v in values] + [float("inf"), float("-inf"), float("nan")]
    _check_format(np.array(values))


def test_format_refuses_bad_arguments_without_a_launch():
    lib = _lib.lib()
    before = _lib.launch_count()
    assert lib.arb_format_g16(None, 4, None, None) == -1
    assert lib.arb_svm_write_chunk(None, 0, 1, None, 1, None, 0, 0, 1, None, None, None) == -1
    assert lib.arb_svm_write_check(None, 7, 1, None, 1, 1, None, None) == -1
    assert _lib.launch_count() == before


def _as_input(c, on_device):
    if not on_device:
        return c["X"], c["y"], c["qid"]
    return torch.from_numpy(np.ascontiguousarray(c["X"])).to(DEV), c["y"], c["qid"]


def _write(X, y, qid=None, zero_based=True, to_path=None):
    if to_path is None:
        f = io.BytesIO()
        writer.write_svm_file(X, y, f, zero_based=zero_based, query_id=qid)
        return f.getvalue()
    writer.write_svm_file(X, y, str(to_path), zero_based=zero_based, query_id=qid)
    return to_path.read_bytes()


CHUNKINGS = {"default": None, "rows": 3, "kb": 4096}


def _chunking(monkeypatch, how, n_features, one_based=0):
    if how == "rows":
        monkeypatch.setattr(writer, "_TEXT_CHUNK", CHUNKINGS["rows"] * writer.worst_row_bytes(n_features, one_based))
        monkeypatch.setattr(writer, "_UPLOAD_CHUNK", 3 * 8 * n_features)
    elif how == "kb":
        monkeypatch.setattr(writer, "_TEXT_CHUNK", CHUNKINGS["kb"])
        monkeypatch.setattr(writer, "_UPLOAD_CHUNK", CHUNKINGS["kb"])


@pytest.mark.parametrize("how", list(CHUNKINGS))
@pytest.mark.parametrize("on_device", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_small_cases_match_sklearn(tmp_path, monkeypatch, name, on_device, how):
    c = CASES[name]
    _chunking(monkeypatch, how, c["X"].shape[1], int(not c["zero_based"]))
    X, y, qid = _as_input(c, on_device)
    want = GOLD[name + ".bytes"].tobytes()
    assert _write(X, y, qid, c["zero_based"]) == want
    assert _write(X, y, qid, c["zero_based"], to_path=tmp_path / "f.txt") == want


@pytest.mark.parametrize("how", list(CHUNKINGS))
@pytest.mark.parametrize("on_device", [False, True])
def test_mslr_block_matches_sklearn(tmp_path, monkeypatch, on_device, how):
    X, y, qid = C.mslr_block()
    _chunking(monkeypatch, how, X.shape[1])
    got = _write(torch.from_numpy(X).to(DEV) if on_device else X, y, qid, to_path=tmp_path / "m.txt")
    assert len(got) == int(GOLD["mslr.length"])
    assert hashlib.sha256(got).hexdigest() == str(GOLD["mslr.sha256"])


@pytest.mark.parametrize("on_device", [False, True])
def test_write_to_libsvm_without_masked_matches_the_reference(tmp_path, on_device):
    Xs, ys = C.ragged_slates()
    if on_device:
        Xs = [torch.from_numpy(x).to(DEV) for x in Xs]
    path = tmp_path / "ragged.txt"
    writer.write_to_libsvm_without_masked(str(path), Xs, ys)
    assert path.read_bytes() == GOLD["ragged.bytes"].tobytes()


def test_live_sklearn_on_fresh_data():
    sk = pytest.importorskip("sklearn.datasets")
    rng = np.random.default_rng(int.from_bytes(os.urandom(4), "little"))
    for dtype in (np.float32, np.float64, np.int64):
        n, F = int(rng.integers(1, 300)), int(rng.integers(1, 150))
        bits = rng.integers(0, 2 ** 63, (n, F), dtype=np.int64)
        X = rng.standard_normal((n, F)) * 10.0 ** rng.integers(-30, 30, (n, F))
        X = X.astype(dtype) if dtype != np.int64 else bits - 2 ** 62
        X[rng.random((n, F)) < 0.5] = 0
        y = rng.integers(0, 5, n) if dtype == np.int64 else rng.standard_normal(n).astype(np.float32)
        qid = np.sort(rng.integers(0, 9, n))
        zero_based = bool(rng.integers(0, 2))
        f = io.BytesIO()
        sk.dump_svmlight_file(X, y, f, query_id=qid, zero_based=zero_based)
        assert _write(X, y, qid, zero_based) == f.getvalue(), dtype


@pytest.mark.parametrize("bad", ["nan_x", "inf_x", "nan_y", "ninf_y", "y_length", "qid_length"])
@pytest.mark.parametrize("on_device", [False, True])
def test_refusals_leave_the_file_alone(tmp_path, bad, on_device):
    X = np.ones((4, 3), np.float32)
    y = np.ones(4)
    qid = None
    if bad == "nan_x":
        X[2, 1] = np.nan
    elif bad == "inf_x":
        X[3, 2] = np.inf
    elif bad == "nan_y":
        y[1] = np.nan
    elif bad == "ninf_y":
        y[3] = -np.inf
    elif bad == "y_length":
        y = y[:3]
    else:
        qid = np.arange(5)
    if on_device:
        X = torch.from_numpy(X).to(DEV)
    old = tmp_path / "old.txt"
    old.write_bytes(b"keep me\n")
    for target in (old, tmp_path / "new.txt"):
        with pytest.raises(ValueError):
            writer.write_svm_file(X, y, str(target), query_id=qid)
    assert old.read_bytes() == b"keep me\n"
    assert not (tmp_path / "new.txt").exists()


def test_round_trip_through_the_device_parser(tmp_path):
    X, y, qid = C.mslr_block(n_rows=5000, seed=9)
    X[:, 0] = np.where(X[:, 0] == 0, np.float32(1), X[:, 0])       # column 0 present: the parser's shift is 0
    X[:, -1] = np.where(X[:, -1] == 0, np.float32(2), X[:, -1])     # and the last column: the width is kept
    path = tmp_path / "rt.txt"
    writer.write_svm_file(X, y, str(path), query_id=qid)
    store = data.SlateStore.from_svm_file(str(path), device=DEV, parser="device")
    assert np.array_equal(store.docs_x.cpu().numpy().view(np.uint32), X.view(np.uint32))
    assert np.array_equal(store.docs_y.cpu().numpy().view(np.uint32), y.view(np.uint32))
    assert np.array_equal(store.offsets_host, data.group_offsets(qid))


def _run_rac(workdir, run_id, patch_write):
    code = ("import functools, runpy, sys\n"
            "sys.path.insert(0, {root!r})\n"
            "import allrank_b200.integration as I\n"
            "I.patch_allrank = functools.partial(I.patch_allrank, patch_write={pw})\n"
            "runner = {runner!r}\n"
            "sys.argv = [runner] + {args!r}\n"
            "runpy.run_path(runner, run_name='__main__')\n").format(
        root=ROOT, pw=patch_write, runner=os.path.join(ROOT, "oracle", "run_reference_rank_and_click.py"),
        args=["--workdir", str(workdir), "--run-id", run_id, "--eta", "0", "--patched", "--patch-clicks"])
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, PYTHONDONTWRITEBYTECODE="1"),
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
def test_rank_and_click_writes_identical_files_with_the_device_writer(tmp_path):
    host = _run_rac(tmp_path, "host_write", False)
    dev = _run_rac(tmp_path, "device_write", True)
    assert host["native_so_loaded"] and dev["native_so_loaded"]
    for name in ("train.txt", "vali.txt"):
        with open(os.path.join(host["output_dir"], name), "rb") as a, open(os.path.join(dev["output_dir"], name), "rb") as b:
            want = a.read()
            assert len(want) > 0 and b.read() == want, name
