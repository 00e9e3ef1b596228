"""Feature normalisation on the GPU (allrank_b200/normalize.py, csrc/normalize.cu, csrc/log_cr.cuh): the device log
against the host build, float64 pass 2 against sklearn, the column statistics and whole folds against
tests/golden/normalize.npz (tools/make_golden_normalize.py), stdout, refusals and a round trip through the parser."""
import contextlib
import hashlib
import io
import os

import numpy as np
import pytest
import torch

from allrank_b200 import data
from allrank_b200 import normalize as N
from tests import normalize_cases as C

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "normalize.npz"))
DEV = torch.device("cuda:0")


@pytest.mark.parametrize("force_accurate", [False, True])
def test_log_cr_device_matches_host(force_accurate):
    rng = np.random.default_rng(5)
    n = 20_000_000 if not force_accurate else 2_000_000
    x = rng.integers(0, 0x7ff0000000000001, n, dtype=np.int64).view(np.float64)
    x[:4] = [0.0, np.inf, 1.0, 5e-324]
    y_dev, n_dev = N.log_cr(torch.from_numpy(x).to(DEV), force_accurate)
    y_host, n_host = N.log_cr(x, force_accurate)
    assert n_dev == n_host
    assert np.array_equal(y_dev.cpu().numpy().view(np.int64), y_host.view(np.int64))


@pytest.mark.parametrize("force_accurate", [False, True])
def test_log_cr_device_hard_cases(force_accurate):
    k = np.arange(1, 4000, dtype=np.float64)
    x = np.concatenate([1 + k * 2.0 ** -52, 1 - k * 2.0 ** -53, 1 - k * 2.0 ** -52, C.near_one_values() + 0.01])
    for name in ("near_one", "mslr_small", "basic"):                 # every logged argument of the golden folds
        for role in C.ROLES:
            text = C.FOLDS[name][0][role].decode().split()
            vals = np.array([float(t.split(":")[1]) for t in text if ":" in t and not t.startswith("qid")])
            x = np.concatenate([x, np.abs(vals) + 0.01])
    y_dev, n_dev = N.log_cr(torch.from_numpy(x).to(DEV), force_accurate)
    y_host, n_host = N.log_cr(x, force_accurate)
    assert n_dev == n_host and n_dev > 0
    assert np.array_equal(y_dev.cpu().numpy().view(np.int64), y_host.view(np.int64))


PARSE = sorted({k.split("/")[1] for k in GOLD.files if k.startswith("parse/")})


@pytest.mark.parametrize("case", PARSE)
def test_float64_pass2_against_sklearn(case):
    text = bytes(GOLD["parse/{}/text".format(case)])
    dev_text = torch.from_numpy(np.frombuffer(text, np.uint8).copy()).to(DEV)
    plan = data.LibSVMPlan(dev_text)
    x = torch.full((plan.n_rows, plan.n_features), 7.0, dtype=torch.float64, device=DEV)
    y = torch.full((plan.n_rows,), 7.0, dtype=torch.float64, device=DEV)
    q = torch.empty((plan.n_rows,), dtype=torch.int64, device=DEV)
    plan.write(x, y, q)
    ref_x, ref_y = GOLD["parse/{}/x".format(case)], GOLD["parse/{}/y".format(case)]
    assert tuple(x.shape) == ref_x.shape
    got_x, got_y = x.cpu().numpy().view(np.int64), y.cpu().numpy().view(np.int64)
    nan_x, nan_y = np.isnan(ref_x.view(np.float64)), np.isnan(ref_y.view(np.float64))
    assert np.array_equal(np.isnan(x.cpu().numpy()), nan_x) and np.array_equal(got_x[~nan_x], ref_x[~nan_x])
    assert np.array_equal(np.isnan(y.cpu().numpy()), nan_y) and np.array_equal(got_y[~nan_y], ref_y[~nan_y])


def _run(tmp_path, name, texts, fwl, fneg):
    fold = str(tmp_path / name)
    C.write_fold(texts, fold)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        out_dir = N.normalize_features(fold, fwl, fneg, device=DEV)
    files = {r: open(os.path.join(out_dir, r + ".txt"), "rb").read() for r in C.ROLES}
    return fold, files, buf.getvalue().replace(fold, "{dir}").rstrip("\n")


@pytest.mark.parametrize("name", sorted(C.FOLDS))
def test_fold_bytes_stdout_and_statistics(tmp_path, name):
    texts, fwl, fneg = C.FOLDS[name]
    fold, files, stdout = _run(tmp_path, name, texts, fwl, fneg)
    for role in C.ROLES:
        assert files[role] == bytes(GOLD["{}/{}".format(name, role)]), role
    assert stdout == bytes(GOLD[name + "/stdout"]).decode()
    roles = [N._load_role(os.path.join(fold, r + ".txt"), DEV)[0] for r in C.ROLES]
    _, mean, std, _ = N.normalize_roles(roles[0], roles[1:], fwl, fneg)
    assert np.array_equal(mean.cpu().numpy().view(np.int64), GOLD[name + "/mean"])
    assert np.array_equal(std.cpu().numpy().view(np.int64), GOLD[name + "/std"])


@pytest.mark.parametrize("name", sorted(C.FOLDS))
def test_fold_without_logarithm_is_the_scripts_bytes(tmp_path, name):
    texts, _, fneg = C.FOLDS[name]
    _, files, _ = _run(tmp_path, name, texts, list(range(200)), fneg)
    for role in C.ROLES:
        assert files[role] == bytes(GOLD["{}/nolog/{}".format(name, role)]), role


def test_large_mslr_fold(tmp_path):
    texts, fwl, fneg = C.mslr_fold(C.LARGE_ROWS, seed=11)
    _, files, stdout = _run(tmp_path, "large", texts, fwl, fneg)
    for role in C.ROLES:
        assert len(files[role]) == int(GOLD["large/{}/len".format(role)])
        assert hashlib.sha256(files[role]).digest() == bytes(GOLD["large/{}/sha256".format(role)])
    assert stdout == bytes(GOLD["large/stdout"]).decode()


@pytest.mark.parametrize("name", sorted(C.REFUSALS))
def test_refusals_create_nothing(tmp_path, name):
    texts, exc = C.REFUSALS[name]
    fold = str(tmp_path / name)
    C.write_fold(texts, fold)
    with contextlib.redirect_stdout(io.StringIO()), pytest.raises(exc):
        N.normalize_features(fold, [], [], device=DEV)
    assert not os.path.exists(fold + "_normalized")


def test_trailing_slash_names_the_directory_like_the_script(tmp_path):
    texts, fwl, fneg = C.FOLDS["basic"]
    fold = str(tmp_path / "f")
    C.write_fold(texts, fold)
    with contextlib.redirect_stdout(io.StringIO()):
        out_dir = N.normalize_features(fold + "/", fwl, fneg, device=DEV)
    assert out_dir == fold + "/_normalized" and os.path.isfile(os.path.join(fold, "_normalized", "vali.txt"))


def test_round_trip_through_the_device_parser(tmp_path):
    texts, fwl, fneg = C.FOLDS["mslr_small"]
    fold, _, _ = _run(tmp_path, "rt", texts, fwl, fneg)
    for role in C.ROLES:
        path = os.path.join(fold + "_normalized", role + ".txt")
        a = data.SlateStore.from_svm_file(path, device=DEV, parser="device")
        b = data.SlateStore.from_svm_file(path, device=DEV, parser="sklearn")
        assert torch.equal(a.docs_x, b.docs_x) and torch.equal(a.docs_y, b.docs_y)
        assert np.array_equal(a.offsets_host, b.offsets_host)


def test_command_line_module(tmp_path):
    texts, fwl, fneg = C.FOLDS["basic"]
    fold = str(tmp_path / "cli")
    C.write_fold(texts, fold)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        N.main(["--ds_path", fold, "--features_without_logarithm", *map(str, fwl), "--features_negative",
                *map(str, fneg)])
    for role in C.ROLES:
        with open(os.path.join(fold + "_normalized", role + ".txt"), "rb") as f:
            assert f.read() == bytes(GOLD["basic/{}".format(role)])
