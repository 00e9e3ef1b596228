"""Click models on the device (allrank_b200.click_models, csrc/clicks.cu) against the reference's golden clicks
(tests/golden/clicks.npz), the CPU oracle (oracle/clicks_ref.py) fed by a host restatement of the counter hash, and
binomial bounds; plus the unmodified `allrank.rank_and_click.run()` end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from allrank_b200 import click_models as cmod
from allrank_b200 import inference
from oracle import clicks_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "clicks.npz"))
CASES = json.loads(str(GOLD["cases"]))
DEV = torch.device("cuda:0")
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "allrank", "rank_and_click.py"))
M32 = 0xFFFFFFFF


def _mix32(h):
    h ^= h >> 16; h = (h * 0x85ebca6b) & M32
    h ^= h >> 13; h = (h * 0xc2b2ae35) & M32
    return h ^ (h >> 16)


def hash_uniform(seed):
    """Host restatement of click_bits / click_uniform (csrc/clicks.cu)."""
    def u(node, slate, item):
        a = _mix32((seed & M32) ^ ((node * 0x9e3779b1 + 0x7f4a7c15) & M32))
        a = _mix32(a ^ (seed >> 32) ^ (((slate & M32) * 0x85ebca6b) & M32))
        a = _mix32(a ^ (((slate >> 32) * 0xc2b2ae35) & M32) ^ ((item * 0x27d4eb2f + 0x165667b1) & M32))
        hi, lo = _mix32(a ^ 0x68e31da4), _mix32((a + 0xb5297a4d) & M32)
        return float((hi << 21) | (lo >> 11)) * 2.0 ** -53
    return u


def data(name):
    return torch.tensor(GOLD[name + "_x"]).to(DEV), torch.tensor(GOLD[name + "_y"]).to(DEV)


def case_id(c):
    return f"{c['id']}-{c['kind']}-{c['spec']['name']}-{c['data']}"


@pytest.mark.parametrize("case", [c for c in CASES if c["kind"] == "deterministic"], ids=case_id)
def test_deterministic_trees_are_bit_identical_to_the_reference(case):
    x, y = data(case["data"])
    got = cmod.click(clicks_ref.build_model(case["spec"], cmod), x, y, seed=77).cpu().numpy()
    assert np.array_equal(got, GOLD[f"case{case['id']}_clicks"])


@pytest.mark.parametrize("case", [c for c in CASES if c["kind"] == "error"], ids=case_id)
def test_errors_have_the_reference_exception_type(case):
    x, y = data(case["data"])
    with pytest.raises(Exception) as info:
        cmod.click(clicks_ref.build_model(case["spec"], cmod), x, y, seed=5)
    assert type(info.value).__name__ == case["error"]


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_every_tree_matches_the_oracle_under_the_counter_hash(case):
    x, y = data(case["data"])
    seed = 0x1234567890ABCDEF + case["id"]
    model = clicks_ref.build_model(case["spec"], cmod)
    got, status = cmod.click(model, x, y, seed=seed, check=False, return_status=True)
    u = hash_uniform(seed)
    status = status.cpu().numpy()
    for b in range(y.shape[0]):
        try:
            want = clicks_ref.click_slates(model, x[b:b + 1].cpu().numpy(), y[b:b + 1].cpu().numpy(),
                                           clicks_ref.TableSource(lambda n, s, j: u(n, b, j)))
        except (IndexError, ValueError) as exc:
            assert status[b] == (cmod.STATUS_INDEX_ERROR if isinstance(exc, IndexError) else cmod.STATUS_VALUE_ERROR)
            continue
        assert status[b] == 0
        assert np.array_equal(got[b].cpu().numpy(), want[0]), (b, got[b], want[0])


def test_reference_instances_compile():
    if not HAVE_REF:
        pytest.skip("oracle/_ref (the installed reference) is not present")
    from oracle.install_reference import import_path
    sys.path[:0] = import_path()
    from tools.make_golden_clicks import reference_classes
    spec = [c for c in CASES if c["kind"] == "deterministic" and c["spec"]["name"] == "DiverseClicksModel"][0]
    x, y = data(spec["data"])
    got = cmod.click(clicks_ref.build_model(spec["spec"], reference_classes()), x, y).cpu().numpy()
    assert np.array_equal(got, GOLD[f"case{spec['id']}_clicks"])


def _bound(p, n):
    return 5.0 * np.sqrt(max(p * (1 - p), 1e-12) / n) + 1e-9


def test_cascade_click_rates_follow_the_observation_probability():
    B, S = 20000, 16
    y = torch.full((B, S), 3.0, device=DEV)
    for eta in (1, 0.5, 2.0):
        c = cmod.click(cmod.BaseCascadeModel(eta, 1), None, y, seed=11).float().mean(0).cpu().numpy()
        p = np.minimum(1.0, np.arange(1, S + 1, dtype=np.float64) ** -float(eta))
        assert np.all(np.abs(c - p) <= [_bound(q, B) for q in p]), (eta, c, p)


def test_multiple_child_frequencies_and_random_marginals():
    B = 20000
    y = torch.zeros((B, 10), device=DEV)
    m = cmod.MultipleClickModel([cmod.FixedClickModel([k]) for k in range(3)], [0.2, 0.3, 0.5])
    freq = cmod.click(m, None, y, seed=3)[:, :3].float().mean(0).cpu().numpy()
    assert np.all(np.abs(freq - [0.2, 0.3, 0.5]) <= [_bound(p, B) for p in (0.2, 0.3, 0.5)]), freq
    c = cmod.click(cmod.RandomClickModel(3), None, y, seed=9)
    assert torch.all(c.sum(1) == 3)
    marg = c.float().mean(0).cpu().numpy()
    assert np.all(np.abs(marg - 0.3) <= _bound(0.3, B)), marg


def test_only_the_chosen_child_raises():
    y = torch.zeros((64, 5), device=DEV)
    ok = cmod.MultipleClickModel([cmod.FixedClickModel([7]), cmod.OnlyRelevantClickModel(1)], [0.0, 1.0])
    assert torch.all(cmod.click(ok, None, y) == 0)
    bad = cmod.MultipleClickModel([cmod.FixedClickModel([7]), cmod.RandomClickModel(9)], [0.5, 0.5])
    with pytest.raises(IndexError):     # slate 0 picks one of the two; either way the first error is an IndexError
        cmod.click(cmod.MultipleClickModel([cmod.FixedClickModel([7])], [1.0]), None, y)
    with pytest.raises((IndexError, ValueError)):
        cmod.click(bad, None, y)


def _slates(B, S, F, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, S, F, generator=g)
    y = torch.randint(0, 5, (B, S), generator=g).float()
    n = torch.randint(0, S + 1, (B,), generator=g)
    y[torch.arange(S)[None, :] >= n[:, None]] = -1.0
    y[:, S // 3] = -1.0 if S > 2 else y[:, S // 3]     # padding in the middle too
    return x, y


TREE = cmod.MaxClicksModel(cmod.DiverseClicksModel(cmod.BaseCascadeModel(0.7, 1), 0.4), 6)


def test_chunking_repeats_and_no_sync_without_check():
    x, y = _slates(12, 240, 136, 1)
    x, y = x.to(DEV), y.to(DEV)
    full = cmod.click(TREE, x, y, seed=42)
    per = cmod.compile_click_model(TREE)
    one = (240 * 239 // 2 * 8 + 255) // 256 * 256        # one slate's distance triangle
    chunked = cmod.click(TREE, x, y, seed=42, workspace_bytes=3 * one)
    assert torch.equal(full, chunked)
    assert torch.equal(full, cmod.click(per, x, y, seed=42))
    halves = torch.cat([cmod.click(TREE, x[:5], y[:5], seed=42), cmod.click(TREE, x[5:], y[5:], seed=42, slate_offset=5)])
    assert torch.equal(full, halves)
    # an uncompiled model never seen before, with a CASCADE node, at a slate length not used before: its
    # observation table is uploaded during the call, and nothing may synchronise
    fresh = cmod.MaxClicksModel(cmod.DiverseClicksModel(cmod.BaseCascadeModel(0.3, 1), 0.5), 4)
    x77, y77 = (t.to(DEV) for t in _slates(6, 77, 46, 2))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        fresh_clicks = cmod.click(fresh, x77, y77, seed=42, check=False)
        cmod.click(per, x, y, seed=42, check=False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(fresh_clicks, cmod.click(fresh, x77, y77, seed=42))
    np.random.seed(0)
    xs, cl = cmod.click_on_slates((x.cpu(), y.cpu()), TREE, include_empty=True)
    np.random.seed(0)
    assert torch.equal(torch.tensor(np.stack(cl)), cmod.click(TREE, x, y, seed=cmod.draw_seed()).cpu())
    assert len(xs) == 12 and xs[0] is not None
    # ragged per-slate lists give the same clicks as the padded batch, one launch per chunk
    lens = [int((y[b] != -1).nonzero().max()) + 1 if bool((y[b] != -1).any()) else 1 for b in range(12)]
    xr = [x[b, :lens[b]].cpu() for b in range(12)]
    yr = [y[b, :lens[b]].cpu() for b in range(12)]
    np.random.seed(0)
    _, cr = cmod.click_on_slates((xr, yr), TREE, include_empty=True)
    assert all(np.array_equal(cr[b], cl[b][:lens[b]]) for b in range(12))
    with pytest.raises(ValueError):
        cmod.click_on_slates((x.cpu(), torch.zeros_like(y).cpu()), cmod.OnlyRelevantClickModel(1), include_empty=False)


@pytest.mark.parametrize("S,F,B", [(1, 136, 4), (240, 46, 3), (240, 136, 3), (240, 700, 2), (1251, 136, 2)])
def test_shapes_match_the_oracle(S, F, B):
    x, y = _slates(B, S, F, S + F)
    models = [cmod.DiverseClicksModel(cmod.BaseCascadeModel(0, 1), 0.5),
              cmod.EverythingButDuplicatesClickModel(float(np.sqrt(2 * F)), "euclidean"),
              cmod.DiverseClicksModel(cmod.RandomClickModel(0), 0.9)]
    for m in models:
        got = cmod.click(m, x.to(DEV), y.to(DEV), seed=8, check=False).cpu().numpy()
        for b in range(B):
            try:
                want = clicks_ref.click_slates(m, x[b:b + 1].numpy(), y[b:b + 1].numpy(),
                                               clicks_ref.TableSource(lambda n, s, j: hash_uniform(8)(n, b, j)))
            except ValueError:
                continue
            assert np.array_equal(got[b], want[0]), (type(m).__name__, S, F, b)


def test_metrics_on_clicked_slates_match_the_reference():
    if not HAVE_REF:
        pytest.skip("oracle/_ref (the installed reference) is not present")
    from oracle.install_reference import import_path
    sys.path[:0] = import_path()
    import allrank.inference.inference_utils as iu
    x, y = _slates(40, 30, 8, 5)
    np.random.seed(1)
    xs, cl = cmod.click_on_slates((x, y), cmod.BaseCascadeModel(1, 1), include_empty=True)
    cl = cl + [np.full(30, -1.0, dtype=np.float32), np.zeros(12, dtype=np.float32)]
    xs = xs + [None, None]
    ref = list(iu.metrics_on_clicked_slates((xs, cl)))
    mine = list(inference.metrics_on_clicked_slates((xs, cl)))
    assert len(ref) == len(mine)
    for r, m in zip(ref, mine):
        assert r == m and type(r["no_of_clicks"]) is type(m["no_of_clicks"]), (r, m)


def _run_rac(workdir, run_id, eta, patched, patch_clicks):
    cmd = [sys.executable, os.path.join(ROOT, "oracle", "run_reference_rank_and_click.py"), "--workdir", str(workdir),
           "--run-id", run_id, "--eta", str(eta)] + (["--patched"] if patched else []) + \
          (["--patch-clicks"] if patch_clicks else [])
    r = subprocess.run(cmd, env=dict(os.environ, PYTHONDONTWRITEBYTECODE="1"), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
def test_rank_and_click_runs_patched_and_device_clicks_write_identical_files(tmp_path):
    host = _run_rac(tmp_path, "host_clicks", 0, patched=True, patch_clicks=False)
    dev = _run_rac(tmp_path, "device_clicks", 0, patched=True, patch_clicks=True)
    assert host["native_so_loaded"] and dev["native_so_loaded"]
    for name in ("train.txt", "vali.txt", "train_metrics.csv", "vali_metrics.csv", "train_metrics_mean.csv",
                 "vali_metrics_mean.csv"):
        with open(os.path.join(host["output_dir"], name), "rb") as a, open(os.path.join(dev["output_dir"], name), "rb") as b:
            assert a.read() == b.read(), name
    shipped = _run_rac(tmp_path, "eta1", 1, patched=True, patch_clicks=True)
    assert os.path.getsize(os.path.join(shipped["output_dir"], "vali_metrics.csv")) > 0


def test_single_slate_click_returns_the_reference_dtype():
    x, y = _slates(1, 9, 4, 3)
    docs = (x[0].numpy(), np.maximum(y[0].numpy(), 0))
    assert cmod.OnlyRelevantClickModel(1).click(docs).dtype == np.bool_
    dup = cmod.EverythingButDuplicatesClickModel(0.5)
    assert dup.click(docs).dtype == np.dtype(np.int_)
    assert cmod.DiverseClicksModel(dup).click(docs).dtype == np.dtype(np.int_)
    masked = cmod.MaskedRemainMasked(cmod.OnlyRelevantClickModel(1)).click((x[0].numpy(), y[0].numpy()))
    assert masked.dtype == np.float32 and np.all(masked[y[0].numpy() == -1] == -1)
