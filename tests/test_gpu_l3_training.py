"""L3 parity (SURVEY.md 8c): the UNMODIFIED reference training driver -- `allrank.main.run()` ->
`train_utils.fit` (allrank/main.py:34-110, allrank/training/train_utils.py:78-147) -- run from oracle/_ref on the
reference's own dummy data (allrank/data/generate_dummy_data.py), twice in the same test:
  * as the pure reference on the host CPU (subprocess with CUDA_VISIBLE_DEVICES=""),
  * with `allrank_b200.integration.patch_allrank()` on cuda:0 (model, losses, metrics, epoch metrics on the GPU).
Anchor: BASELINE config 1 reaches val ndcg_5 = 0.5709 on the reference (BASELINE.md section 2).

oracle/_ref is produced by oracle/install_reference.py (pip install of an allRank source tree with --no-deps, run by
__graft_entry__.build() where one is readable); without it the tests skip.
"""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUNNER = os.path.join(ROOT, "oracle", "run_reference_main.py")
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "allrank", "main.py"))


def run_main(workdir, config, run_id, patched):
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    if not patched:
        env["CUDA_VISIBLE_DEVICES"] = ""
    cmd = [sys.executable, RUNNER, "--workdir", str(workdir), "--config", os.path.join(ROOT, "tests", "configs", config),
           "--run-id", run_id] + (["--patched"] if patched else [])
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
def test_unmodified_main_run_config1_matches_the_reference_anchor(tmp_path):
    """FC[64] + listNet, batch 32, slate_length 120, Adam 1e-3, StepLR(3, 0.5), 4 epochs, seeds 42: the same seeded
    initialisation and the same data order => the patched GPU run follows the CPU reference's trajectory."""
    cpu = run_main(tmp_path, "baseline_cfg1.json", "cpu", patched=False)
    gpu = run_main(tmp_path, "baseline_cfg1.json", "gpu", patched=True)
    assert gpu["native_so_loaded"] and not cpu["native_so_loaded"]
    assert abs(cpu["val_metrics/ndcg_5"] - 0.5709) < 2e-3          # BASELINE.md anchor, reproduced on this host
    assert abs(gpu["val_metrics/ndcg_5"] - cpu["val_metrics/ndcg_5"]) < 1e-2, (gpu, cpu)
    assert abs(gpu["train_metrics/ndcg_5"] - cpu["train_metrics/ndcg_5"]) < 1e-2, (gpu, cpu)
    assert gpu["num_params"] == cpu["num_params"] == 1409
    print("L3 cfg1: reference", cpu["val_metrics/ndcg_5"], "patched GPU", gpu["val_metrics/ndcg_5"])


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
def test_unmodified_main_run_transformer_config_trains_like_the_reference(tmp_path):
    """Transformer(N=2, h=2) + approxNDCG with dropout 0.1, 6 epochs.  Dropout streams differ (counter hash vs
    Philox), so the final metrics agree within run-to-run noise, not bit for bit."""
    cpu = run_main(tmp_path, "transformer_cfg.json", "cpu", patched=False)
    gpu = run_main(tmp_path, "transformer_cfg.json", "gpu", patched=True)
    assert gpu["native_so_loaded"]
    assert gpu["num_params"] == cpu["num_params"]
    for k in ("val_metrics/ndcg_5", "val_metrics/ndcg_10", "val_metrics/mrr_5"):
        assert abs(gpu[k] - cpu[k]) < 4e-2, (k, gpu[k], cpu[k])
    assert gpu["val_metrics/ndcg_5"] > 0.70
    print("L3 transformer: reference", cpu, "patched GPU", gpu)
