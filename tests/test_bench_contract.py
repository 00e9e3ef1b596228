"""bench.py contract on the CPU side: the reference arm (`--impl reference`) runs without a GPU -- the unmodified
allRank package from oracle/_ref when it is installed (oracle/install_reference.py), else the oracle port -- and
prints ONE JSON line with the keys the driver reads."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, r.stdout[-2000:]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "slates/sec" and d["unit"] == "slates/s"
    assert d["higher_is_better"] is True and d["n_gpus"] == 1 and d["value"] > 0
    assert d["config"]["workload"].startswith("cfg2") and d["config"]["slate_len"] == 240
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("reference", "port") and cb["cores"] >= 1 and cb["value"] == d["value"]
    assert d["e2e"]["value"] == d["value"] and d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0


def test_bench_refuses_to_run_the_gpu_arm_without_a_device():
    """No CPU fallback: without a CUDA device the default arm exits with a message instead of measuring something else."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "3", "--no-cpu-baseline"],
                       capture_output=True, text=True, timeout=300, cwd=ROOT, env=env)
    assert r.returncode != 0
    assert "no CUDA device" in (r.stderr + r.stdout)
