"""Run the UNMODIFIED `allrank.main.run()` (oracle/_ref) on `generate_dummy_data.py` data -- TEST INFRASTRUCTURE for
the L3 parity layer (SURVEY.md 8c): once as the pure reference on the CPU, once with `patch_allrank()` on cuda:0.

    python oracle/run_reference_main.py --workdir DIR --config CONFIG.json [--patched] [--run-id NAME]

The script is launched as a subprocess by tests/test_gpu_l3_training.py (the CPU arm with CUDA_VISIBLE_DEVICES="",
which the reference needs because get_torch_device() hard-wires cuda:0, allrank/models/model_utils.py:13-18).
It prints one JSON line: {"val_metrics": ..., "train_metrics": ..., "native_so_loaded": bool}.
"""
import argparse
import json
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workdir", required=True)
    ap.add_argument("--config", required=True)
    ap.add_argument("--patched", action="store_true")
    ap.add_argument("--run-id", default="run")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    from oracle.install_reference import import_path, installed
    if not installed():
        raise SystemExit("oracle/_ref is missing: run oracle/install_reference.py (needs an allRank source tree, $ALLRANK_REFERENCE)")
    sys.path[:0] = import_path()
    os.makedirs(a.workdir, exist_ok=True)
    os.chdir(a.workdir)
    if not os.path.exists(os.path.join("dummy_data", "train.txt")):
        # the reference's own generator, run exactly as scripts/run_example.sh does (np.random.seed(42) inside)
        import allrank.data.generate_dummy_data as gen
        argv, sys.argv = sys.argv, ["generate_dummy_data.py"]
        try:
            runpy.run_path(gen.__file__, run_name="__main__")
        finally:
            sys.argv = argv
    cfg = json.load(open(a.config))
    cfg["data"]["path"] = os.path.join(a.workdir, "dummy_data")
    used = os.path.join(a.workdir, f"config_{a.run_id}.json")
    json.dump(cfg, open(used, "w"))
    if a.patched:
        from allrank_b200.integration import patch_allrank
        patch_allrank()
    import allrank.main as ref_main
    sys.argv = ["allrank", "--config-file-name", used, "--run-id", a.run_id, "--job-dir", os.path.join(a.workdir, "out")]
    ref_main.run()
    res = json.load(open(os.path.join(a.workdir, "out", "results", a.run_id, "experiment_result.json")))
    so_loaded = any("liballrank_b200.so" in line for line in open("/proc/self/maps"))
    keep = {k: v for k, v in res.items() if k.startswith(("val_metrics", "train_metrics", "epochs", "num_params"))}
    keep["native_so_loaded"] = so_loaded
    print("RESULT " + json.dumps(keep))


if __name__ == "__main__":
    main()
