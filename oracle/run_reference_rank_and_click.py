"""Run the UNMODIFIED `allrank.rank_and_click.run()` (oracle/_ref) on `generate_dummy_data.py` data -- TEST
INFRASTRUCTURE for tests/test_gpu_clicks.py.

    python oracle/run_reference_rank_and_click.py --workdir DIR --run-id NAME --eta ETA [--patched] [--patch-clicks]

The config is the reference's shipped scripts/local_config_click_model.json (tests/golden/) with the data path and
eta overridden: FC[64] + Transformer(N=1, h=1, d_ff=64) + 4 sigmoid outputs, built by the reference's make_model from
torch.manual_seed(0) and saved as DIR/model.pkl, and DiverseClicksModel(BaseCascadeModel(eta, 2), 0.5) as click
model (eta = 0 makes it deterministic; the shipped value is 1).  Prints
"RESULT {json}" with the output directory and whether liballrank_b200.so was loaded.
"""
import argparse
import json
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


SHIPPED_CONFIG = os.path.join(ROOT, "tests", "golden", "local_config_click_model.json")


def config(data_path, eta):
    """The reference's scripts/local_config_click_model.json (kept as a fixture) with the data path and the inner
    cascade's eta set."""
    with open(SHIPPED_CONFIG) as fh:
        cfg = json.load(fh)
    cfg["data"]["path"] = data_path
    cfg["click_model"]["args"]["inner_click_model"]["args"]["eta"] = eta
    return cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workdir", required=True)
    ap.add_argument("--run-id", default="run")
    ap.add_argument("--eta", type=float, default=0.0)
    ap.add_argument("--patched", action="store_true")
    ap.add_argument("--patch-clicks", action="store_true")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    from oracle.install_reference import import_path, installed
    if not installed():
        raise SystemExit("oracle/_ref is missing: run oracle/install_reference.py")
    sys.path[:0] = import_path()
    os.makedirs(a.workdir, exist_ok=True)
    os.chdir(a.workdir)
    if not os.path.exists(os.path.join("dummy_data", "train.txt")):
        import allrank.data.generate_dummy_data as gen
        argv, sys.argv = sys.argv, ["generate_dummy_data.py"]
        try:
            runpy.run_path(gen.__file__, run_name="__main__")
        finally:
            sys.argv = argv
    eta = int(a.eta) if float(a.eta).is_integer() else a.eta
    cfg = config(os.path.join(a.workdir, "dummy_data"), eta)
    used = os.path.join(a.workdir, f"config_{a.run_id}.json")
    with open(used, "w") as fh:
        json.dump(cfg, fh)
    import torch
    model_path = os.path.join(a.workdir, "model.pkl")
    if not os.path.exists(model_path):
        from attr import asdict
        from allrank.config import Config
        from allrank.data.dataset_loading import load_libsvm_dataset_role
        from allrank.models.model import make_model
        n_features = load_libsvm_dataset_role("vali", cfg["data"]["path"], 240).shape[-1]
        torch.manual_seed(0)
        model = make_model(n_features=n_features, **asdict(Config.from_json(used).model, recurse=False))
        torch.save(model.state_dict(), model_path)
    if a.patched:
        from allrank_b200.integration import patch_allrank
        patch_allrank(patch_clicks=a.patch_clicks)
    import allrank.rank_and_click as rac
    out = os.path.join(a.workdir, "out")
    sys.argv = ["rank_and_click", "--job-dir", out, "--run-id", a.run_id, "--config-file-name", used,
                "--input-model-path", model_path, "--roles", "train,vali"]
    rac.run()
    so_loaded = any("liballrank_b200.so" in line for line in open("/proc/self/maps"))
    print("RESULT " + json.dumps({"output_dir": os.path.join(out, "results", a.run_id), "native_so_loaded": so_loaded}))


if __name__ == "__main__":
    main()
