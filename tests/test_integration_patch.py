"""patch_allrank() against the reference package.  The call surfaces are compared with the reference's signatures
stored in tests/golden/reference_signatures.json (written from the unmodified package); the rebinding mechanics
INTEGRATION.md describes run against the installed copy in oracle/_ref (oracle/install_reference.py) when it is
present.  The kernels themselves are covered by the GPU tests."""
import inspect
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "allrank", "main.py"))


def test_call_surfaces_match_the_reference_signatures():
    from allrank_b200 import data, inference, integration, losses, metrics, model, training
    with open(os.path.join(ROOT, "tests", "golden", "reference_signatures.json")) as fh:
        ref = json.load(fh)
    sig = lambda f: list(inspect.signature(f).parameters)
    # same call surface: every patched callable accepts the reference's parameter names in the same order
    assert sorted(ref["losses"]) == sorted(integration.LOSS_NAMES)
    for name, ref_params in ref["losses"].items():
        mine = sig(getattr(losses, name))
        assert mine[:len(ref_params)] == ref_params, (name, ref_params, mine)
    assert sorted(ref["metrics"]) == sorted(integration.METRIC_NAMES)
    for name, ref_params in ref["metrics"].items():
        assert sig(getattr(metrics, name)) == ref_params, name
    ref_params = ref["model"]["make_model"]
    mine = sig(model.make_model)
    assert mine[:len(ref_params)] == ref_params and mine[len(ref_params):] == ["compute_dtype"]   # one extension
    # the callers either side of the path: same parameter names as the reference functions they replace
    for key, mine_mod in (("train_utils", training), ("inference_utils", inference), ("dataset_loading", data)):
        for name, ref_params in ref[key].items():
            mine = sig(getattr(mine_mod, name))
            assert mine[:len(ref_params)] == ref_params, (name, ref_params, mine)
    assert data.PADDED_Y_VALUE == ref["constants"]["PADDED_Y_VALUE"]
    assert data.PADDED_INDEX_VALUE == ref["constants"]["PADDED_INDEX_VALUE"]


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
def test_patch_and_unpatch_rebinds_the_reference_names():
    from oracle.install_reference import import_path
    paths = import_path()
    sys.path[:0] = paths
    try:
        import allrank.models.losses as ref_losses
        import allrank.models.metrics as ref_metrics
        import allrank.models.model as ref_model
        import allrank.training.train_utils as ref_tu
        import allrank.inference.inference_utils as ref_iu
        import allrank.data.dataset_loading as ref_dl
        from allrank_b200 import data, inference, integration, losses, metrics, model, training
        originals = {n: getattr(ref_losses, n) for n in integration.LOSS_NAMES}
        orig_cm, orig_loader = ref_tu.compute_metrics, ref_dl.create_data_loaders
        saved = integration.patch_allrank(patch_data=True)
        try:
            assert ref_losses.lambdaLoss is losses.lambdaLoss
            assert ref_losses.ordinal is losses.ordinal
            assert ref_metrics.ndcg is metrics.ndcg
            assert ref_model.make_model is model.make_model
            assert ref_tu.compute_metrics is training.compute_metrics
            assert ref_iu.rank_slates is inference.rank_slates
            assert ref_dl.create_data_loaders is data.create_data_loaders
            import allrank.main as ref_main
            assert ref_main.load_libsvm_dataset is data.load_libsvm_dataset
        finally:
            integration.unpatch_allrank(saved)
        for n, fn in originals.items():
            assert getattr(ref_losses, n) is fn
        assert ref_tu.compute_metrics is orig_cm and ref_dl.create_data_loaders is orig_loader
    finally:
        for p in paths:
            if p in sys.path:
                sys.path.remove(p)
