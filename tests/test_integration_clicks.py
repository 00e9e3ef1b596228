"""patch_allrank() and allrank/rank_and_click.py: the names rank_and_click.py imported (make_model,
CustomDataParallel, rank_slates, metrics_on_clicked_slates, click_on_slates) and inference_utils'
metrics_on_clicked_slates are rebound, click_on_slates only with patch_clicks=True, and unpatch_allrank restores
them all.  Runs against the installed reference copy in oracle/_ref when it is present."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "allrank", "rank_and_click.py"))


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref (the installed reference) is not present")
@pytest.mark.parametrize("patch_clicks", [False, True])
def test_rank_and_click_bindings(patch_clicks):
    from oracle.install_reference import import_path
    paths = import_path()
    sys.path[:0] = paths
    try:
        import allrank.click_models.click_utils as ref_cu
        import allrank.inference.inference_utils as ref_iu
        import allrank.rank_and_click as rac
        from allrank_b200 import click_models, inference, integration, model
        names = ("make_model", "CustomDataParallel", "rank_slates", "metrics_on_clicked_slates", "click_on_slates")
        before = {n: getattr(rac, n) for n in names}
        before_iu, before_cu = ref_iu.metrics_on_clicked_slates, ref_cu.click_on_slates
        saved = integration.patch_allrank(patch_clicks=patch_clicks)
        try:
            assert rac.make_model is model.make_model
            assert rac.CustomDataParallel is integration.single_process_model
            assert rac.rank_slates is inference.rank_slates
            assert rac.metrics_on_clicked_slates is inference.metrics_on_clicked_slates
            assert ref_iu.metrics_on_clicked_slates is inference.metrics_on_clicked_slates
            if patch_clicks:
                assert rac.click_on_slates is ref_cu.click_on_slates is click_models.click_on_slates
            else:
                assert rac.click_on_slates is before["click_on_slates"] and ref_cu.click_on_slates is before_cu
        finally:
            integration.unpatch_allrank(saved)
        assert {n: getattr(rac, n) for n in names} == before
        assert ref_iu.metrics_on_clicked_slates is before_iu and ref_cu.click_on_slates is before_cu
    finally:
        for p in paths:
            if p in sys.path:
                sys.path.remove(p)
