"""The click-model oracle (oracle/clicks_ref.py) against tests/golden/clicks.npz, written from the unmodified reference
by tools/make_golden_clicks.py: deterministic trees, the reference's exception types, and random trees replayed
from the same numpy seed in the reference's draw order.  Also: allrank_b200.click_models has the reference's public
signatures (tests/golden/click_signatures.json)."""
import inspect
import json
import os

import numpy as np
import pytest

from allrank_b200 import click_models, inference
from oracle import clicks_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "clicks.npz"))
CASES = json.loads(str(GOLD["cases"]))


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c['id']}-{c['kind']}-{c['spec']['name']}-{c['data']}")
def test_oracle_reproduces_the_reference(case):
    model = clicks_ref.build_model(case["spec"], click_models)
    x, y = GOLD[case["data"] + "_x"], GOLD[case["data"] + "_y"]
    np.random.seed(case["seed"])
    if case["error"]:
        with pytest.raises(Exception) as info:
            clicks_ref.click_slates(model, x, y, clicks_ref.NumpySource())
        assert type(info.value).__name__ == case["error"]
        return
    got = clicks_ref.click_slates(model, x, y, clicks_ref.NumpySource())
    want = GOLD[f"case{case['id']}_clicks"]
    assert got.dtype == want.dtype and np.array_equal(got, want)


def _params(fn):
    return [[p.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
            for p in inspect.signature(fn).parameters.values()]


def test_public_signatures_match_the_reference():
    with open(os.path.join(ROOT, "tests", "golden", "click_signatures.json")) as fh:
        ref = json.load(fh)
    for name, params in ref.items():
        if name == "click_on_slates":
            assert _params(click_models.click_on_slates) == params
        elif name == "metrics_on_clicked_slates":
            assert _params(inference.metrics_on_clicked_slates)[:len(params)] == params
        else:
            assert _params(getattr(click_models, name).__init__) == params, name


def test_compile_flattens_breadth_first_and_refuses_unknown_models():
    m = click_models.DiverseClicksModel(click_models.MultipleClickModel(
        [click_models.OnlyRelevantClickModel(1), click_models.BaseCascadeModel(0.5, 2)], [0.4, 0.6]), 0.3)
    cm = click_models.compile_click_model(click_models.MaskedRemainMasked(m))
    kinds = [n.kind for n in cm.nodes]
    assert kinds == [click_models.DIVERSE, click_models.MULTIPLE, click_models.RELEVANT, click_models.CASCADE]
    assert (cm.nodes[0].first_child, cm.nodes[0].n_children) == (1, 1)
    assert (cm.nodes[1].first_child, cm.nodes[1].n_children) == (2, 2)
    assert list(cm.values)[:2] == [0.4, 1.0] and cm.etas == [0.5]
    assert cm.needs_x and cm.random
    assert clicks_ref.number_nodes(m)[id(m.inner_click_model.inner_click_models[1])] == 3

    class Custom(click_models.ClickModel):
        pass
    with pytest.raises(NotImplementedError):
        click_models.compile_click_model(Custom())
    with pytest.raises(NotImplementedError):
        click_models.compile_click_model(click_models.ConditionedClickModel([Custom()], np.sum))
    with pytest.raises(NotImplementedError):
        click_models.compile_click_model(click_models.EverythingButDuplicatesClickModel(1.0, "cosine"))
