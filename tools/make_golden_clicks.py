"""Golden data for the click models: the UNMODIFIED reference's `click_on_slates` (allrank/click_models/click_utils.py)
on seeded slates -> tests/golden/clicks.npz, and the public signatures -> tests/golden/click_signatures.json.

    python tools/make_golden_clicks.py          (needs oracle/_ref: python oracle/install_reference.py)

Every case is a model spec ({"name", "args"} nested like allRank's click_model config), a dataset, the numpy seed set
right before the call and either the clicks [B,S] (float32, -1 at padding) or the exception type raised.  Random
models consume np.random in the reference's own order, which oracle.clicks_ref.NumpySource replays.
"""
import inspect
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def datasets():
    rng = np.random.RandomState(2024)
    out = {}

    def make(B, S, F, n_real, grid):
        x = (rng.randint(0, 3, (B, S, F)).astype(np.float32) if grid else rng.randn(B, S, F).astype(np.float32))
        y = np.full((B, S), -1.0, dtype=np.float32)
        for b, n in enumerate(n_real):
            pos = np.sort(rng.choice(S, n, replace=False))           # padding anywhere, not only at the end
            y[b, pos] = rng.randint(0, 5, n).astype(np.float32)
            if n >= 4:                                                # an exact duplicate row
                x[b, pos[3]] = x[b, pos[1]]
        x[y == -1] = 0.0
        return x, y

    out["d4"] = make(8, 12, 4, [0, 1, 2, 12, 9, 7, 5, 11], grid=True)
    out["d4f"] = make(6, 12, 4, [3, 12, 9, 7, 5, 11], grid=True)
    out["d4two"] = make(5, 9, 4, [2, 2, 2, 2, 2], grid=False)
    out["d46"] = make(6, 20, 46, [20, 17, 8, 13, 4, 19], grid=False)
    out["d136"] = make(5, 24, 136, [24, 21, 9, 16, 5], grid=False)
    return out


def M(name, **args):
    return {"name": name, "args": args}


REL = lambda t: M("OnlyRelevantClickModel", relevancy_threshold=t)   # noqa: E731
CAS = lambda e, t: M("BaseCascadeModel", eta=e, threshold=t)          # noqa: E731
FIX = lambda p: M("FixedClickModel", click_positions=p)              # noqa: E731
DUP = lambda m, metric: M("EverythingButDuplicatesClickModel", duplicate_margin=m, metric=metric)  # noqa: E731
DIV = lambda inner, q: M("DiverseClicksModel", inner_click_model=inner, q_percentile=q)           # noqa: E731

DETERMINISTIC = [
    (REL(2), "d4"), (REL(0.5), "d46"), (CAS(0, 2), "d4"), (CAS(0, 0), "d46"), (FIX([0, 2, -1]), "d4f"),
    (FIX([-2]), "d46"), (M("MaxClicksModel", inner_click_model=REL(1), max_clicks=2), "d4"),
    (M("MaxClicksModel", inner_click_model=REL(1), max_clicks=None), "d46"),
    (M("ConditionedClickModel", inner_click_models=[REL(1), FIX([0, 1, 2])], combiner="np.all"), "d4f"),
    (M("ConditionedClickModel", inner_click_models=[REL(3), FIX([1])], combiner="np.any"), "d4f"),
    (DUP(1.0, "euclidean"), "d4f"), (DUP(2.0, "sqeuclidean"), "d4f"), (DUP(3.0, "cityblock"), "d46"),
    (DUP(1.0, "chebyshev"), "d4f"), (DUP(9.0, "euclidean"), "d46"), (DUP(0.0, "euclidean"), "d136"),
    (DIV(REL(1), 0.0), "d4"), (DIV(REL(1), 0.25), "d4"), (DIV(REL(1), 0.5), "d4"), (DIV(REL(1), 0.9), "d4"),
    (DIV(REL(1), 1.0), "d4"), (DIV(REL(1), 0.5), "d46"), (DIV(REL(0), 0.25), "d136"), (DIV(CAS(0, 1), 0.5), "d136"),
    (DIV(CAS(0, 2), 0.9), "d46"), (DIV(M("RandomClickModel", n_clicks=2), 0.5), "d4two"),
    (M("MultipleClickModel", inner_click_models=[FIX([99]), REL(1)], probabilities=[0.0, 1.0]), "d4"),
    (M("MultipleClickModel", inner_click_models=[REL(2), FIX([99])], probabilities=[1.0, 0.0]), "d4"),
    (M("MaxClicksModel", inner_click_model=DIV(REL(0), 0.5), max_clicks=3), "d46"),
]
ERRORS = [(FIX([5]), "d4"), (FIX([-13]), "d4f"), (M("RandomClickModel", n_clicks=3), "d4"), (DUP(1.0, "euclidean"), "d4"),
          (M("ConditionedClickModel", inner_click_models=[REL(1), FIX([2])], combiner="np.any"), "d4")]
RANDOM = [
    (M("RandomClickModel", n_clicks=2), "d4f"), (CAS(1, 1), "d46"), (CAS(0.5, 2), "d136"),
    (M("MultipleClickModel", inner_click_models=[REL(1), CAS(0.5, 2)], probabilities=[0.3, 0.7]), "d46"),
    (DIV(CAS(0.5, 2), 0.5), "d136"), (M("MaxClicksModel", inner_click_model=M("RandomClickModel", n_clicks=3),
                                         max_clicks=2), "d4f"),
    (M("ConditionedClickModel", inner_click_models=[CAS(1, 1), M("RandomClickModel", n_clicks=2)], combiner="np.any"),
     "d4f"),
]


def reference_classes():
    import allrank.click_models.base as base
    import allrank.click_models.cascade_models as cascade
    import allrank.click_models.click_utils as cu
    import allrank.click_models.duplicate_aware as dup
    classes = {}
    for mod in (base, cascade, dup, cu):
        classes.update({n: getattr(mod, n) for n in dir(mod) if isinstance(getattr(mod, n), type)})
    return classes


CLASS_NAMES = ["ClickModel", "RandomClickModel", "FixedClickModel", "MultipleClickModel", "ConditionedClickModel",
               "MaxClicksModel", "OnlyRelevantClickModel", "BaseCascadeModel", "DiverseClicksModel",
               "EverythingButDuplicatesClickModel", "MaskedRemainMasked"]


def params(fn):
    return [[p.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
            for p in inspect.signature(fn).parameters.values()]


def main():
    from oracle.clicks_ref import build_model
    from oracle.install_reference import import_path, installed
    if not installed():
        raise SystemExit("oracle/_ref is missing: python oracle/install_reference.py")
    sys.path[:0] = import_path()
    import allrank.click_models.click_utils as cu
    import allrank.inference.inference_utils as iu
    classes = reference_classes()
    data = datasets()
    arrays = {f"{k}_{part}": v for k, (x, y) in data.items() for part, v in (("x", x), ("y", y))}
    cases = []
    for kind, table in (("deterministic", DETERMINISTIC), ("error", ERRORS), ("random", RANDOM)):
        for spec, ds in table:
            k = len(cases)
            seed = 1000 + k
            x, y = data[ds]
            np.random.seed(seed)
            case = {"id": k, "kind": kind, "spec": spec, "data": ds, "seed": seed}
            try:
                _, clicks = cu.click_on_slates((torch.tensor(x), torch.tensor(y)), build_model(spec, classes),
                                               include_empty=True)
                arrays[f"case{k}_clicks"] = np.stack(clicks).astype(np.float32)
                case["error"] = None
            except Exception as exc:        # noqa: BLE001 -- the exception type is the golden value
                case["error"] = type(exc).__name__
            assert (case["error"] is None) == (kind != "error"), (spec, case["error"])
            cases.append(case)
    arrays["cases"] = np.array(json.dumps(cases))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "clicks.npz"), **arrays)
    sigs = {n: params(classes[n].__init__) for n in CLASS_NAMES if n != "ClickModel"}
    sigs["click_on_slates"] = params(cu.click_on_slates)
    sigs["metrics_on_clicked_slates"] = params(iu.metrics_on_clicked_slates)
    with open(os.path.join(ROOT, "tests", "golden", "click_signatures.json"), "w") as fh:
        json.dump(sigs, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print(f"wrote {len(cases)} cases")


if __name__ == "__main__":
    main()
