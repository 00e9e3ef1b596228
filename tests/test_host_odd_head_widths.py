"""Head widths d_model / h that are not a multiple of 4, on the host (no GPU): the scorer pads each head to the next
multiple of 4 inside its workspace only, so the model packs with the reference's parameters, state_dict keys and
shapes; bf16 mode still refuses these widths, and padded heads beyond 1024 columns in all are refused with an error
that states the rule."""
import ctypes

import numpy as np
import pytest
import torch

SHAPES = [(144, 8), (96, 32), (136, 8), (100, 4), (260, 2), (1020, 4)]   # widths 18, 3, 17, 25, 130, 255


def _make(d, h, **kw):
    from allrank_b200.model import make_model
    return make_model(fc_model={"sizes": [d], "input_norm": False, "activation": None, "dropout": 0.0},
                      transformer={"N": 2, "d_ff": 2 * d, "h": h, "positional_encoding": None, "dropout": 0.1},
                      post_model={"d_output": 1, "output_activation": None}, n_features=136, **kw)


def _param_count(m):
    from allrank_b200 import _lib
    L = _lib.lib()
    L.arb_scorer_param_count.restype = ctypes.c_int64
    return int(L.arb_scorer_param_count(ctypes.byref(m._cfg))), L.arb_last_error().decode()


@pytest.mark.parametrize("d,h", SHAPES, ids=[f"d{d}-h{h}" for d, h in SHAPES])
def test_models_with_padded_heads_pack_like_the_reference(d, h):
    from oracle.scorer_ref import make_ref_model
    assert (d // h) % 4 != 0
    ref = make_ref_model(136, [d], 2, h, 2 * d)
    m = _make(d, h)
    want = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == want
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in ref.parameters())
    n, err = _param_count(m)
    assert n >= sum(p.numel() for p in m.parameters()), err
    m.load_state_dict(ref.state_dict())
    m._pack(torch.device("cpu"))          # the flat buffer of the C ABI's layout (asserts its length)
    assert m.flat_parameters.numel() == n
    got = m.state_dict()
    assert {k: tuple(v.shape) for k, v in got.items()} == want
    for k, v in ref.state_dict().items():
        assert torch.equal(got[k], v), k


@pytest.mark.parametrize("d,h", SHAPES, ids=[f"d{d}-h{h}" for d, h in SHAPES])
def test_bf16_mode_still_refuses_padded_heads(d, h):
    with pytest.raises(NotImplementedError, match="8, 16, 24 or 32"):
        _make(d, h, compute_dtype="bf16")


@pytest.mark.parametrize("d,h", [(1020, 60), (1000, 40), (1020, 1020)])
def test_padded_heads_beyond_1024_columns_are_refused(d, h):
    cfg = _make_cfg(d, h)
    n, err = _param_count(cfg)
    assert n <= 0 and "1024" in err, (n, err)


def _make_cfg(d, h):
    """A model object carrying only the ScorerConfig (constructing a 1020-head module is slow and not needed)."""
    from allrank_b200.model import ScorerConfig

    class _M:
        _cfg = ScorerConfig(136, d, 1, h, 2 * d, 0, 1e-6, 0.0, 0.0, 0, 0)
    return _M()


@pytest.mark.parametrize("name", ["d144h8", "d96h32"])
def test_golden_models_rebuild_the_reference_initialisation(golden, name):
    """tests/golden/scorer_odd_heads.npz (tools/make_golden_odd_heads.py): make_model under the generator's seeds gives
    the reference's parameter values (checksums of every tensor) and state_dict keys."""
    from tests.test_gpu_attention_odd_widths import _golden_model
    g = golden("scorer_odd_heads")
    sd = _golden_model(g, name).state_dict()
    assert list(sd.keys()) == [k.split(":c:")[1] for k in g.files if k.startswith(name + ":c:")]
    for k, v in sd.items():
        got = np.array([v.double().sum().item(), v.double().abs().sum().item()])
        assert np.array_equal(got, g[name + ":c:" + k]), k
