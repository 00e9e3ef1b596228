"""The scorer's head-width limit on the host (no GPU): the C ABI lays out the parameters of one- and two-head models up
to 256 columns per head, and refuses wider heads with an error that names the limit (LTRModel raises that as
NotImplementedError when it first packs its parameters)."""
import ctypes

import pytest


def _make(d, h):
    from allrank_b200.model import make_model
    return make_model(fc_model={"sizes": [d], "input_norm": False, "activation": None, "dropout": 0.0},
                      transformer={"N": 1, "d_ff": 2 * d, "h": h, "positional_encoding": None, "dropout": 0.1},
                      post_model={"d_output": 1, "output_activation": None}, n_features=136)


def _param_count(m):
    from allrank_b200 import _lib
    L = _lib.lib()
    L.arb_scorer_param_count.restype = ctypes.c_int64
    return int(L.arb_scorer_param_count(ctypes.byref(m._cfg))), L.arb_last_error().decode()


@pytest.mark.parametrize("d,h", [(136, 1), (192, 1), (256, 1), (320, 2), (512, 2)])
def test_heads_up_to_256_columns_have_a_layout(d, h):
    m = _make(d, h)
    n, _ = _param_count(m)
    assert n >= sum(p.numel() for p in m.parameters())
    lin = m.encoder.layers[0].self_attn.linears
    assert tuple(lin[0].weight.shape) == (d, d) and tuple(lin[3].weight.shape) == (d, d)


@pytest.mark.parametrize("d,h", [(260, 1), (520, 2), (1024, 1)])
def test_heads_wider_than_256_columns_are_refused(d, h):
    n, err = _param_count(_make(d, h))
    assert n <= 0 and "256" in err, (n, err)
