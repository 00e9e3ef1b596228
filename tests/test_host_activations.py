"""The activation classes of the FC block and the output head, on the host (no GPU): make_model accepts every
parameter-free elementwise class of torch.nn.modules.activation whose derivative follows from its output, in both
positions, with the reference's state_dict; every other class raises NotImplementedError; the ids of the first four
activations are those of the earlier ABI."""
import pytest
import torch

NEW = ["LeakyReLU", "ELU", "CELU", "SELU", "Softplus", "Softsign", "Hardtanh", "ReLU6", "Hardsigmoid", "LogSigmoid",
       "Hardshrink", "Softshrink"]
REFUSED = ["GELU", "SiLU", "Mish", "Hardswish", "Tanhshrink", "PReLU", "RReLU", "GLU", "Softmax", "Softmin",
           "LogSoftmax", "Softmax2d", "Threshold", "MultiheadAttention"]


def _make(act, out_act, transformer=None, d_output=1):
    from allrank_b200.model import make_model
    return make_model(fc_model={"sizes": [50, 30], "input_norm": False, "activation": act, "dropout": 0.1},
                      transformer=transformer, post_model={"d_output": d_output, "output_activation": out_act},
                      n_features=46)


@pytest.mark.parametrize("name", NEW)
@pytest.mark.parametrize("where", ["fc", "output"])
def test_make_model_accepts_the_activation_with_the_reference_state_dict(name, where):
    from oracle.scorer_ref import make_ref_model
    act, out_act = (name, None) if where == "fc" else ("ReLU", name)
    m = _make(act, out_act)
    ref = make_ref_model(46, [50, 30], 0, 1, 4, output_activation=out_act, fc_activation=act, seed=5)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == \
        [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    assert (m.fc_activation, m.output_activation) == (act, out_act)
    m.load_state_dict(ref.state_dict(), strict=True)


@pytest.mark.parametrize("name", NEW)
def test_encoder_and_multi_output_models_accept_the_activation(name):
    tr = {"N": 1, "d_ff": 64, "h": 2, "positional_encoding": None, "dropout": 0.1}
    m = _make(name, name, transformer=tr, d_output=3)
    assert tuple(m.output_layer.w_1.weight.shape) == (3, 30)


@pytest.mark.parametrize("name", REFUSED)
@pytest.mark.parametrize("where", ["fc", "output"])
def test_other_activation_classes_raise_not_implemented(name, where):
    act, out_act = (name, None) if where == "fc" else (None, name)
    with pytest.raises(NotImplementedError, match="derivative"):
        _make(act, out_act)


def test_ids_of_the_first_four_activations_are_unchanged():
    from allrank_b200.model import _ACTS
    assert {k: _ACTS[k] for k in (None, "Tanh", "Sigmoid", "ReLU")} == {None: 0, "Tanh": 1, "Sigmoid": 2, "ReLU": 3}
    ids = [_ACTS[n] for n in NEW]
    assert ids == list(range(5, 17)) and 4 not in _ACTS.values()


def test_the_reference_names_are_torch_classes_without_parameters():
    """Every accepted name is a class of torch.nn.modules.activation that constructs without arguments and owns no
    parameter, so the reference's state_dict has no entry for it."""
    import torch.nn.modules.activation as A
    for n in NEW:
        mod = getattr(A, n)()
        assert not list(mod.parameters()), n
        z = torch.linspace(-5, 5, 11)
        assert mod(z).shape == z.shape
