"""Layer widths that are not multiples of 4, on the host (no GPU): every FC / feed-forward weight is stored in the flat
buffer as a zero-padded [round_up(out, 4), round_up(in, 4)] block, every bias, LayerNorm vector and learned positional
row padded to round_up(width, 4), and the head's weight as [d_output, round_up(d_model, 4)] (DESIGN.md 4.16); the
attention linears keep the reference's layout.  The parameters are views of the real part, so the model keeps the
reference's state_dict keys, order, shapes and seeded initialisation; the pads are +0.  bf16 mode keeps its rules,
and input_norm still needs n_features % 4 == 0."""
import ctypes
import json

import numpy as np
import pytest
import torch

# n_features, sizes, activation, d_output
FC_SHAPES = [(10, [10], None, 1), (10, [10, 6], "ReLU", 1), (46, [50, 30], "ReLU", 1), (46, [50, 30], "Tanh", 3),
             (46, [100, 50], "Sigmoid", 1), (46, [46], None, 1), (20, [1], None, 1), (20, [7, 8193 - 2, 3], "ReLU", 2)]
GOLDEN = ["f10s10", "f46s10_6", "f46s50_30t", "f46s50_30s", "f46s46_64e", "d10h2", "d46h2f30", "d130h2", "d6h3o3"]


def _make(F, sizes, act, d_output, transformer=None, **kw):
    from allrank_b200.model import make_model
    return make_model(fc_model={"sizes": list(sizes), "input_norm": False, "activation": act, "dropout": 0.1},
                      transformer=transformer, post_model={"d_output": d_output, "output_activation": None},
                      n_features=F, **kw)


def _param_count(m):
    from allrank_b200 import _lib
    L = _lib.lib()
    L.arb_scorer_param_count.restype = ctypes.c_int64
    return int(L.arb_scorer_param_count(ctypes.byref(m._cfg))), L.arb_last_error().decode()


def _pad4(n):
    return (n + 3) // 4 * 4


def _ids(shapes):
    return [f"F{F}-{'x'.join(map(str, s))}-{a}-o{o}" for F, s, a, o in shapes]


@pytest.mark.parametrize("F,sizes,act,d_output", FC_SHAPES, ids=_ids(FC_SHAPES))
def test_fc_models_pack_like_the_reference_with_zero_pads(F, sizes, act, d_output):
    from oracle.scorer_ref import make_ref_model
    ref = make_ref_model(F, list(sizes), 0, 1, 4, d_output=d_output, fc_activation=act, seed=5)
    m = _make(F, sizes, act, d_output)
    want = [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == want
    n, err = _param_count(m)
    dims = [_pad4(F)] + [_pad4(s) for s in sizes]
    expect = sum(a * b + a for a, b in zip(dims[1:], dims[:-1])) + d_output * _pad4(sizes[-1]) + d_output
    assert n == expect, (n, expect, err)
    m.load_state_dict(ref.state_dict())
    m._pack(torch.device("cpu"))
    flat = m.flat_parameters
    assert flat.numel() == n
    got = m.state_dict()
    assert [(k, tuple(v.shape)) for k, v in got.items()] == want
    for k, v in ref.state_dict().items():
        assert torch.equal(got[k], v), k
    # everything outside the parameters' views is +0
    covered = torch.zeros(n, dtype=torch.bool)
    for p in m.parameters():
        idx = torch.arange(n, dtype=torch.float32)
        view = idx.as_strided(p.shape, p.stride(), p.storage_offset())
        covered[view.long().flatten()] = True
    rest = flat[~covered]
    assert rest.numel() == n - sum(p.numel() for p in m.parameters())
    assert torch.equal(rest.view(torch.int32), torch.zeros_like(rest).view(torch.int32))


def test_multiple_of_4_layouts_are_unchanged():
    """Models whose widths are multiples of 4 keep the parameter count they always had: the plain sum of the
    parameters' sizes (FC-only) and contiguous parameters."""
    for F, sizes, dout in [(136, [128], 1), (20, [32, 48, 32], 3), (44, [8], 1)]:
        m = _make(F, sizes, None, dout)
        n, _ = _param_count(m)
        assert n == sum(p.numel() for p in m.parameters())
        m._pack(torch.device("cpu"))
        assert all(p.is_contiguous() for p in m.parameters())


def test_odd_fc_hidden_widths_pack_in_front_of_an_encoder():
    from oracle.scorer_ref import make_ref_model
    ref = make_ref_model(46, [46, 64], 1, 4, 128, fc_activation="ReLU", seed=5)
    m = _make(46, [46, 64], "ReLU", 1, {"N": 1, "d_ff": 128, "h": 4, "positional_encoding": None, "dropout": 0.1})
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == \
        [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    m.load_state_dict(ref.state_dict())
    m._pack(torch.device("cpu"))
    for k, v in ref.state_dict().items():
        assert torch.equal(m.state_dict()[k], v), k


ENC_SHAPES = [(10, 2, 20, None), (46, 2, 92, None), (130, 2, 262, None), (254, 2, 508, None), (6, 3, 14, None),
              (64, 4, 30, None), (128, 2, 258, None), (10, 2, 22, ("learned", 20)), (46, 2, 30, ("fixed", 20))]


@pytest.mark.parametrize("d,h,dff,pos", ENC_SHAPES, ids=[f"d{d}-h{h}-f{f}-{p and p[0]}" for d, h, f, p in ENC_SHAPES])
def test_encoders_of_any_width_pack_like_the_reference_with_zero_pads(d, h, dff, pos):
    """Attention linears in the reference's layout, everything from b_o on at dw = round_up(d, 4) and
    fw = round_up(d_ff, 4) (16-byte aligned), the learned table [rows, dw]; every pad is +0."""
    from oracle.scorer_ref import make_ref_model
    ref = make_ref_model(46, [d], 2, h, dff, seed=5, positional=pos)
    pe = None if pos is None else {"strategy": pos[0], "max_indices": pos[1]}
    m = _make(46, [d], None, 1, {"N": 2, "d_ff": dff, "h": h, "positional_encoding": pe, "dropout": 0.1})
    want = [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == want
    n, err = _param_count(m)
    assert n > 0, err
    m.load_state_dict(ref.state_dict())
    m._pack(torch.device("cpu"))
    flat = m.flat_parameters
    assert flat.numel() == n
    for k, v in ref.state_dict().items():
        assert torch.equal(m.state_dict()[k], v), k
    covered = torch.zeros(n, dtype=torch.bool)
    for p in m.parameters():
        covered[torch.arange(n).as_strided(p.shape, p.stride(), p.storage_offset()).flatten()] = True
    rest = flat[~covered]
    assert torch.equal(rest.view(torch.int32), torch.zeros_like(rest).view(torch.int32))
    if d % 4 == 0 and dff % 4 == 0:
        assert n - sum(p.numel() for p in m.parameters()) < 8      # only the encoder section's alignment


def test_a_fixed_table_at_an_odd_d_model_fails_as_in_the_reference():
    """positional.py's sinusoidal table cannot be built at an odd width; neither model invents one."""
    from oracle.scorer_ref import make_ref_model
    with pytest.raises(RuntimeError):
        make_ref_model(46, [9], 1, 3, 18, seed=5, positional=("fixed", 20))
    with pytest.raises(RuntimeError):
        _make(46, [9], None, 1, {"N": 1, "d_ff": 18, "h": 3, "positional_encoding": {"strategy": "fixed",
                                                                                   "max_indices": 20}, "dropout": 0.0})


def test_fc_widths_beyond_8192_are_refused():
    m = _make(20, [8193, 8], None, 1)
    n, err = _param_count(m)
    assert n <= 0 and "8192" in err, (n, err)


def test_bf16_and_input_norm_keep_their_refusals():
    with pytest.raises(NotImplementedError, match="multiples of 8"):
        _make(46, [46], None, 1, {"N": 1, "d_ff": 92, "h": 2, "positional_encoding": None, "dropout": 0.0},
              compute_dtype="bf16")
    from allrank_b200.model import make_model
    with pytest.raises(NotImplementedError, match="input_norm"):
        make_model(fc_model={"sizes": [10], "input_norm": True, "activation": None, "dropout": 0.0},
                   transformer=None, post_model={"d_output": 1}, n_features=10)


def golden_model(g, name):
    """make_model under the generator's seeds (tools/make_golden_odd_widths.py)."""
    from allrank_b200.model import make_model
    m = json.loads(str(g[name + ":model"]))
    torch.manual_seed(87)
    model = make_model(fc_model=m["fc_model"], transformer=m["transformer"], post_model=m["post_model"],
                       n_features=int(g[name + ":F"]))
    gen = torch.Generator().manual_seed(88)
    with torch.no_grad():
        for _, p in model.named_parameters():
            if p.dim() == 1:
                p.add_(0.1 * torch.randn(p.shape, generator=gen))
    return model


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_models_rebuild_the_reference_initialisation(golden, name):
    """tests/golden/scorer_odd_widths.npz: make_model under the generator's seeds gives the reference's parameter
    values (checksums of every tensor) and state_dict keys, before and after packing into the padded flat buffer."""
    g = golden("scorer_odd_widths")
    model = golden_model(g, name)
    keys = [k.split(":c:")[1] for k in g.files if k.startswith(name + ":c:")]
    for packed in (False, True):
        if packed:
            model._pack(torch.device("cpu"))
        sd = model.state_dict()
        assert list(sd.keys()) == keys
        for k, v in sd.items():
            got = np.array([v.double().sum().item(), v.double().abs().sum().item()])
            assert np.array_equal(got, g[name + ":c:" + k]), k
