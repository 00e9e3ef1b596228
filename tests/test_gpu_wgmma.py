"""The fp32 K-major GEMMs on warpgroup MMA (wgmma) and the scorer's TF32 weight copy: the forward rounds the weights
(and their transposes, the K-major operands of the input gradients) into its workspace on every call, CUDA-graph
replays included, so the products never see stale weights; ragged N / K edges; truncation mode."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

CFG = dict(fc_model={"sizes": [128], "input_norm": False, "activation": None, "dropout": 0.0},
           transformer={"N": 2, "d_ff": 256, "h": 4, "positional_encoding": None, "dropout": 0.0},
           post_model={"d_output": 1, "output_activation": None}, n_features=136)


def _model(seed=3):
    from allrank_b200.model import make_model
    torch.manual_seed(seed)
    return make_model(**CFG).cuda().train()


def _fresh_copy(model):
    fresh = _model(seed=99)
    fresh.load_state_dict(model.state_dict())
    return fresh


def test_scores_after_adam_steps_equal_a_fresh_model_with_the_same_weights():
    from allrank_b200.losses import approxNDCGLoss
    from allrank_b200.optim import FlatAdam
    from allrank_b200.synth import make_slates
    batches = [make_slates(16, 48, 136, seed=20 + k) for k in range(4)]
    batches = [(x.cuda(), y.cuda()) for x, y, _ in batches]
    model = _model()
    opt = FlatAdam(model, lr=1e-2)
    for x, y in batches[:3]:
        loss = approxNDCGLoss(model(x, y == -1, None), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
    x, y = batches[3]
    with torch.no_grad():
        want = _fresh_copy(model)(x, y == -1, None)
        got = model(x, y == -1, None)
    assert torch.equal(got, want)


def test_graph_replays_use_the_weights_of_the_latest_adam_step():
    from allrank_b200.graph import GraphedTrainStep
    from allrank_b200.losses import approxNDCGLoss
    from allrank_b200.optim import FlatAdam
    from allrank_b200.synth import make_slates
    batches = [make_slates(16, 48, 136, seed=30 + k) for k in range(4)]
    batches = [(x.cuda(), y.cuda()) for x, y, _ in batches]
    model = _model()
    opt = FlatAdam(model, lr=1e-2, capturable=True)
    step = GraphedTrainStep(model, approxNDCGLoss, opt, *batches[0], warmup=2)
    for x, y in batches[:3]:
        step(x, y)
    x, y = batches[3]
    fresh = _fresh_copy(model)             # the weights after the last replay's Adam step
    got = step(x, y).clone()               # this replay's loss is computed with those weights
    with torch.no_grad():
        want = approxNDCGLoss(fresh(x, y == -1, None), y)
    assert torch.equal(got, want), (got.item(), want.item())


def test_input_gradient_at_136_features_matches_the_oracle():
    """d loss / d x goes through the FC layer's input-gradient product: N = 136, a ragged last column tile."""
    from allrank_b200.losses import approxNDCGLoss
    from allrank_b200.synth import make_slates
    from oracle import losses_ref
    from oracle.scorer_ref import make_ref_model
    torch.manual_seed(0)
    ref = make_ref_model(136, [128], 2, 4, 256).train()
    mine = _model()
    mine.load_state_dict(ref.state_dict())
    x, y, idx = make_slates(8, 240, 136, seed=7)
    xr = x.clone().requires_grad_(True)
    losses_ref.approxNDCGLoss(ref(xr, y == -1, idx), y).backward()
    xm = x.cuda().requires_grad_(True)
    approxNDCGLoss(mine(xm, y.cuda() == -1, None), y.cuda()).backward()
    real = ~(y == -1)
    g, g_ref = xm.grad.cpu()[real], xr.grad[real]
    rel = (g - g_ref).norm().item() / g_ref.norm().item()
    assert rel < 5e-2, rel


@pytest.fixture(scope="module")
def gemm():
    from allrank_b200 import _lib
    c_p, c_i, c_f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float
    _lib.register("arb_gemm_tf32", c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_i, c_i, c_i, c_i, ctypes.c_int64,
                                         ctypes.c_int64, ctypes.c_int64, c_i, c_i, c_f, c_i, c_p])
    _lib.register("arb_set_tf32_round_on_load", None, [ctypes.c_int32])

    def call(A, B, C, M, N, K, block_n):
        rc = _lib.lib().arb_gemm_tf32(_lib.ptr(A), _lib.ptr(B), _lib.ptr(C), None, None, M, N, K, 0, 0, 1, 0, 0, 0,
                                      block_n, 0, 1.0, 1, _lib.stream_ptr())
        _lib.check(rc, "arb_gemm_tf32")
        torch.cuda.synchronize()
    return call


def _tf32(x, nearest):
    """fp32 -> tf32 on the host: round to nearest even, or truncate."""
    b = x.view(torch.int32)
    if nearest:
        b = b + 0xFFF + ((b >> 13) & 1)
    return (b & ~0x1FFF).view(torch.float32)


@pytest.mark.parametrize("block_n", [32, 64, 128])
def test_ragged_last_k_block_and_truncation_mode(gemm, block_n):
    """K = 136: the last k-block holds 8 of 32 columns (the rest zero-filled by TMA).  With rounding on the product is
    the one of the nearest-rounded operands, with it off the one of the truncated operands (each within fp32
    accumulation error, far below the gap between the two)."""
    from allrank_b200 import _lib
    torch.manual_seed(block_n)
    M, N, K = 300, 200, 136
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(N, K, device="cuda")
    out = {}
    try:
        for nearest in (1, 0):
            _lib.lib().arb_set_tf32_round_on_load(nearest)
            C = torch.full((M, N), float("nan"), device="cuda")
            gemm(A, B, C, M, N, K, block_n)
            out[nearest] = C
    finally:
        _lib.lib().arb_set_tf32_round_on_load(1)
    scale = A.abs().double() @ B.abs().double().t()
    for nearest, C in out.items():
        ref = _tf32(A, nearest).double() @ _tf32(B, nearest).double().t()
        other = _tf32(A, 1 - nearest).double() @ _tf32(B, 1 - nearest).double().t()
        err = ((C.double() - ref).abs() / scale).max().item()
        gap = ((other - ref).abs() / scale).max().item()
        assert err < 1e-5 and gap > 10 * err, (nearest, err, gap)
