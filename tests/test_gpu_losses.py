"""CUDA parity of the fused loss kernels (through the C ABI) against the reference's known answers,
the golden vectors produced by the unmodified reference, and the CPU oracle on seeded slates.

Tolerance (BASELINE.json north_star): loss values within 1e-5 relative in fp32; gradients within
1e-5 of the largest reference gradient entry (looser, stated bounds where the reference's own fp32
evaluation noise is larger -- measured against its fp64 run)."""
import ast
import math

import numpy as np
import pytest
import torch

from tests import cases

pytestmark = pytest.mark.gpu

REL = 1e-5


@pytest.fixture(scope="module")
def L():
    from allrank_b200 import losses
    return losses


def dev(x):
    return torch.as_tensor(x, dtype=torch.float32).cuda()


def run(fn, yp, yt, **kw):
    p = dev(yp).clone().requires_grad_(True)
    val = fn(p, dev(yt), **kw)
    val.backward()
    return val.item(), p.grad.cpu().numpy()


@pytest.mark.parametrize("name,kw,yp,yt,expected", cases.LOSS_KNOWN)
def test_known_answers(L, name, kw, yp, yt, expected):
    kw = dict(kw)
    if name == "listMLE":
        kw["perm"] = torch.arange(len(yp))
    val, grad = run(getattr(L, name), [yp], [yt], **kw)
    assert math.isfinite(val) and np.isfinite(grad).all()
    assert val == pytest.approx(expected, rel=1e-5)


@pytest.mark.parametrize("yp,yt,eps", cases.LISTNET_KNOWN)
def test_listnet_closed_form(L, yp, yt, eps):
    val, _ = run(L.listNet, [yp], [yt], eps=eps)
    assert val == pytest.approx(cases.listnet_closed_form(yp, yt, eps), rel=1e-5)


@pytest.mark.parametrize("yp,yt,kw", cases.NEURALNDCG_EQUIV)
def test_neuralndcg_low_temperature_equals_ndcg(L, yp, yt, kw):
    from allrank_b200 import metrics
    val, grad = run(L.neuralNDCG, [yp], [yt], **kw)
    k = kw.get("k")
    expected = metrics.ndcg(dev([yp]), dev([yt]), ats=None if k is None else [k]).mean().item()
    assert math.isfinite(val) and np.isfinite(grad).all()
    assert -val == pytest.approx(expected, rel=1e-5)


def test_golden_losses(L, golden):
    g = golden("losses")
    table = [ast.literal_eval(str(c)) for c in g["cases"]]
    worst = {}
    for key in g["keys"]:
        key = str(key)
        name, kw = table[int(key.split("_")[0][1:])]
        val, grad = run(getattr(L, name), g[key + "_pred"], g[key + "_true"], **kw)
        ref, gref = float(g[key + "_loss32"]), g[key + "_grad32"]
        # the reference's own fp32 rounding noise, measured against its fp64 evaluation where available
        noise = abs(float(g[key + "_loss64"]) - ref) if key + "_loss64" in g.files else 0.0
        # a non-default Sinkhorn tolerance makes the early-exit point matter: the reference tests the whole batch,
        # the kernel each slate, so values agree to a fraction of `tol` only
        tol = (REL + 0.5 * kw.get("tol", 0.0)) * abs(ref) + 2 * noise + 1e-7
        assert abs(val - ref) <= tol, (key, name, kw, val, ref)
        scale = max(np.abs(gref).max(), 1e-12)
        gnoise = np.abs(g[key + "_grad64"] - gref).max() if key + "_grad64" in g.files else 0.0
        gtol = (1e-5 if not name.startswith("neuralNDCG") else 2e-4 + 20 * kw.get("tol", 0.0)) * scale + 2 * gnoise
        err = np.abs(grad - gref).max()
        worst[name] = max(worst.get(name, 0.0), err / scale)
        assert err <= gtol, (key, name, kw, err, scale)
    print("worst relative gradient error per loss:", worst)


def test_golden_listmle(L, golden):
    g = golden("listmle")
    for key in g["keys"]:
        key = str(key)
        perm = torch.tensor(g[key + "_perm"])
        ref, gref = float(g[key + "_loss32"]), g[key + "_grad32"]
        # realised tie order fed through the debug hook: must agree for integer labels too
        val, grad = run(L.listMLE, g[key + "_pred"], g[key + "_true"], perm=perm, order=torch.tensor(g[key + "_order"]))
        assert abs(val - ref) <= REL * abs(ref), key
        assert np.abs(grad - gref).max() <= 1e-5 * np.abs(gref).max() + 1e-7, key
        if key.endswith("distinct"):   # tie-free labels: device sort must give the same value for any shuffle
            val2, grad2 = run(L.listMLE, g[key + "_pred"], g[key + "_true"], perm=perm)
            assert abs(val2 - ref) <= REL * abs(ref), key
            assert np.abs(grad2 - gref).max() <= 1e-5 * np.abs(gref).max() + 1e-7, key
            val3, _ = run(L.listMLE, g[key + "_pred"], g[key + "_true"])
            assert abs(val3 - ref) <= 2 * REL * abs(ref), key


ORACLE_CASES = [
    ("listNet", {}),
    ("approxNDCGLoss", {"alpha": 1.0}),
    ("lambdaLoss", {"weighing_scheme": "ndcgLoss2PP_scheme"}),
    ("lambdaLoss", {"weighing_scheme": "ndcgLoss1_scheme", "k": 20}),
    ("lambdaLoss", {"weighing_scheme": "lambdaRank_scheme", "reduction": "mean", "reduction_log": "natural"}),
    ("neuralNDCG", {"temperature": 1.0}),
]


@pytest.mark.parametrize("name,kw", ORACLE_CASES)
@pytest.mark.parametrize("B,S", [(64, 240), (16, 120), (2, 1251)])
def test_against_oracle_on_synthetic_slates(L, name, kw, B, S):
    from oracle import losses_ref
    from allrank_b200.synth import make_slates, make_scores
    if name == "neuralNDCG":       # the oracle materialises [B,S,S] x 50 iterations under autograd: 2 GB at (2, 1251)
        B = min(B, 8)
    _, y, _ = make_slates(B, S, n_features=1, seed=5)
    yp = make_scores(B, S, seed=6)
    p = yp.clone().double().requires_grad_(True)
    ref = losses_ref.LOSSES[name](p.float() if name == "neuralNDCG" else p, y.double() if name != "neuralNDCG" else y, **kw)
    ref.backward()
    val, grad = run(getattr(L, name), yp, y, **kw)
    gref = p.grad.numpy()
    rel = 1e-5 if name != "neuralNDCG" else 5e-5
    assert abs(val - ref.item()) <= rel * abs(ref.item()) + 1e-7, (val, ref.item())
    scale = np.abs(gref).max()
    gtol = (2e-5 if name != "neuralNDCG" else 5e-4) * scale
    assert np.abs(grad - gref).max() <= gtol, (np.abs(grad - gref).max(), scale)


@pytest.mark.parametrize("name,kw", ORACLE_CASES)
def test_padding_and_item_permutation_invariance(L, name, kw):
    """Size-independent properties at the bench shape: appending padded items and permuting items within
    a slate must not change the loss; gradients permute accordingly (tie-free scores)."""
    from allrank_b200.synth import make_slates, make_scores
    B, S = 32, 240
    _, y, _ = make_slates(B, S, n_features=1, seed=11)
    yp = make_scores(B, S, seed=12)
    if name == "neuralNDCG":
        B = 4
        y, yp = y[:B], yp[:B]
    val, grad = run(getattr(L, name), yp, y, **kw)
    # (1) extra padded columns
    extra = 16
    y2 = torch.cat([y, torch.full((B, extra), -1.0)], dim=1)
    yp2 = torch.cat([yp, torch.randn(B, extra)], dim=1)
    val2, grad2 = run(getattr(L, name), yp2, y2, **kw)
    assert val2 == pytest.approx(val, rel=2e-6)
    assert np.abs(grad2[:, :S] - grad).max() <= 2e-6 * np.abs(grad).max()
    assert (grad2[:, S:] == 0).all()
    # (2) permute the items of every slate (keeps pads as pads); NeuralSort's scaling uses positions of the
    #     valid block, so keep the valid prefix a prefix: permute only inside the valid prefix
    g = torch.Generator().manual_seed(3)
    perm = torch.stack([torch.cat([torch.randperm(int((y[b] >= 0).sum()), generator=g),
                                   torch.arange(int((y[b] >= 0).sum()), S)]) for b in range(B)])
    val3, grad3 = run(getattr(L, name), yp.gather(1, perm), y.gather(1, perm), **kw)
    assert val3 == pytest.approx(val, rel=5e-6)
    back = np.take_along_axis(grad, perm.numpy(), axis=1)
    assert np.abs(grad3 - back).max() <= 1e-5 * np.abs(grad).max() + 1e-9


def test_error_conventions(L):
    p, t = dev([[0.5, 0.3]]), dev([[1.0, 0.0]])
    with pytest.raises(ValueError):
        L.lambdaLoss(p, t, reduction="median")
    with pytest.raises(ValueError):
        L.lambdaLoss(p, t, reduction_log="decimal")
    with pytest.raises(KeyError):
        L.lambdaLoss(p, t, weighing_scheme="nope")
    with pytest.raises(Exception):
        L.listNet(torch.tensor([[0.5, 0.3]]), torch.tensor([[1.0, 0.0]]))   # CPU tensors: no fallback


def test_inputs_are_not_modified_and_eval_mode_skips_grad(L):
    from allrank_b200.synth import make_slates, make_scores
    _, y, _ = make_slates(8, 60, n_features=1, seed=1)
    yp = make_scores(8, 60, seed=2)
    a, b = yp.cuda(), y.cuda()
    a0, b0 = a.clone(), b.clone()
    for fn in (L.listNet, L.listMLE, L.approxNDCGLoss, L.lambdaLoss, L.neuralNDCG):
        with torch.no_grad():
            v = fn(a, b)
        assert not v.requires_grad and torch.isfinite(v)
    assert torch.equal(a, a0) and torch.equal(b, b0)


def test_all_padded_or_no_relevant_slates(L):
    y = dev([[0.0, 0.0, 0.0, -1.0], [1.0, 0.0, 2.0, -1.0]])
    p = dev([[0.3, 0.1, 0.2, 0.0], [0.5, 0.4, 0.1, 0.9]])
    for fn in (L.approxNDCGLoss, L.lambdaLoss, L.neuralNDCG, L.listMLE, L.listNet):
        q = p.clone().requires_grad_(True)
        v = fn(q, y)
        v.backward()
        assert torch.isfinite(v) and torch.isfinite(q.grad).all()
    # neuralNDCG with every slate dead returns 0 (neuralNDCG.py:66-67)
    z = L.neuralNDCG(p, dev([[0.0, 0.0, 0.0, -1.0], [0.0, 0.0, -1.0, -1.0]]))
    assert z.item() == 0.0


def test_stochastic_neuralndcg_statistics(L):
    """Gumbel-perturbed NeuralSort (loss_utils.py:84-112): the RNG stream cannot match the reference, so parity is
    statistical -- with beta -> 0 it must reproduce the deterministic loss of log-transformed scores, it must be
    finite with a finite gradient, and its mean over many samples must sit close to the small-beta value."""
    from allrank_b200.synth import make_slates, make_scores
    _, y, _ = make_slates(6, 40, n_features=1, seed=41, mean_len=30, std_len=6)
    yp = make_scores(6, 40, seed=42)
    p = dev(yp).clone().requires_grad_(True)
    t = dev(y)
    torch.manual_seed(0)
    v = L.neuralNDCG(p, t, stochastic=True, n_samples=64, beta=0.1, temperature=1.0)
    v.backward()
    assert torch.isfinite(v) and torch.isfinite(p.grad).all() and p.grad.abs().max() > 0
    # beta = 0: every sample is the deterministic loss of log(scores + |min|)
    det_scores = torch.log(p.detach() + p.detach().min().abs() + 1e-10)
    ref = L.neuralNDCG(det_scores, t, temperature=1.0)
    zero = L.neuralNDCG(p.detach(), t, stochastic=True, n_samples=3, beta=0.0, temperature=1.0)
    assert zero.item() == pytest.approx(ref.item(), rel=1e-5)
    small = L.neuralNDCG(p.detach(), t, stochastic=True, n_samples=256, beta=0.01, temperature=1.0)
    assert abs(small.item() - ref.item()) < 0.02
    # the transposed name is the same bilinear form
    a = L.neuralNDCG(p.detach(), t, temperature=0.7, k=7)
    b = L.neuralNDCG_transposed(p.detach(), t, temperature=0.7, k=7)
    assert a.item() == b.item()


def test_golden_bce_and_padding(L, golden):
    g = golden("bce")
    for key in g["keys"]:
        key = str(key)
        val, grad = run(L.bce, g[key + "_pred"], g[key + "_true"])
        ref, gref = float(g[key + "_loss32"]), g[key + "_grad32"]
        assert abs(val - ref) <= REL * abs(ref), key
        assert np.abs(grad - gref).max() <= 1e-5 * np.abs(gref).max(), key
        # appended padded items (label -1) are ignored -- the intended semantics of bce.py:24-25
        b, s = g[key + "_pred"].shape
        yp2 = np.concatenate([g[key + "_pred"], np.full((b, 3), 0.5, dtype=np.float32)], axis=1)
        yt2 = np.concatenate([g[key + "_true"], np.full((b, 3), -1.0, dtype=np.float32)], axis=1)
        val2, grad2 = run(L.bce, yp2, yt2)
        assert val2 == pytest.approx(val, rel=1e-6)
        assert (grad2[:, s:] == 0).all()


@pytest.mark.parametrize("name,kw", [("rankNet", {}), ("rankNet_weightByGTDiff", {}), ("binary_listNet", {}),
                                     ("pointwise_rmse", {"no_of_levels": 4})])
def test_next_row_losses_against_oracle_at_bench_shape(L, name, kw):
    from oracle import losses_ref
    from allrank_b200.synth import make_slates, make_scores
    B, S = 32, 240
    _, y, _ = make_slates(B, S, n_features=1, seed=51)
    yp = make_scores(B, S, seed=52)
    p = yp.clone().double().requires_grad_(True)
    ref = losses_ref.LOSSES[name](p, y.double(), **kw)
    ref.backward()
    val, grad = run(getattr(L, name), yp, y, **kw)
    assert abs(val - ref.item()) <= 1e-5 * abs(ref.item())
    assert np.abs(grad - p.grad.numpy()).max() <= 2e-5 * np.abs(p.grad.numpy()).max()


@pytest.mark.parametrize("yp,yt,n,expected", cases.ORDINAL_KNOWN)
def test_ordinal_known_answers(L, yp, yt, n, expected):
    val, grad = run(L.ordinal, [yp], [yt], n=n)
    assert math.isfinite(val) and np.isfinite(grad).all()
    assert val == pytest.approx(expected, rel=1e-5)


def test_with_ordinals_known_answer(L):
    y, n, expected = cases.WITH_ORDINALS_KNOWN
    assert L.with_ordinals(dev([y]), n).tolist() == [expected]
    assert L.with_ordinals(dev([[1.0, cases.PAD]]), 2).tolist() == [[[1.0, 0.0], [cases.PAD, cases.PAD]]]


def test_golden_ordinal_and_padding(L, golden):
    g = golden("ordinal")
    for key in g["keys"]:
        key = str(key)
        n = int(key.split("_")[0][1:])
        val, grad = run(L.ordinal, g[key + "_pred"], g[key + "_true"], n=n)
        ref, gref = float(g[key + "_loss32"]), g[key + "_grad32"]
        assert abs(val - ref) <= REL * abs(ref), key
        assert np.abs(grad - gref).max() <= 1e-5 * np.abs(gref).max(), key
        # appended padded items (label -1) change nothing: they add no BCE terms and no valid items (ordinal.py:40-48)
        b, s, _ = g[key + "_pred"].shape
        yp2 = np.concatenate([g[key + "_pred"], np.full((b, 3, n), 0.5, dtype=np.float32)], axis=1)
        yt2 = np.concatenate([g[key + "_true"], np.full((b, 3), -1.0, dtype=np.float32)], axis=1)
        val2, grad2 = run(L.ordinal, yp2, yt2, n=n)
        assert val2 == pytest.approx(val, rel=1e-6)
        assert (grad2[:, s:] == 0).all()
        assert np.array_equal(grad2[:, :s], grad)


def test_ordinal_against_oracle_at_bench_shape(L):
    from oracle import losses_ref
    from allrank_b200.synth import make_slates
    B, S, n = 64, 240, 4
    _, y, _ = make_slates(B, S, n_features=1, seed=61)
    prob = torch.sigmoid(2.0 * torch.randn(B, S, n, generator=torch.Generator().manual_seed(62)))
    p = prob.clone().double().requires_grad_(True)
    ref = losses_ref.ordinal(p, y.double(), n)
    ref.backward()
    val, grad = run(L.ordinal, prob, y, n=n)
    assert abs(val - ref.item()) <= 1e-5 * abs(ref.item())
    assert np.abs(grad - p.grad.numpy()).max() <= 2e-5 * np.abs(p.grad.numpy()).max()
    assert (grad[(y == -1).numpy()] == 0).all()


def test_ordinal_saturated_probabilities_follow_bceloss(L):
    """p = 0 / p = 1: nn.BCELoss (what ordinal.py:42 calls) clamps the logs at -100 and its backward divides by
    max(p(1-p), 1e-12); the kernel follows both conventions."""
    y = torch.tensor([[3.0, 0.0, 1.0]])
    prob = torch.tensor([[[0.0, 1.0, 0.3], [0.0, 1.0, 0.5], [1.0, 0.0, 0.25]]])
    p = prob.clone().requires_grad_(True)
    targets = (y.unsqueeze(2) >= torch.arange(1.0, 4.0)).float()
    ref = torch.nn.functional.binary_cross_entropy(p, targets, reduction="sum") / 3.0
    ref.backward()
    val, grad = run(L.ordinal, prob, y, n=3)
    assert val == pytest.approx(ref.item(), rel=1e-6)
    assert np.allclose(grad, p.grad.numpy(), rtol=1e-5)


def test_ordinal_rejects_bad_shapes(L):
    with pytest.raises(ValueError):
        L.ordinal(dev(np.zeros((2, 5), dtype=np.float32)), dev(np.zeros((2, 5), dtype=np.float32)), n=2)
    with pytest.raises(ValueError):
        L.ordinal(dev(np.zeros((2, 5, 3), dtype=np.float32)), dev(np.zeros((2, 5), dtype=np.float32)), n=2)



def test_neural_sort_and_sinkhorn_matrices_match_the_reference(golden):
    """SURVEY.md 8(a) rows a17 / a18 pinned directly: the matrices the fused neuralNDCG kernel works with
    (arb_neural_sort_debug) against loss_utils.deterministic_neural_sort and loss_utils.sinkhorn_scaling of the
    unmodified reference, on the block of real items (the reference fills the padded block with softmax(1) rows and
    zeroes it after the scaling; the kernel never forms it)."""
    from allrank_b200 import losses
    g = golden("neural_sort")
    for key in g["keys"]:
        key = str(key)
        tau, iters, tol = [float(v) for v in g[key + "_args"]]
        yp, yt = torch.tensor(g[key + "_pred"]).cuda(), torch.tensor(g[key + "_true"]).cuda()
        p0, p = losses.neural_sort_matrices(yp, yt, temperature=tau, max_iter=int(iters), tol=tol)
        real = (yt != -1)
        block = (real[:, :, None] & real[:, None, :]).cpu().numpy()
        # rank rows beyond the number of real items belong to the padded block as well
        n_real = real.sum(1).cpu().numpy()
        alive = (yt > 0).any(1).cpu().numpy()       # the loss kernel skips slates whose ideal DCG is zero
        for b in range(block.shape[0]):
            block[b, n_real[b]:, :] = False
            if not alive[b]:
                block[b] = False
        r0, r1 = g[key + "_p0"], g[key + "_p"]
        # the reference's row j of the real block is the j-th RANK; its columns are the items
        # fp32 logits are O(n * |s|) / tau: at tau = 0.1 their ulp (2.4e-4 at 3000) bounds what exp() can reproduce
        tol0 = 1e-5 if tau >= 1.0 else 1e-4
        assert np.abs(p0.cpu().numpy() - r0)[block].max() <= tol0, key
        assert np.abs(p.cpu().numpy() - r1)[block].max() <= 2 * tol0, key
        assert (p.cpu().numpy()[~block] == 0).all()
