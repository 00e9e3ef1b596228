"""CUDA parity of the metrics kernel: bit-exact argsort and values against the reference's golden
vectors (tie-free scores), the reference's known answers, and the CPU oracle at bench sizes."""
import numpy as np
import pytest
import torch

from tests import cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def M():
    from allrank_b200 import metrics
    return metrics


def dev(x):
    return torch.as_tensor(x, dtype=torch.float32).cuda()


def same_valid_prefix(order, ref_order, y_true):
    """Bit-exact argsort on the real items; the relative order of the padded (-inf) tail is a tie the
    reference's unstable sort leaves unspecified and that no metric reads (metrics.py:35)."""
    order, ref_order, y_true = np.asarray(order), np.asarray(ref_order), np.asarray(y_true)
    for b in range(order.shape[0]):
        n = int((y_true[b] != -1).sum())
        if not np.array_equal(order[b, :n], ref_order[b, :n]):
            return False
        if sorted(order[b, n:].tolist()) != sorted(ref_order[b, n:].tolist()):
            return False
    return True


@pytest.mark.parametrize("yp,yt,ats,expected,exact", cases.NDCG_KNOWN)
def test_ndcg_known(M, yp, yt, ats, expected, exact):
    out = M.ndcg(dev([yp]), dev([yt]), ats=ats).cpu().numpy()[0]
    assert out == pytest.approx(expected)
    if exact:
        assert out[0] == np.float32(expected[0])


@pytest.mark.parametrize("yp,yt,ats,expected", cases.MRR_KNOWN)
def test_mrr_known(M, yp, yt, ats, expected):
    out = M.mrr(dev(yp), dev(yt), ats=ats).cpu().numpy()
    assert (out == np.array(expected, dtype=np.float32)).all()


def test_golden_bit_exact(M, golden):
    g = golden("metrics")
    ats = [int(a) for a in g["ats"]]
    for key in g["keys"]:
        key = str(key)
        yp, yt = dev(g[key + "_pred"]), dev(g[key + "_true"])
        assert same_valid_prefix(M.ranking(yp, yt).cpu().numpy(), g[key + "_order"], g[key + "_true"]), key
        assert np.array_equal(M.dcg(yp, yt, ats=ats).cpu().numpy(), g[key + "_dcg"]), key
        assert np.array_equal(M.ndcg(yp, yt, ats=ats).cpu().numpy(), g[key + "_ndcg"]), key
        assert np.array_equal(M.mrr(yp, yt, ats=ats).cpu().numpy(), g[key + "_mrr"]), key
        assert np.array_equal(M.ndcg(yp, yt).cpu().numpy(), g[key + "_ndcg_none"]), key
        assert np.array_equal(M.dcg(yp, yt, ats=[3, 10], gain_function=lambda x: x).cpu().numpy(),
                              g[key + "_dcg_identity"]), key


@pytest.mark.parametrize("B,S", [(64, 240), (256, 120), (4, 1251), (3, 1), (2, 2049), (1, 4096)])
def test_against_oracle_bit_exact(M, B, S):
    from oracle import metrics_ref
    from allrank_b200.synth import make_slates, make_scores
    _, y, _ = make_slates(B, S, n_features=1, seed=21, mean_len=0.5 * S + 1, std_len=0.3 * S)
    yp = make_scores(B, S, seed=22)
    ats = [1, 5, 10, 30, 60, 5000]
    assert same_valid_prefix(M.ranking(yp.cuda(), y.cuda()).cpu().numpy(), metrics_ref.ranking(yp, y).numpy(), y.numpy())
    for name in ("ndcg", "dcg", "mrr"):
        got = getattr(M, name)(yp.cuda(), y.cuda(), ats=ats).cpu().numpy()
        ref = getattr(metrics_ref, name)(yp, y, ats=ats).numpy()
        assert np.array_equal(got, ref), name
    fused = M.all_metrics(yp.cuda(), y.cuda(), ats)
    assert np.array_equal(fused["ndcg"].cpu().numpy(), metrics_ref.ndcg(yp, y, ats=ats).numpy())
    assert np.array_equal(fused["mrr"].cpu().numpy(), metrics_ref.mrr(yp, y, ats=ats).numpy())


def test_sortedness_and_permutation_property(M):
    """Size-independent property at a large batch: the returned order is a permutation of each slate that
    sorts the masked scores descending; ndcg of the ideal ordering is exactly 1."""
    from allrank_b200.synth import make_slates, make_scores
    B, S = 2048, 240
    _, y, _ = make_slates(B, S, n_features=1, seed=31)
    yp = make_scores(B, S, seed=32).cuda()
    y = y.cuda()
    order = M.ranking(yp, y).long()
    assert torch.equal(order.sort(dim=1).values, torch.arange(S, device="cuda").expand(B, S))
    masked = yp.masked_fill(y == -1, float("-inf")).gather(1, order)
    assert (masked[:, 1:] <= masked[:, :-1]).all()
    ideal = M.ndcg(y.masked_fill(y == -1, -5.0), y, ats=[10, S])
    assert torch.equal(ideal, torch.ones_like(ideal))


def test_ties_resolve_by_position_and_inputs_untouched(M):
    yp = dev([[0.5, 0.5, 0.5, 0.1]])
    yt = dev([[0.0, 2.0, 1.0, 3.0]])
    a, b = yp.clone(), yt.clone()
    assert M.ranking(yp, yt).cpu().tolist() == [[0, 1, 2, 3]]
    assert torch.equal(yp, a) and torch.equal(yt, b)


def test_cpu_tensors_raise(M):
    with pytest.raises(Exception):
        M.ndcg(torch.tensor([[0.5, 0.2]]), torch.tensor([[1.0, 0.0]]))
