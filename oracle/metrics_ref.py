"""Oracle restatement of allRank's ranking metrics (TEST INFRASTRUCTURE, see oracle/__init__.py).

Reference: /root/reference/allrank/models/metrics.py
  ndcg  :7-28     dcg :41-77 (+ helper :31-38)     mrr :80-113

Semantics that matter for parity (SURVEY.md section 7, quirks Q5/Q7):
  * padded items (label == padding_indicator) get score -inf and label 0, then the
    slate is sorted by score, descending, with torch's default (unstable) sort -- or, with
    `stable=True`, with the stable sort whose order (ties by position) the CUDA kernel documents;
  * discount_j = 1 / log2(j + 2), evaluated in fp32 *on the host*;
  * `ats` larger than the slate are clipped to the slate length;
  * ndcg: slates with ideal DCG == 0 get `filler_value` (1.0 by default);
  * mrr: rank of the first item carrying the slate's MAX label; the
    "no relevant item" rule is a batch-wide scalar (sum of all per-slate maxima == 0).
"""
import torch

PAD = -1  # allrank/data/dataset_loading.py:15  PADDED_Y_VALUE


def pow2_gain(labels):
    return torch.pow(2, labels) - 1


def _labels_in_score_order(scores, labels, pad, stable=False):
    # metrics.py:31-38
    scores = scores.clone()
    labels = labels.clone()
    is_pad = labels == pad
    scores[is_pad] = float("-inf")
    labels[is_pad] = 0.0
    order = scores.sort(descending=True, stable=stable, dim=-1).indices
    return labels.gather(1, order), order


def discount_table(n, device="cpu"):
    # metrics.py:64  (computed on the host in fp32, then moved)
    return (torch.tensor(1) / torch.log2(torch.arange(n, dtype=torch.float) + 2.0)).to(device)


def dcg(y_pred, y_true, ats=None, gain_function=pow2_gain, padding_indicator=PAD, stable=False):
    # metrics.py:41-77
    n = y_true.shape[1]
    ats = [n] if ats is None else list(ats)
    ats = [min(a, n) for a in ats]
    ranked, _ = _labels_in_score_order(y_pred, y_true, padding_indicator, stable)
    weighted = (gain_function(ranked) * discount_table(n, ranked.device))[:, :max(ats)]
    running = torch.cumsum(weighted, dim=1)
    return running[:, torch.tensor(ats, dtype=torch.long) - 1]


def ndcg(y_pred, y_true, ats=None, gain_function=pow2_gain, padding_indicator=PAD, filler_value=1.0, stable=False):
    # metrics.py:7-28
    ideal = dcg(y_true, y_true, ats, gain_function, padding_indicator, stable)
    out = dcg(y_pred, y_true, ats, gain_function, padding_indicator, stable) / ideal
    out[ideal == 0] = filler_value
    return out


def mrr(y_pred, y_true, ats=None, padding_indicator=PAD, stable=False):
    # metrics.py:80-113
    n_slates = y_true.shape[0]
    ats = [y_true.shape[1]] if ats is None else list(ats)
    ranked, _ = _labels_in_score_order(y_pred, y_true, padding_indicator, stable)
    best, first_pos = ranked.max(dim=1)
    pos = first_pos.type_as(best).view(-1, 1).expand(n_slates, len(ats))
    cutoffs = torch.tensor(ats, dtype=torch.float32, device=pos.device).expand(n_slates, len(ats))
    out = torch.tensor(1.0) / (pos + torch.tensor(1.0))
    if bool(best.sum() == 0.0):  # batch-wide rule, metrics.py:108-109
        out = torch.zeros_like(out)
    return out * (pos < cutoffs).float()


def ranking(y_pred, y_true, padding_indicator=PAD, stable=False):
    """The argsort the metrics are built on (for bit-exact order checks)."""
    return _labels_in_score_order(y_pred, y_true, padding_indicator, stable)[1]
