"""Drop-in replacements for allrank.models.metrics -- same names, arguments and defaults
(/root/reference/allrank/models/metrics.py: ndcg :7-28, dcg :41-77, mrr :80-113), computed by one
sm_90a kernel launch per call (csrc/slate_kernels.cu: metrics_kernel) through the C ABI.

`metric(y_pred, y_true, ats=...) -> [B, len(ats)]` fp32 on the input device, as consumed by
allrank/training/train_utils.py:32-56.
"""
import ctypes

import torch

from . import _lib

PADDED_Y_VALUE = -1

GAIN_POW2, GAIN_IDENTITY = 0, 1


def pow2_gain(x):
    """Default gain 2^x - 1 (metrics.py:7,41)."""
    return torch.pow(2, x) - 1


def identity_gain(x):
    return x


_DISCOUNTS = {}


def discount_table(n, device):
    """1/log2(j+2), evaluated on the HOST in fp32 exactly like metrics.py:64, cached per (n, device)."""
    key = (int(n), str(device))
    if key not in _DISCOUNTS:
        host = torch.tensor(1) / torch.log2(torch.arange(n, dtype=torch.float) + 2.0)
        _DISCOUNTS[key] = host.to(device)
    return _DISCOUNTS[key]


def _gain_mode(fn):
    if fn is pow2_gain:
        return GAIN_POW2
    if fn is identity_gain:
        return GAIN_IDENTITY
    probe = torch.tensor([0.0, 1.0, 2.0, 3.0, 4.0, 0.5, 2.25])
    try:
        out = fn(probe)
    except Exception as exc:  # pragma: no cover
        raise NotImplementedError("gain_function must accept a tensor") from exc
    if torch.equal(out, probe):
        return GAIN_IDENTITY
    if torch.allclose(out, torch.pow(2, probe) - 1, rtol=1e-6, atol=0):
        return GAIN_POW2
    raise NotImplementedError(
        "allrank_b200 metrics support the two gain functions allRank uses (2^x-1 and identity) natively; "
        "there is no CPU fallback for arbitrary callables")


def _prep(y_pred, y_true):
    _lib.require_cuda(y_pred, y_true)
    if y_pred.dim() != 2 or y_pred.shape != y_true.shape:
        raise ValueError("y_pred and y_true must both be [batch_size, slate_length]")
    return y_pred.detach().float().contiguous(), y_true.detach().float().contiguous()


def dcg_cutoffs(ats, S):
    """The cut-offs the reference's dcg evaluates for `ats` on slates of S items (metrics.py:58-75), each in [1, S].

    Every `at` is clipped to S.  The reference then keeps the first max(clipped) cumulative columns (a Python slice, so
    a negative maximum keeps all but that many) and reads column `at - 1` of them, so a cut-off <= 0 counts from the
    end: 0 is the last kept column, -1 the one before.  An index before the first column raises IndexError, and an
    empty list ValueError (the reference's np.max), like the reference.
    """
    clipped = [min(int(a), S) for a in ats]
    if not clipped:
        raise ValueError("ats must name at least one cut-off")
    kept = len(range(S)[:max(clipped)])
    out = []
    for a in clipped:
        at = a if a > 0 else kept + a
        if at < 1:
            raise IndexError(f"cut-off {a} reads before the first of {kept} cumulative DCG columns")
        out.append(at)
    return out


def _ats_array(ats):
    if ats is None:
        return None
    if len(ats) > 32:
        raise ValueError("at most 32 evaluation ranks per call")
    return (ctypes.c_int32 * len(ats))(*[int(a) for a in ats])


def _launch(y_pred, y_true, ats_dcg, ats_mrr, gain_mode, pad, filler, want):
    """ats_dcg: cut-offs in [1, S] (None when no DCG output is wanted); ats_mrr: raw cut-offs (None likewise)."""
    B, S = y_pred.shape
    dev = y_pred.device
    n = len(ats_dcg if ats_dcg is not None else ats_mrr)
    outs = {k: torch.empty((B, n), dtype=torch.float32, device=dev) for k in want if k != "order"}
    if "order" in want:
        outs["order"] = torch.empty((B, S), dtype=torch.int32, device=dev)
    if B == 0:
        return outs
    scratch = torch.empty(2 * B, dtype=torch.float32, device=dev) if "mrr" in want else None
    need_disc = any(k in want for k in ("dcg", "idcg", "ndcg"))
    disc = discount_table(S, dev) if need_disc else None
    with torch.cuda.device(dev):
        rc = _lib.lib().arb_rank_metrics(
            _lib.ptr(y_pred), _lib.ptr(y_true), B, S, _lib.ptr(disc), _ats_array(ats_dcg), _ats_array(ats_mrr), n,
            gain_mode, float(pad), float(filler), _lib.ptr(outs.get("dcg")), _lib.ptr(outs.get("idcg")),
            _lib.ptr(outs.get("ndcg")), _lib.ptr(outs.get("mrr")), _lib.ptr(outs.get("order")), _lib.ptr(scratch),
            _lib.stream_ptr(dev))
    _lib.check(rc, "arb_rank_metrics")
    return outs


def dcg(y_pred, y_true, ats=None, gain_function=pow2_gain, padding_indicator=PADDED_Y_VALUE):
    """Discounted Cumulative Gain at k -- metrics.py:41-77."""
    yp, yt = _prep(y_pred, y_true)
    S = yt.shape[1]
    cut = dcg_cutoffs([S] if ats is None else list(ats), S)
    return _launch(yp, yt, cut, None, _gain_mode(gain_function), padding_indicator, 0.0, ("dcg",))["dcg"]


def ndcg(y_pred, y_true, ats=None, gain_function=pow2_gain, padding_indicator=PADDED_Y_VALUE, filler_value=1.0):
    """Normalized DCG at k; slates whose ideal DCG is 0 get `filler_value` -- metrics.py:7-28."""
    yp, yt = _prep(y_pred, y_true)
    S = yt.shape[1]
    cut = dcg_cutoffs([S] if ats is None else list(ats), S)
    return _launch(yp, yt, cut, None, _gain_mode(gain_function), padding_indicator, filler_value, ("ndcg",))["ndcg"]


def mrr(y_pred, y_true, ats=None, padding_indicator=PADDED_Y_VALUE):
    """Mean Reciprocal Rank at k (rank of the first max-label item; batch-wide zero rule) -- metrics.py:80-113."""
    yp, yt = _prep(y_pred, y_true)
    S = yt.shape[1]
    ats = [S] if ats is None else list(ats)
    return _launch(yp, yt, None, [int(a) for a in ats], GAIN_POW2, padding_indicator, 0.0, ("mrr",))["mrr"]


def ranking(y_pred, y_true, padding_indicator=PADDED_Y_VALUE):
    """The descending argsort the metrics are built on (int32 [B,S]); stable, bit-exact on tie-free scores."""
    yp, yt = _prep(y_pred, y_true)
    S = yt.shape[1]
    return _launch(yp, yt, [S], [S], GAIN_POW2, padding_indicator, 0.0, ("order",))["order"]


def all_metrics(y_pred, y_true, ats, padding_indicator=PADDED_Y_VALUE, filler_value=1.0):
    """One launch for dcg + ndcg + mrr (what a fused eval step wants); returns a dict of [B,len(ats)] tensors."""
    yp, yt = _prep(y_pred, y_true)
    S = yt.shape[1]
    return _launch(yp, yt, dcg_cutoffs(ats, S), [int(a) for a in ats], GAIN_POW2, padding_indicator, filler_value,
                   ("dcg", "idcg", "ndcg", "mrr"))
