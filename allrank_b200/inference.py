"""Device-side replacement for allrank/inference/inference_utils.py:12-60 (`rank_slates` / `__rank_slates`):
score every slate, rank its items by descending score (padded items last) and return X and y in that order.

The reference does this with `scores.sort` + two `torch.gather`s per batch and a `.cpu()` per batch; here the ranking is
the metrics kernel's `out_order` (the same 64-bit-key sort every metric uses, so the ranked labels are exactly the
sequence dcg/ndcg/mrr see) and one gather kernel (`arb_gather_slates`, csrc/slates.cu) moves the rows.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from . import metrics as _metrics

PADDED_Y_VALUE = -1

c_p, c_i = ctypes.c_void_p, ctypes.c_int32
_lib.register("arb_gather_slates", c_i, [c_p, c_p, c_p, c_i, c_i, c_i, c_p, c_p, c_p])


def reorder_slates(X, y_true, order):
    """X [B,S,F], y_true [B,S] re-ordered along the slate axis by `order` [B,S] (int32 positions)."""
    _lib.require_cuda(X, y_true, order)
    if X.dim() != 3 or y_true.shape != X.shape[:2] or order.shape != y_true.shape:
        raise ValueError("X must be [batch, slate, features], y_true and order [batch, slate]")
    x = X.detach().float().contiguous()
    y = y_true.detach().float().contiguous()
    order = order.to(torch.int32).contiguous()
    B, S, F = x.shape
    x_out, y_out = torch.empty_like(x), torch.empty_like(y)
    if B == 0:
        return x_out, y_out
    with torch.cuda.device(x.device):
        rc = _lib.lib().arb_gather_slates(_lib.ptr(x), _lib.ptr(y), _lib.ptr(order), B, S, F, _lib.ptr(x_out),
                                          _lib.ptr(y_out), _lib.stream_ptr(x.device))
    _lib.check(rc, "arb_gather_slates")
    return x_out, y_out


def rank_batch(model, X, y_true):
    """One batch of inference_utils.__rank_slates (:44-57): returns (X, y_true) in descending score order, on device.
    The reference passes all-ones `indices` to the model (:49) -- so does this."""
    mask = y_true == PADDED_Y_VALUE
    indices = torch.ones_like(y_true).long()
    with torch.no_grad():
        scores = model.score(X, mask, indices)
    order = _metrics.ranking(scores, y_true)        # padded items rank last, like scores[mask] = -inf + sort (:51-52)
    return reorder_slates(X, y_true, order)


def rank_dataloader(dataloader, model):
    """inference_utils.__rank_slates: all batches of a loader, concatenated on the host (:37-60)."""
    model.eval()
    dev = next(model.parameters()).device
    ranked_x, ranked_y = [], []
    for xb, yb, _ in dataloader:
        x, y = rank_batch(model, xb.float().to(dev), yb.to(dev))
        ranked_x.append(x.cpu())
        ranked_y.append(y.cpu().to(yb.dtype))
    return torch.cat(ranked_x), torch.cat(ranked_y)


def _as_loader(ds, config):
    """What inference_utils.__create_data_loader (:33-34) does for the reference's LibSVMDataset -- any map-style
    torch Dataset of (x[S,F], y[S], indices[S]) samples is batched with config.data.batch_size, unshuffled; a
    SlateStore becomes a device loader; anything already yielding batches (a DataLoader, a DeviceSlateLoader, a list
    of batches) is used as it is."""
    from torch.utils.data import DataLoader, Dataset
    from .data import DeviceSlateLoader, SlateStore
    if isinstance(ds, SlateStore):
        return DeviceSlateLoader(ds, config.data.batch_size, shuffle=False)
    if isinstance(ds, Dataset):
        return DataLoader(ds, batch_size=config.data.batch_size, num_workers=getattr(config.data, "num_workers", 0),
                          shuffle=False)
    return ds


def rank_slates(datasets, model, config):
    """inference_utils.rank_slates (:12-30): role -> (X, y) ranked by the model.  `datasets` maps a role to the
    reference's LibSVMDataset (or any map-style Dataset), a SlateStore (allrank_b200.data) or a ready loader yielding
    (xb, yb, indices); batch size from config.data."""
    return {role: rank_dataloader(_as_loader(ds, config), model) for role, ds in datasets.items()}


def metrics_on_clicked_slates(clicked_slates, chunk=8192):
    """inference_utils.metrics_on_clicked_slates (:63-82): per clicked slate {"slate_length", "no_of_clicks", "dcg",
    "ndcg"}, the metrics of the clicks (-1 = padding) under the order the slate is in (scores S..1).  One
    arb_rank_metrics launch per chunk of equal-length slates computes dcg and ndcg (bit-identical to the reference's
    ndcg / dcg); no_of_clicks is sum(y > 0) of the caller's row, numpy's integer for an array."""
    Xs, ys = clicked_slates
    ys = list(ys)
    lengths = np.array([len(y) for y in ys], dtype=np.int64)
    dcgs, ndcgs = [0.0] * len(ys), [0.0] * len(ys)
    dev = torch.device("cuda", torch.cuda.current_device())
    for S in np.unique(lengths):
        idx = np.flatnonzero(lengths == S)
        y_pred = torch.arange(int(S), 0, -1, dtype=torch.float32, device=dev)
        for c0 in range(0, len(idx), chunk):
            part = idx[c0:c0 + chunk]
            labels = torch.as_tensor(np.stack([np.asarray(ys[k], dtype=np.float32) for k in part])).to(dev)
            out = _metrics._launch(y_pred.expand(len(part), int(S)).contiguous(), labels, [int(S)], [int(S)],
                                   _metrics.GAIN_POW2, PADDED_Y_VALUE, 1.0, ("dcg", "ndcg"))
            for k, d, n in zip(part, out["dcg"][:, 0].tolist(), out["ndcg"][:, 0].tolist()):
                dcgs[k], ndcgs[k] = d, n
    for y, d, n in zip(ys, dcgs, ndcgs):
        clicked = y > 0
        yield {"slate_length": len(y), "no_of_clicks": clicked.sum(), "dcg": d, "ndcg": n}


__all__ = ["rank_slates", "rank_dataloader", "rank_batch", "reorder_slates", "metrics_on_clicked_slates"]
