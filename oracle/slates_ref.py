"""Oracle restatement of the slate movers either side of the scorer (TEST INFRASTRUCTURE, see oracle/__init__.py).

Reference: /root/reference/allrank/data/dataset_loading.py     LibSVMDataset grouping :104-111, FixLength :32-93
           /root/reference/allrank/inference/inference_utils.py __rank_slates :37-60
           /root/reference/allrank/training/train_utils.py      metric_on_epoch / compute_metrics :37-56

`_sample` takes its random draws from a source, as oracle/clicks_ref.py does:
* `NumpySource` (the default) draws from numpy's global stream with the same calls in the same order as the
  reference, so with the same np.random.seed `fix_length` reproduces the reference's slates exactly -- pinned by
  tests/golden/slates.npz (oracle/make_golden.py).
* `HashSource` restates the CUDA kernel's counter hash (csrc/slates.cu, sample_hash): with it, `assemble` is what
  `arb_assemble_slates` writes, bit for bit.  The redraw and append rules are the reference's, in `_sample` only, so
  the kernel is checked against the reference's logic and not against a copy of itself.
The rules themselves are pinned against the unmodified reference driven by scripted draws
(tests/golden/slates_rules.npz, tools/make_golden_slates_rules.py).
"""
import numpy as np
import torch

PAD_Y = -1
PAD_INDEX = -1
MAX_ATTEMPTS = 1024        # csrc/slates.cu ASM_MAX_ATTEMPTS


class NumpySource:
    """np.random.choice, called exactly as dataset_loading.py:70 and :74 call it."""
    max_attempts = None    # the reference recurses until it draws a relevant item (or hits RecursionError)

    def choice_n(self, n, k, attempt):
        return np.random.choice(n, k, replace=False)

    def choice_sub(self, idx, k):
        return np.random.choice(idx, k, replace=False)


_M32 = np.uint64(0xFFFFFFFF)


def _mix32(h):
    # csrc/dropout.cuh mix32, on uint64 arrays holding 32-bit values
    h = h ^ (h >> np.uint64(16))
    h = (h * np.uint64(0x85EBCA6B)) & _M32
    h = h ^ (h >> np.uint64(13))
    h = (h * np.uint64(0xC2B2AE35)) & _M32
    return h ^ (h >> np.uint64(16))


def sample_hash(seed, slate, attempt, items):
    """csrc/slates.cu sample_hash(seed, slate, attempt, item) for an array of items: uint32 values as uint64."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    lo, hi = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    h = _mix32(np.array([lo ^ np.uint64((int(slate) * 0x9E3779B1) & 0xFFFFFFFF)], dtype=np.uint64))
    h = _mix32(h ^ hi ^ np.uint64((int(attempt) * 0x85EBCA6B + 0x7F4A7C15) & 0xFFFFFFFF))
    items = np.asarray(items, dtype=np.uint64)
    return _mix32(h ^ ((items * np.uint64(0xC2B2AE35) + np.uint64(0x165667B1)) & _M32))


class HashSource:
    """The draws of slate `slate` of a batch sampled with `seed` by assemble_slates_kernel.

    choice_n(n, k, attempt): the k smallest keys (hash(seed, slate, attempt, i) << 32) | i, in key order -- a uniform
    sample without replacement in random order, like np.random.choice(n, k, replace=False).  The low half carries
    the index; it never decides the order, since for a fixed (seed, slate, attempt) the hash is a bijection of the
    item (mix32 is invertible) and no two keys of a draw share a high half.
    choice_sub(idx, k): the first k entries, which are already in random order.
    max_attempts: the 1024th draw is kept whatever it holds, where the reference would recurse until RecursionError
    (a query whose labels sum to more than 0, but whose relevant items are too rare to be drawn in 1024 tries)."""
    max_attempts = MAX_ATTEMPTS

    def __init__(self, seed, slate):
        self.seed, self.slate = int(seed) & 0xFFFFFFFFFFFFFFFF, int(slate)

    def keys(self, n, attempt):
        i = np.arange(n, dtype=np.uint64)
        return (sample_hash(self.seed, self.slate, attempt, i) << np.uint64(32)) | i

    def choice_n(self, n, k, attempt):
        return (np.sort(self.keys(n, attempt))[:k] & _M32).astype(np.int64)

    def choice_sub(self, idx, k):
        return np.asarray(idx)[:k]


NUMPY = NumpySource()


def group_offsets(query_ids):
    # dataset_loading.py:106-111: groups in order of first appearance, each `count` consecutive rows
    _, first, counts = np.unique(np.asarray(query_ids), return_index=True, return_counts=True)
    return np.concatenate([[0], np.cumsum(counts[np.argsort(first)])]).astype(np.int64)


def _pad(x, y, n, slate_length):
    # dataset_loading.py:76-93
    fx = np.pad(x, ((0, slate_length - n), (0, 0)), "constant")
    fy = np.pad(y, (0, slate_length - n), "constant", constant_values=PAD_Y)
    idx = np.pad(np.arange(0, n), (0, slate_length - n), "constant", constant_values=PAD_INDEX)
    return fx, fy, idx


def _sample(x, y, n, slate_length, source=NUMPY):
    # dataset_loading.py:55-74.  The reference redraws by recursing; the loop makes the same draws in the same order
    # and stops where the source caps the attempts.
    attempt = 0
    while True:
        idx = source.choice_n(n, slate_length, attempt)
        fy = y[idx]
        if fy.sum() == 0:
            if y.sum() == 1:
                idx = np.concatenate([source.choice_sub(idx, slate_length - 1), [np.argmax(y)]])
                fy = y[idx]
            elif y.sum() > 0 and (source.max_attempts is None or attempt + 1 < source.max_attempts):
                attempt += 1
                continue
        return x[idx], fy, idx


def fix_length(x, y, slate_length, source=NUMPY):
    # dataset_loading.py:41-53: shorter -> pad, otherwise (including equal length) -> sample
    n = len(y)
    return _pad(x, y, n, slate_length) if n < slate_length else _sample(x, y, n, slate_length, source)


def assemble(X, y, offsets, queries, slate_length, seed):
    """What arb_assemble_slates writes for a batch: (x [B,S,F] fp32, y [B,S] fp32, indices [B,S] int64).  Slate b
    is fix_length of query queries[b] with HashSource(seed, b); a query number outside [0, Q) gives a slate of
    padding only.  X, y: the store's fp32 rows; offsets: its CSR offsets [Q+1]."""
    X, y = np.asarray(X, dtype=np.float32), np.asarray(y, dtype=np.float32)
    offsets = np.asarray(offsets, dtype=np.int64)
    queries = np.asarray(queries, dtype=np.int64).reshape(-1)
    B, S, Q = len(queries), int(slate_length), len(offsets) - 1
    xo = np.zeros((B, S, X.shape[1]), dtype=np.float32)
    yo = np.full((B, S), PAD_Y, dtype=np.float32)
    io = np.full((B, S), PAD_INDEX, dtype=np.int64)
    for b, q in enumerate(queries):
        if 0 <= q < Q:
            lo, hi = offsets[q], offsets[q + 1]
            xo[b], yo[b], io[b] = fix_length(X[lo:hi], y[lo:hi], S, HashSource(seed, b))
    return xo, yo, io


def sample_is_admissible(y_query, idx, slate_length):
    """The rules a sampled slate obeys whatever the random stream (dataset_loading.py:55-74)."""
    idx = np.asarray(idx)
    n = len(y_query)
    if len(idx) != slate_length or idx.min() < 0 or idx.max() >= n or len(np.unique(idx)) != slate_length:
        return False
    if y_query.sum() > 0 and y_query[idx].sum() == 0:
        return False                      # a relevant item exists but the sample has none: must have been redrawn
    return True


def rank_batch(scores, X, y_true):
    # inference_utils.py:49-57
    scores = scores.clone()
    scores[y_true == PAD_Y] = float("-inf")
    _, order = scores.sort(descending=True, dim=-1)
    order_x = torch.unsqueeze(order, -1).repeat_interleave(X.shape[-1], -1)
    return torch.gather(X, dim=1, index=order_x), torch.gather(y_true, dim=1, index=order), order


def metric_on_epoch(metric, score_fn, batches):
    # train_utils.py:37-46: mean over all slates of the per-slate metric rows
    rows = [metric(score_fn(xb, yb == PAD_Y, idx), yb) for xb, yb, idx in batches]
    return torch.mean(torch.cat(rows), dim=0).numpy()
