"""allRank's click models (allrank/click_models/*) on the device.

The ten reference classes keep their names and constructor arguments; `compile_click_model` flattens a model tree
(made of these classes or of the reference's own instances) into the node array of `arb_click_slates`
(csrc/clicks.cu), which evaluates it for a whole batch of slates, one CTA per slate:

    clicks = click(model, X, y)                       # [B,S] on the device, y's dtype; -1 at padding
    Xs, clicks = click_on_slates((X, y), model, include_empty=False)    # click_utils.click_on_slates

Deterministic models reproduce the reference bit for bit (distances in fp64 summed like scipy's cdist, numpy's
linear quantile).  Random draws come from a counter hash of (seed, node, slate, position) instead of numpy's stream;
the seed is drawn from numpy's global generator unless given, so `np.random.seed` makes runs repeatable.  A model the
kernel does not know raises NotImplementedError: there is no CPU fallback.
"""
import ctypes
import math
from typing import Callable, List

import numpy as np
import torch

from . import _lib

PADDED_Y_VALUE = -1
WORKSPACE_BUDGET = 1 << 30          # fp64 distance triangles held at once; larger batches run in chunks
HOST_CHUNK_BYTES = 256 << 20        # features uploaded at once by click_on_slates

FIXED, RANDOM, RELEVANT, CASCADE, MULTIPLE, CONDITIONED, MAXCLICKS, DUPLICATES, DIVERSE = range(9)
METRICS = {"euclidean": 0, "sqeuclidean": 1, "cityblock": 2, "chebyshev": 3}
MAX_NODES, MAX_SLATE, MAX_LIST = 32, 4096, 1024
STATUS_INDEX_ERROR, STATUS_VALUE_ERROR = 1, 2


class ClickNode(ctypes.Structure):
    """arb_click_node (include/allrank_b200.h)."""
    _fields_ = [("kind", ctypes.c_int32), ("first_child", ctypes.c_int32), ("n_children", ctypes.c_int32),
                ("iparam", ctypes.c_int32), ("list_offset", ctypes.c_int32), ("n_list", ctypes.c_int32),
                ("fparam0", ctypes.c_double), ("fparam1", ctypes.c_double)]


c_p, c_i, c_sz = ctypes.c_void_p, ctypes.c_int32, ctypes.c_size_t
_lib.register("arb_click_workspace_bytes", c_sz, [c_p, c_i, c_i, c_i, c_i])
_lib.register("arb_click_slates", c_i, [c_p, c_i, c_p, c_i, c_p, c_p, c_p, c_i, c_i, c_i, ctypes.c_float,
                                        ctypes.c_int64, ctypes.c_uint64, c_p, c_p, c_p, c_sz, c_p])


# ---------------------------------------------------------------------------------------------------- model classes
class ClickModel:
    """Base class (click_models/base.py:9-26).  `click((X, y))` runs one slate through the device kernel and returns
    its click mask in the reference's dtype (_reference_dtype); every item of the slate counts as real, as in the
    reference."""

    def click(self, documents):
        X, y = documents
        y_t = torch.as_tensor(np.asarray(y, dtype=np.float32))
        x_t = torch.as_tensor(np.asarray(X, dtype=np.float32)) if compile_click_model(self).needs_x else None
        dev = torch.device("cuda", torch.cuda.current_device())
        out = click(self, None if x_t is None else x_t[None].to(dev), y_t[None].to(dev), pad=float("nan"))
        return (out[0].cpu().numpy() > 0).astype(_reference_dtype(self))


def _reference_dtype(m):
    """dtype of the reference's .click() result: a bool mask, int for EverythingButDuplicatesClickModel (`1 * mask`),
    the inner model's for Diverse and MaxClicks, and the children's common type for Multiple (the reference returns
    the chosen child's)."""
    name = type(m).__name__
    if name == "EverythingButDuplicatesClickModel":
        return np.dtype(np.int_)
    if name in ("DiverseClicksModel", "MaxClicksModel"):
        return _reference_dtype(m.inner_click_model)
    if name == "MultipleClickModel":
        return np.result_type(*[_reference_dtype(k) for k in m.inner_click_models])
    return np.dtype(bool)


class RandomClickModel(ClickModel):
    """Clicks `n_clicks` distinct items uniformly at random (base.py:29-46)."""

    def __init__(self, n_clicks: int):
        self.n_clicks = n_clicks


class FixedClickModel(ClickModel):
    """Clicks the items at `click_positions` (numpy indexing: negative positions count from the end; base.py:49-65)."""

    def __init__(self, click_positions: List[int]):
        self.click_positions = click_positions


class MultipleClickModel(ClickModel):
    """Runs one of the inner models per slate, chosen with the given probabilities (base.py:68-87)."""

    def __init__(self, inner_click_models: List[ClickModel], probabilities: List[float]):
        self.inner_click_models = inner_click_models
        total = float(np.sum(probabilities))
        if not math.isclose(total, 1.0, abs_tol=1e-5):      # the reference asserts this (AssertionError)
            raise AssertionError(f"MultipleClickModel: probabilities {list(probabilities)} add up to {total}, not 1")
        self.probabilities = np.cumsum(np.asarray(probabilities, dtype=np.float64))


class ConditionedClickModel(ClickModel):
    """Combines the inner models' clicks with np.all or np.any (base.py:90-106)."""

    def __init__(self, inner_click_models: List[ClickModel], combiner: Callable):
        self.inner_click_models = inner_click_models
        self.combiner = combiner


class MaxClicksModel(ClickModel):
    """Keeps the first `max_clicks` clicks of the inner model; None keeps all (base.py:109-129)."""

    def __init__(self, inner_click_model: ClickModel, max_clicks: int):
        self.inner_click_model = inner_click_model
        self.max_clicks = max_clicks


class OnlyRelevantClickModel(ClickModel):
    """Clicks iff relevance >= `relevancy_threshold` (base.py:132-146)."""

    def __init__(self, relevancy_threshold: float):
        self.relevancy_threshold = relevancy_threshold


class BaseCascadeModel(ClickModel):
    """Observes position p (1-based) with probability min(1, p^-eta); clicks an observed item whose relevance is
    >= `threshold` (cascade_models.py:12-32; with threshold <= 0 unobserved items click too, like the reference)."""

    def __init__(self, eta: float, threshold: float):
        self.eta = eta
        self.threshold = threshold


class DiverseClicksModel(ClickModel):
    """Keeps an inner click iff its euclidean distance to every kept item exceeds the `q_percentile` quantile of the
    slate's pairwise distances (cascade_models.py:35-90)."""

    def __init__(self, inner_click_model, q_percentile=0.5):
        self.inner_click_model = inner_click_model
        self.q_percentile = q_percentile


class EverythingButDuplicatesClickModel(ClickModel):
    """Clicks item j iff its distance to every earlier item exceeds `duplicate_margin` (duplicate_aware.py:10-34)."""

    def __init__(self, duplicate_margin: float = 0, metric: str = "euclidean"):
        self.duplicate_margin = duplicate_margin
        self.metric = metric


class MaskedRemainMasked(ClickModel):
    """Runs the inner model on the real items (y != -1) and marks padded items -1 (click_utils.py:30-53)."""

    def __init__(self, inner_click_model: ClickModel):
        self.inner_click_model = inner_click_model

    def click(self, documents):
        X, y = documents
        y_np = np.asarray(y)
        x_t = torch.as_tensor(np.asarray(X, dtype=np.float32)) if compile_click_model(self).needs_x else None
        dev = torch.device("cuda", torch.cuda.current_device())
        out = click(self, None if x_t is None else x_t[None].to(dev),
                    torch.as_tensor(y_np.astype(np.float32))[None].to(dev))
        return out[0].cpu().numpy().astype(np.zeros_like(y).dtype)


# ---------------------------------------------------------------------------------------------------- compilation
class CompiledClickModel:
    """A click-model tree flattened for arb_click_slates: children of a node are contiguous later nodes."""

    def __init__(self, nodes, values, etas, model):
        self.n_nodes = len(nodes)
        self.nodes = (ClickNode * self.n_nodes)(*nodes)
        self.values = (ctypes.c_double * max(1, len(values)))(*values)
        self.n_values = len(values)
        self.etas = etas
        kinds = {n.kind for n in nodes}
        self.needs_x = bool(kinds & {DUPLICATES, DIVERSE})
        self.random = bool(kinds & {RANDOM, CASCADE, MULTIPLE})
        self.model = model

    def tables(self, S, device):
        """The CASCADE nodes' observation tables [n_cascade, S] fp64 on `device` (None without CASCADE nodes)."""
        return observe_tables(self.etas, S, device) if self.etas else None


_TABLES = {}


def observe_tables(etas, S, device):
    """1 / np.arange(1, S+1) ** eta for each eta, evaluated by numpy exactly as cascade_models.py:31, cached per
    (etas, S, device).  The first upload of a key goes from pinned memory without blocking, so `click(check=False)`
    never synchronises, not even on a model it has not seen."""
    key = (tuple((type(e).__name__, e) for e in etas), int(S), str(device))
    if key not in _TABLES:
        host = np.stack([np.asarray(1 / np.arange(1, S + 1) ** eta, dtype=np.float64) for eta in etas])
        _TABLES[key] = torch.from_numpy(host).pin_memory().to(device, non_blocking=True)
    return _TABLES[key]


def _is_combiner(fn, ref):
    return fn is ref or (getattr(fn, "__name__", None) == ref.__name__ and getattr(fn, "__module__", "").startswith("numpy"))


def _children(m):
    """(kind, params, children) of one model, recognised by class name and attributes (ours or the reference's)."""
    name = type(m).__name__
    if name == "FixedClickModel":
        pos = np.atleast_1d(np.asarray(m.click_positions))
        if pos.size and not np.issubdtype(pos.dtype, np.integer):
            raise IndexError("arrays used as indices must be of integer (or boolean) type")
        return FIXED, {"list": [float(p) for p in pos.ravel()]}, []
    if name == "RandomClickModel":
        if int(m.n_clicks) < 0:
            raise ValueError("negative dimensions are not allowed")
        return RANDOM, {"iparam": int(m.n_clicks)}, []
    if name == "OnlyRelevantClickModel":
        return RELEVANT, {"fparam0": float(m.relevancy_threshold)}, []
    if name == "BaseCascadeModel":
        return CASCADE, {"eta": m.eta, "fparam1": float(m.threshold)}, []
    if name == "MultipleClickModel":
        cum = np.asarray(m.probabilities, dtype=np.float64).ravel()
        if len(cum) != len(m.inner_click_models):
            raise ValueError("MultipleClickModel needs one probability per inner model")
        return MULTIPLE, {"list": [float(c) for c in cum]}, list(m.inner_click_models)
    if name == "ConditionedClickModel":
        if _is_combiner(m.combiner, np.all):
            mode = 0
        elif _is_combiner(m.combiner, np.any):
            mode = 1
        else:
            raise NotImplementedError("ConditionedClickModel runs on the device with np.all or np.any as combiner")
        return CONDITIONED, {"iparam": mode}, list(m.inner_click_models)
    if name == "MaxClicksModel":
        limit = math.inf if m.max_clicks is None else float(m.max_clicks)
        return MAXCLICKS, {"fparam0": limit}, [m.inner_click_model]
    if name == "EverythingButDuplicatesClickModel":
        if m.metric not in METRICS:
            raise NotImplementedError(f"metric {m.metric!r}: the device supports {sorted(METRICS)}")
        return DUPLICATES, {"iparam": METRICS[m.metric], "fparam0": float(m.duplicate_margin)}, []
    if name == "DiverseClicksModel":
        q = float(m.q_percentile)
        if not 0.0 <= q <= 1.0:
            raise ValueError("Quantiles must be in the range [0, 1]")
        return DIVERSE, {"fparam0": q}, [m.inner_click_model]
    raise NotImplementedError(f"{type(m).__module__}.{name} has no device implementation (no CPU fallback)")


def _unmask(m):
    """MaskedRemainMasked is implied: every model of the kernel sees only the real items."""
    while type(m).__name__ == "MaskedRemainMasked":
        m = m.inner_click_model
    return m


def compile_click_model(m):
    """Flatten a click-model tree breadth first (node 0 = root, each node's children contiguous)."""
    if isinstance(m, CompiledClickModel):
        return m
    m = _unmask(m)
    models, specs = [m], []
    i = 0
    while i < len(models):
        kind, params, kids = _children(models[i])
        kids = [_unmask(k) for k in kids]
        specs.append((kind, params, len(models), len(kids)))
        models.extend(kids)
        if len(models) > MAX_NODES:
            raise NotImplementedError(f"click-model trees of more than {MAX_NODES} models are not supported")
        i += 1
    nodes, values, etas = [], [], []
    for kind, params, first, count in specs:
        lst = params.get("list", [])
        iparam = params.get("iparam", 0)
        if kind == CASCADE:
            iparam = len(etas)
            etas.append(params["eta"])
        nodes.append(ClickNode(kind, first if count else 0, count, iparam, len(values), len(lst),
                               params.get("fparam0", 0.0), params.get("fparam1", 0.0)))
        values.extend(lst)
    if len(values) > MAX_LIST:
        raise NotImplementedError(f"at most {MAX_LIST} click positions and probabilities per tree")
    return CompiledClickModel(nodes, values, etas, m)


def draw_seed():
    """A 64-bit seed from numpy's global generator (np.random.seed makes click streams repeatable)."""
    return int(np.random.randint(0, 2 ** 64, dtype=np.uint64))


# ---------------------------------------------------------------------------------------------------- device entry
def _raise_status(status, slate_offset=0):
    bad = np.flatnonzero(status)
    if len(bad) == 0:
        return
    b = int(bad[0])
    if status[b] == STATUS_INDEX_ERROR:
        raise IndexError(f"slate {slate_offset + b}: a click position is out of bounds for the slate's real items")
    raise ValueError(f"slate {slate_offset + b}: Cannot take a larger sample than population when 'replace=False' "
                     "or compute distances over an empty slate")


def click(click_model, X, y, seed=None, check=True, pad=PADDED_Y_VALUE, slate_offset=0, workspace_bytes=None,
          return_status=False):
    """Clicks of `click_model` on a batch of slates, on y's device: y [B,S] (pad marks padding), X [B,S,F] (read only
    when the model measures distances; may be None otherwise).  Returns clicks [B,S] in y's dtype: 0/1 on real items,
    `pad` on padded ones.

    seed: 64-bit seed of the counter-based random draws (default: drawn from numpy's global generator).
    check: read the per-slate status once and raise the reference's exception (IndexError for FixedClickModel
    positions, ValueError for RandomClickModel with more clicks than items or duplicates over an empty slate).  With
    check=False nothing synchronises; return_status=True then also returns the int32 status [B] (0 = ok).
    slate_offset: global index of the first slate (the hash counter), so chunked calls agree with one call.
    workspace_bytes: cap on the distance workspace (default 1 GiB); the batch is processed in chunks that fit."""
    cm = compile_click_model(click_model)
    _lib.require_cuda(y)
    if y.dim() != 2:
        raise ValueError("y must be [batch, slate]")
    B, S = y.shape
    if S > MAX_SLATE:
        raise _lib.ArbError(f"slates above {MAX_SLATE} items are not supported")
    dev = y.device
    yf = y.detach().to(torch.float32).contiguous()
    F = 1
    xf = None
    if cm.needs_x:
        if X is None:
            raise ValueError("this click model measures distances between items and needs X [batch, slate, features]")
        _lib.require_cuda(X)
        if X.dim() != 3 or X.shape[:2] != y.shape:
            raise ValueError("X must be [batch, slate, features] matching y")
        xf = X.detach().to(torch.float32).contiguous()
        F = xf.shape[2]
    if seed is None:
        seed = draw_seed() if cm.random else 0
    clicks = torch.empty((B, S), dtype=torch.float32, device=dev)
    status = torch.empty((B,), dtype=torch.int32, device=dev)
    ws = None
    need = int(_lib.lib().arb_click_workspace_bytes(cm.nodes, cm.n_nodes, max(B, 1), S, F)) if B else 0
    if need:
        per = need // B
        cap = WORKSPACE_BUDGET if workspace_bytes is None else int(workspace_bytes)
        ws = torch.empty(max(per, min(need, cap // per * per)), dtype=torch.uint8, device=dev)
    tables = cm.tables(S, dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().arb_click_slates(
            cm.nodes, cm.n_nodes, cm.values, cm.n_values, _lib.ptr(tables), _lib.ptr(xf), _lib.ptr(yf), B, S, F,
            float(pad), int(slate_offset), int(seed) & (2 ** 64 - 1), _lib.ptr(clicks), _lib.ptr(status), _lib.ptr(ws),
            0 if ws is None else ws.numel(), _lib.stream_ptr(dev))
    _lib.check(rc, "arb_click_slates")
    out = clicks if y.dtype == torch.float32 else clicks.to(y.dtype)
    if check:
        _raise_status(status.cpu().numpy(), slate_offset)
    return (out, status) if return_status else out


def _host(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _rows(a, c0, c1):
    """Rows c0..c1 of a batch (tensor, array or list of rows) as one host array."""
    if hasattr(a, "shape"):
        return _host(a[c0:c1])
    return np.stack([_host(a[k]) for k in range(c0, c1)])


def click_on_slates(slates, click_model, include_empty):
    """click_utils.click_on_slates (:10-27) on the device: returns (list of the slates' X, list of click arrays in y's
    dtype with -1 at padding), dropping slates without a click unless include_empty (ValueError when none is left,
    as in the reference).  X and y are tensors / arrays [N,S,F] and [N,S], or lists of per-slate rows of any lengths
    (padded with -1 to the longest for the kernel, which changes no click).  Only y is uploaded unless the model
    measures distances; slates go up in chunks of at most HOST_CHUNK_BYTES, one launch and one status read each, and
    slate k always draws with hash counter k."""
    X, y = slates
    cm = compile_click_model(click_model)
    seed = draw_seed() if cm.random else 0
    dev = torch.device("cuda", torch.cuda.current_device())
    N = len(y)
    dense = hasattr(y, "shape") and len(y.shape) == 2
    lengths = None if dense else [len(r) for r in y]
    S = int(y.shape[1]) if dense else max(lengths, default=1)
    F = int(_host(X[0]).shape[-1]) if cm.needs_x and N else 1
    step = max(1, HOST_CHUNK_BYTES // (S * F * 4))
    clicks, has_click = [], []
    for c0 in range(0, N, step):
        c1 = min(N, c0 + step)
        if dense:
            yb = _rows(y, c0, c1)
            xb = _rows(X, c0, c1) if cm.needs_x else None
        else:
            yb = np.full((c1 - c0, S), PADDED_Y_VALUE, dtype=np.float32)
            xb = np.zeros((c1 - c0, S, F), dtype=np.float32) if cm.needs_x else None
            for r, k in enumerate(range(c0, c1)):
                yb[r, :lengths[k]] = _host(y[k])
                if xb is not None:
                    xb[r, :lengths[k]] = _host(X[k])
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)   # noqa: E731
        out = click(cm, None if xb is None else up(xb), up(yb), seed=seed, slate_offset=c0).cpu().numpy()
        has_click.append((out > 0).any(axis=1))
        if dense:
            clicks.extend(out.astype(yb.dtype, copy=False))
        else:
            clicks.extend(out[r, :lengths[k]].astype(_host(y[k]).dtype) for r, k in enumerate(range(c0, c1)))
    keep = np.flatnonzero(np.concatenate(has_click)) if has_click and not include_empty else np.arange(N)
    if len(keep) == 0:
        raise ValueError("click_on_slates: no slate is left (include_empty=False drops the slates without a click)")
    return [X[int(k)] for k in keep], [clicks[int(k)] for k in keep]


__all__ = ["ClickModel", "RandomClickModel", "FixedClickModel", "MultipleClickModel", "ConditionedClickModel",
           "MaxClicksModel", "OnlyRelevantClickModel", "BaseCascadeModel", "DiverseClicksModel",
           "EverythingButDuplicatesClickModel", "MaskedRemainMasked", "compile_click_model", "click",
           "click_on_slates", "CompiledClickModel"]
