"""CPU restatement of allRank's click models (allrank/click_models/*) that takes its random draws from an explicit
source -- TEST INFRASTRUCTURE for allrank_b200.click_models.

    clicks = click_slates(model, X, y, source)       # [B,S] float32, -1 at padding (MaskedRemainMasked)

`model` is a tree of the reference's classes or of allrank_b200.click_models' (recognised by class name).  Nodes are
numbered breadth first with each node's children contiguous, the numbering arb_click_slates uses.  The source
supplies the draws, in the reference's order (depth first, children in order):
    NumpySource()        np.random.rand / np.random.choice exactly where the reference calls them (golden data)
    TableSource(fn)      fn(node, slate, position) -> uniform in [0, 1); RANDOM takes the n_clicks smallest
                         uniforms, ties to the lower position (the device's counter hash, restated by the tests)
Distances are float64 sums over the features in order of (a_k - b_k)^2 / |a_k - b_k| (scipy's cdist loop); the
DIVERSE margin is np.quantile.  Errors are the reference's exception types.
"""
import numpy as np

PADDED_Y_VALUE = -1


class NumpySource:
    def rand(self, node, slate, n):
        return np.random.rand(n)

    def rand1(self, node, slate):
        return np.random.rand()

    def choice(self, node, slate, n, k):
        return np.random.choice(range(n), size=k, replace=False)


class TableSource:
    def __init__(self, fn):
        self.fn = fn

    def rand(self, node, slate, n):
        return np.array([self.fn(node, slate, j) for j in range(n)], dtype=np.float64)

    def rand1(self, node, slate):
        return self.fn(node, slate, 0)

    def choice(self, node, slate, n, k):
        if k > n:
            raise ValueError("Cannot take a larger sample than population when 'replace=False'")
        u = self.rand(node, slate, n)
        return np.argsort(u, kind="stable")[:k]


def _unmask(m):
    while type(m).__name__ == "MaskedRemainMasked":
        m = m.inner_click_model
    return m


def _kids(m):
    name = type(m).__name__
    if name in ("MultipleClickModel", "ConditionedClickModel"):
        return [_unmask(k) for k in m.inner_click_models]
    if name in ("MaxClicksModel", "DiverseClicksModel"):
        return [_unmask(m.inner_click_model)]
    return []


def number_nodes(model):
    """{id(model object): node index} in breadth-first order (children contiguous)."""
    order, i = [_unmask(model)], 0
    while i < len(order):
        order.extend(_kids(order[i]))
        i += 1
    return {id(m): k for k, m in enumerate(order)}


def pair_distances(X, metric="euclidean"):
    """d[i, j] for all i, j: float64 of float32 features, summed over the features in order."""
    X = np.asarray(X, dtype=np.float32).astype(np.float64)
    n = X.shape[0]
    acc = np.zeros((n, n), dtype=np.float64)
    for k in range(X.shape[1]):
        d = X[:, None, k] - X[None, :, k]
        if metric in ("euclidean", "sqeuclidean"):
            acc = acc + d * d
        elif metric == "cityblock":
            acc = acc + np.abs(d)
        elif metric == "chebyshev":
            acc = np.maximum(acc, np.abs(d))
        else:
            raise NotImplementedError(metric)
    return np.sqrt(acc) if metric == "euclidean" else acc


def _eval(m, X, y, ids, source, slate):
    """Clicks (bool [n]) of model m on the real items X [n,F], y [n]."""
    name, node, n = type(m).__name__, ids[id(m)], len(y)
    if name == "FixedClickModel":
        c = np.zeros(n, dtype=bool)
        c[m.click_positions] = 1
        return c
    if name == "RandomClickModel":
        c = np.zeros(n, dtype=bool)
        c[source.choice(node, slate, n, m.n_clicks)] = 1
        return c
    if name == "OnlyRelevantClickModel":
        return y >= np.float32(m.relevancy_threshold)
    if name == "BaseCascadeModel":
        observed = (1 / np.arange(1, n + 1) ** m.eta) >= source.rand(node, slate, n)
        return y * observed.astype(np.float32) >= np.float32(m.threshold)
    if name == "MultipleClickModel":
        u = source.rand1(node, slate)
        k = int(np.argmax(u < np.asarray(m.probabilities)))
        return _eval(_unmask(m.inner_click_models[k]), X, y, ids, source, slate)
    if name == "ConditionedClickModel":
        parts = [_eval(_unmask(k), X, y, ids, source, slate) for k in m.inner_click_models]
        if m.combiner is np.all:
            return np.all(parts, 0)
        if m.combiner is np.any:
            return np.any(parts, 0)
        raise NotImplementedError("combiner")
    if name == "MaxClicksModel":
        c = _eval(_unmask(m.inner_click_model), X, y, ids, source, slate)
        if m.max_clicks is None:
            return c
        return (c * (c.cumsum() <= m.max_clicks)).astype(bool)
    if name == "EverythingButDuplicatesClickModel":
        if n == 0:
            raise ValueError("zero-size array to reduction operation minimum which has no identity")
        d = pair_distances(X, m.metric)
        d[np.tril_indices(n)] = np.inf
        return (d > m.duplicate_margin).min(0).astype(bool)
    if name == "DiverseClicksModel":
        d = pair_distances(X)
        tri = d[np.triu_indices(n, 1)]
        margin = 0 if len(tri) == 0 else np.quantile(tri, q=m.q_percentile)
        c = _eval(_unmask(m.inner_click_model), X, y, ids, source, slate).astype(bool).copy()
        kept = []
        for j in np.flatnonzero(c):
            if all(d[k, j] > margin for k in kept) and np.inf > margin:
                kept.append(j)
            else:
                c[j] = False
        return c
    raise NotImplementedError(name)


def click_slates(model, X, y, source=None):
    """MaskedRemainMasked(model) on every slate: clicks [B,S] float32 (0/1, -1 at y == -1)."""
    source = NumpySource() if source is None else source
    m = _unmask(model)
    ids = number_nodes(m)
    X = np.asarray(X, dtype=np.float32)
    y = np.asarray(y, dtype=np.float32)
    out = np.zeros(y.shape, dtype=np.float32)
    for b in range(y.shape[0]):
        real = y[b] != PADDED_Y_VALUE
        out[b, ~real] = PADDED_Y_VALUE
        out[b, real] = _eval(m, X[b][real], y[b][real], ids, source, b)
    return out


def build_model(spec, classes):
    """A model tree from a {"name": class name, "args": {...}} spec (nested like allRank's click_model config), with
    the classes of `classes` (the reference's modules merged into a dict, or allrank_b200.click_models)."""
    get = classes.get if isinstance(classes, dict) else (lambda n: getattr(classes, n))
    args = {}
    for k, v in spec.get("args", {}).items():
        if isinstance(v, dict) and "name" in v:
            v = build_model(v, classes)
        elif isinstance(v, list) and v and isinstance(v[0], dict):
            v = [build_model(s, classes) for s in v]
        elif v in ("np.all", "np.any"):
            v = np.all if v == "np.all" else np.any
        args[k] = v
    return get(spec["name"])(**args)
