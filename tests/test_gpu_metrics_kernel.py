"""The ranking-metrics kernel (metrics_kernel + mrr_finalize_kernel, csrc/slate_kernels.cu) against a restatement of
the reference's metrics (allrank/models/metrics.py:7-113) with a STABLE sort, at every slate length it accepts.

`launch` drives arb_rank_metrics directly and asks for all five outputs at once: dcg, idcg, ndcg, mrr and the order.
Every float output is filled with NaN and the order with -7 first, so an element the kernel does not write cannot
pass.  Every case runs twice: the two runs must give the same bits, and the inputs must be untouched.

Contracts (DESIGN section 5, metrics row):
  * order: the stable descending sort of the masked scores (padded items -inf), bit for bit at every position, the
    padded tail included -- NaN first, +0 and -0 equal, a real -inf item tied with the padded ones by position;
  * integer labels from -149 to 128, both gains: dcg, idcg, ndcg and mrr bit for bit (NaN where the reference gives
    NaN, e.g. ndcg = inf / inf when a label of 128 makes 2^128 - 1 overflow);
  * fractional labels: mrr and the order bit for bit; dcg, idcg and ndcg within `fractional_bound`, which follows the
    kernel's own operations (exp2f at 2 ulp, the subtraction and the product with the fp32 discount at half an ulp
    each, the double running sum, the final fp32 rounding).  torch's own fp32 evaluation must lie inside the bound
    too, so the bound is attainable, and the worst observed ratio of error to bound is printed.

The reference restatement (`reference`) is the reference's computation in fp32 on the CPU: the host discount table,
the same masking, sequential torch.cumsum, the filler rule and the batch-wide MRR rule.
"""
import ctypes
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
E_INVALID, E_UNSUPPORTED = -1, -2           # ARB_E_INVALID_ARG, ARB_E_UNSUPPORTED (include/allrank_b200.h)
POW2, IDENTITY = 0, 1
S_MAX = 6684                                 # slate_smem_bytes(6684) fits the 227 KB opt-in; 6685 does not
SLATE_LENGTHS = [1, 2, 16, 17, 255, 256, 257, 4096, 4097, 5000, 6144, 6683, 6684]
LONG_BATCH = 60                              # 5 lengths above 4096 x 60 slates = 300 slates
PADS, FILLERS = [-1.0, 0.0, -5.0], [1.0, 0.0, 0.25]
WORST = {"ratio": 0.0, "torch": 0.0}


# ------------------------------------------------------------------------------------------------ the kernel
def c_ints(values):
    return None if values is None else (ctypes.c_int32 * len(values))(*values)


def launch(yp, yt, cut, mrr_ats, gain, pad, filler):
    """One arb_rank_metrics call with every output requested, into NaN / -7 prefilled buffers.  `cut` (DCG cut-offs
    in [0, S]) and `mrr_ats` (raw MRR cut-offs) are the same length: the C entry takes one count for both."""
    assert len(cut) == len(mrr_ats)
    from allrank_b200 import _lib
    from allrank_b200.metrics import discount_table
    B, S = yt.shape
    n = len(cut)
    out = {k: torch.full((B, n), NAN, device="cuda") for k in ("dcg", "idcg", "ndcg", "mrr")}
    out["order"] = torch.full((B, S), -7, dtype=torch.int32, device="cuda")
    scratch = torch.full((2 * B,), NAN, device="cuda")
    P = _lib.ptr
    rc = _lib.lib().arb_rank_metrics(P(yp), P(yt), B, S, P(discount_table(S, yp.device)), c_ints(cut),
                                     c_ints(mrr_ats), n, gain, pad, filler, P(out["dcg"]), P(out["idcg"]),
                                     P(out["ndcg"]), P(out["mrr"]), P(out["order"]), P(scratch),
                                     _lib.stream_ptr(yp.device))
    _lib.check(rc, "arb_rank_metrics")
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def bits(t):
    return np.ascontiguousarray(np.asarray(t, dtype=np.float32)).view(np.uint32)


def run(yp, yt, cut, mrr_ats, gain, pad, filler):
    """Twice on the device: the same bits both times, inputs untouched."""
    yp_d, yt_d = yp.cuda(), yt.cuda()
    first = launch(yp_d, yt_d, cut, mrr_ats, gain, pad, filler)
    second = launch(yp_d, yt_d, cut, mrr_ats, gain, pad, filler)
    for k in first:
        assert np.array_equal(first[k].view(np.uint32), second[k].view(np.uint32)), f"{k} differs between runs"
    assert np.array_equal(bits(yp_d.cpu()), bits(yp)) and np.array_equal(bits(yt_d.cpu()), bits(yt)), "input written"
    return first


# ------------------------------------------------------------------------------------------------ the reference
def stable_rankings(yp, yt, pad):
    """Order by score (padded items -inf), labels in that order (padded 0), and the ideal label sequence: what
    metrics.py:31-38 computes for dcg(y_pred, y_true) and dcg(y_true, y_true), with the sort made stable."""
    is_pad = yt == pad
    labels = yt.masked_fill(is_pad, 0.0)
    order = yp.masked_fill(is_pad, -INF).sort(dim=1, descending=True, stable=True).indices
    ideal_order = yt.masked_fill(is_pad, -INF).sort(dim=1, descending=True, stable=True).indices
    return order, labels.gather(1, order), labels.gather(1, ideal_order)


def gain_fn(gain):
    return (lambda x: torch.pow(2, x) - 1) if gain == POW2 else (lambda x: x)


def reference(yp, yt, cut, mrr_ats, gain, pad, filler):
    """metrics.py:7-113 in fp32 on the CPU at cut-offs in [0, S] (0: the empty prefix, DCG 0)."""
    from oracle.metrics_ref import discount_table
    B, S = yt.shape
    order, ranked, ideal = stable_rankings(yp, yt, pad)
    disc = discount_table(S)
    top = max(cut)

    def dcg(lab):
        cum = torch.cumsum((gain_fn(gain)(lab) * disc)[:, :top], dim=1)
        return torch.stack([cum[:, a - 1] if a > 0 else torch.zeros(B) for a in cut], dim=1)

    d, i = dcg(ranked), dcg(ideal)
    nd = d / i
    nd[i == 0] = filler
    best = ranked.max(dim=1).values
    pos = torch.where(ranked == best[:, None], torch.arange(S), S).min(dim=1).values.float()[:, None]
    r = torch.tensor(1.0) / (pos + torch.tensor(1.0))
    if bool(best.sum() == 0.0):
        r = torch.zeros_like(r)
    m = r * (pos < torch.tensor(mrr_ats, dtype=torch.float32)).float()
    return {"dcg": d.numpy(), "idcg": i.numpy(), "ndcg": nd.numpy(), "mrr": m.numpy(),
            "order": order.to(torch.int32).numpy()}


def ulp32(v):
    """ulp of fp32 at magnitude |v| (the spacing above |v| rounded to fp32: never below the ulp at |v|)."""
    return np.spacing(np.abs(np.asarray(v, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def fractional_bound(yp, yt, cut, gain, pad):
    """fp64 DCG / IDCG / NDCG and bounds on the error of the kernel's fp32 evaluation at cut-offs in [1, S].

    Per item, with exact gain t = 2^x - 1 (or x) and the fp32 discount d:
      exp2f(x) is within 2 ulp of 2^x (CUDA programming guide); subtracting 1 adds half an ulp; the product with d
      adds half an ulp of the result.  The running sum is kept in double (k additions, each within 2^-53 of the
      partial sum, bounded by the sum of magnitudes) and rounded to fp32 once (half an ulp).  fp64 evaluation error
      of the exact values is covered by 2^-50 of the sum of magnitudes.
    NDCG: |d/i - D/I| <= (Bd |I| + |D| Bi) / (|I| (|I| - Bi)) where |I| > Bi, plus half an ulp of the quotient."""
    from oracle.metrics_ref import discount_table
    _, ranked, ideal = stable_rankings(yp, yt, pad)
    disc = discount_table(yt.shape[1]).double().numpy()
    top = max(cut)
    idx = np.array(cut) - 1

    def dcg(lab):
        x = lab.double().numpy()[:, :top]
        if gain == POW2:
            p = np.exp2(x)
            e = 2.0 * ulp32(p)
            t = p - 1.0
            g_err = e + 0.5 * ulp32(np.abs(t) + e)
        else:
            t, g_err = x, np.zeros_like(x)
        d = disc[:top]
        w, w_err = t * d, g_err * d
        w_err = w_err + 0.5 * ulp32(np.abs(w) + w_err)
        mag = np.cumsum(np.abs(w) + w_err, axis=1)
        k = np.arange(1, top + 1)
        cum, cum_err = np.cumsum(w, axis=1), np.cumsum(w_err, axis=1) + (k * 2.0 ** -53 + 2.0 ** -50) * mag
        cum_err = cum_err + 0.5 * ulp32(np.abs(cum) + cum_err)
        return cum[:, idx], cum_err[:, idx]

    D, Bd = dcg(ranked)
    I, Bi = dcg(ideal)
    zero = np.stack([(ideal[:, :a] == 0).all(dim=1).numpy() for a in cut], axis=1)   # exactly 0: the filler case
    assert ((np.abs(I) > Bi) | zero).all(), "an ideal DCG too close to 0 to bound the quotient"
    with np.errstate(divide="ignore", invalid="ignore"):
        N = D / I
        Bn = (Bd * np.abs(I) + np.abs(D) * Bi) / (np.abs(I) * (np.abs(I) - Bi))
        Bn = Bn + 0.5 * ulp32(np.abs(N) + Bn)
    return {"dcg": (D, Bd), "idcg": (I, Bi), "ndcg": (N, Bn)}, zero


# ------------------------------------------------------------------------------------------------ comparisons
def assert_same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype == np.int32:
        bad = got != want
    else:
        g, w = got.astype(np.float32), want.astype(np.float32)
        bad = (np.isnan(g) != np.isnan(w)) | (~np.isnan(g) & (g.view(np.uint32) != w.view(np.uint32)))
    if bad.any():
        at = tuple(int(i) for i in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ, first at {at}: {got[at]!r} vs {want[at]!r}")


def assert_within(got, want, bound, what, torch_value=None, zero=None, filler=None):
    """|got - exact| <= bound; for ndcg, `filler` exactly where the ideal DCG is exactly 0 (`zero`)."""
    got = np.asarray(got, dtype=np.float64)
    live = np.ones(got.shape, dtype=bool)
    if zero is not None:
        assert (got[zero] == np.float32(filler)).all(), f"{what}: filler"
        live = ~zero
    err = np.abs(got[live] - want[live])
    ok = err <= bound[live]
    assert ok.all(), f"{what}: {int((~ok).sum())} outside the bound, worst ratio {np.max(err / bound[live]):.3g}"
    if err.size:
        WORST["ratio"] = max(WORST["ratio"], float(np.max(err / bound[live])))
    if torch_value is not None:
        terr = np.abs(np.asarray(torch_value, dtype=np.float64)[live] - want[live])
        assert (terr <= bound[live]).all(), f"{what}: torch's fp32 value lies outside the bound"
        if terr.size:
            WORST["torch"] = max(WORST["torch"], float(np.max(terr / bound[live])))


def check_case(yp, yt, cut, mrr_ats, pad, filler, fractional, gains=(POW2, IDENTITY)):
    for gain in gains:
        got = run(yp, yt, cut, mrr_ats, gain, pad, filler)
        want = reference(yp, yt, cut, mrr_ats, gain, pad, filler)
        tag = f"gain {gain} pad {pad} filler {filler}"
        assert_same(got["order"], want["order"], "order " + tag)
        assert_same(got["mrr"], want["mrr"], "mrr " + tag)
        if not fractional:
            for k in ("dcg", "idcg", "ndcg"):
                assert_same(got[k], want[k], f"{k} {tag}")
            continue
        live = [a for a in cut if a > 0]
        cols = [q for q, a in enumerate(cut) if a > 0]
        exact, zero = fractional_bound(yp, yt, live, gain, pad)
        for k in ("dcg", "idcg"):
            assert_within(got[k][:, cols], *exact[k], f"{k} {tag}", want[k][:, cols])
        assert_within(got["ndcg"][:, cols], *exact["ndcg"], f"ndcg {tag}", want["ndcg"][:, cols], zero, filler)
        at0 = [q for q, a in enumerate(cut) if a == 0]
        assert (got["dcg"][:, at0] == 0).all() and (got["idcg"][:, at0] == 0).all()
        assert (got["ndcg"][:, at0] == np.float32(filler)).all()


# ------------------------------------------------------------------------------------------------ inputs
def make_scores(kind, B, S, g):
    s = torch.randint(0, 3, (B, S), generator=g).float()           # heavy ties
    if kind == "special":
        r = torch.rand(B, S, generator=g)
        s[r < 0.05] = NAN
        s[(r >= 0.05) & (r < 0.10)] = INF
        s[(r >= 0.10) & (r < 0.20)] = -INF
        s[(r >= 0.20) & (r < 0.30)] = 0.0
        s[(r >= 0.30) & (r < 0.40)] = -0.0
    return s


INT_RANGES = [(0, 5), (-149, 31), (31, 128), (-149, 129)]


def make_labels(kind, B, S, pad, g):
    """Per slate b: a label range (b % 4 for integers) and a padding layout (b % 6): full, a random tail, random
    holes, a single real item, all-zero labels, all padded."""
    y = torch.empty(B, S)
    for b in range(B):
        if kind == "int":
            lo, hi = INT_RANGES[b % 4]
            y[b] = torch.randint(lo, hi, (S,), generator=g).float()
            y[b][(y[b] == 0) & (torch.rand(S, generator=g) < 0.5)] = -0.0
        elif kind == "frac_pos":
            y[b] = torch.rand(S, generator=g) * 5.0
        else:       # (-1, 0), kept 2^-10 from 0: nearer, 2^x - 1 is smaller than exp2f's own error at 1
            y[b] = -(2.0 ** -10 + (1.0 - 2.0 ** -9) * torch.rand(S, generator=g))
        layout = b % 6
        if layout == 1:
            y[b, int(torch.randint(1, S + 1, (1,), generator=g)):] = pad
        elif layout == 2:
            y[b][torch.rand(S, generator=g) < 0.3] = pad
        elif layout == 3:
            keep = int(torch.randint(0, S, (1,), generator=g))
            v = y[b, keep].clone()
            y[b] = pad
            y[b, keep] = v
        elif layout == 4:
            y[b] = 0.0
            y[b, S // 2 + 1:] = pad
        elif layout == 5:
            y[b] = pad
    return y


def dcg_cuts(S, g):
    """32 cut-offs in [0, S]: unsorted, duplicated, 1, S, 0 and the warp / block edges."""
    fixed = [S, 1, 0, S, 1, min(2, S), min(16, S), min(17, S), min(255, S), min(256, S), min(257, S), S - 1]
    return fixed + torch.randint(0, S + 1, (32 - len(fixed),), generator=g).tolist()


def mrr_cuts(S, g):
    """32 raw MRR cut-offs: not clipped, so above S, 0 and negative ones too."""
    fixed = [S, 1, 0, -1, S + 1, 2 * S, 7, 7, 1 << 30, -(1 << 30), S - 1, 2]
    return fixed + torch.randint(-2, S + 3, (32 - len(fixed),), generator=g).tolist()


CASES = [(S, scores, labels) for S in SLATE_LENGTHS for scores in ("ties", "special")
         for labels in ("int", "frac_pos", "frac_neg")]


@pytest.mark.parametrize("S,scores,labels", CASES, ids=[f"S{S}-{s}-{l}" for S, s, l in CASES])
def test_kernel_against_stable_reference(S, scores, labels):
    n = CASES.index((S, scores, labels))
    g = torch.Generator().manual_seed(1000 + n)
    pad, filler = PADS[n % 3], FILLERS[(n // 3) % 3]
    B = LONG_BATCH if S > 4096 else 24
    yp = make_scores(scores, B, S, g)
    yt = make_labels(labels, B, S, pad, g)
    check_case(yp, yt, dcg_cuts(S, g), mrr_cuts(S, g), pad, filler, labels != "int")


@pytest.mark.parametrize("labels", ["int", "frac_pos"])
def test_one_slate_at_the_longest_length(labels):
    g = torch.Generator().manual_seed(77)
    yp = make_scores("special", 1, S_MAX, g)
    yt = make_labels(labels, 1, S_MAX, -1.0, g)
    check_case(yp, yt, dcg_cuts(S_MAX, g), mrr_cuts(S_MAX, g), -1.0, 1.0, labels != "int")


def test_exactly_32_cutoffs_in_order_and_every_cutoff_from_1_to_32():
    g = torch.Generator().manual_seed(78)
    yp, yt = make_scores("ties", 12, 40, g), make_labels("int", 12, 40, -1.0, g)
    check_case(yp, yt, list(range(1, 33)), list(range(1, 33)), -1.0, 1.0, False)


def test_integer_labels_every_value_both_gains():
    """Each integer label from -149 to 128 alone at the top of a slate, so its gain is the first DCG term."""
    labels = torch.arange(-149, 129, dtype=torch.float32)
    B = labels.numel()
    yt = torch.full((B, 3), -1.0)
    yt[:, 0] = labels
    yt[:, 1] = 0.0
    yt[:, 2] = -1000.0
    yp = torch.tensor([[2.0, 1.0, 0.0]]).expand(B, 3).contiguous()
    check_case(yp, yt, [1, 2, 3], [1, 2, 3], -1000.0, 1.0, False)


# ------------------------------------------------------------------------------------------------ the MRR batch rule
def mrr_batch(B, S, relevant, g):
    """Labels 0 or padded everywhere, except slates `relevant` which carry one label 2 at a random position."""
    yt = torch.zeros(B, S)
    yt[torch.rand(B, S, generator=g) < 0.3] = -1.0
    for b in relevant:
        yt[b, int(torch.randint(0, S, (1,), generator=g))] = 2.0
    return make_scores("ties", B, S, g), yt


@pytest.mark.parametrize("B,S,relevant", [(300, 40, []), (300, 40, [299]), (300, 40, [0, 257]),
                                          (70000, 3, []), (70000, 3, [69999]), (70000, 3, "random")],
                         ids=["zero-300", "last-300", "two-300", "zero-70000", "last-70000", "random-70000"])
def test_mrr_batch_wide_zero_rule(B, S, relevant):
    """The 'no relevant item' rule is one scalar over the whole batch: it zeroes every slate when no slate has a
    label above 0, and must not fire when a single slate past the finalisation block's first 256 has one."""
    g = torch.Generator().manual_seed(B + S + len(relevant))
    if relevant == "random":
        yp, yt = make_scores("ties", B, S, g), torch.randint(-1, 5, (B, S), generator=g).float()
    else:
        yp, yt = mrr_batch(B, S, relevant, g)
    got = run(yp, yt, [1, 2, S, S], [1, 2, S, S + 5], POW2, -1.0, 1.0)
    want = reference(yp, yt, [1, 2, S, S], [1, 2, S, S + 5], POW2, -1.0, 1.0)
    assert_same(got["mrr"], want["mrr"], "mrr")
    assert_same(got["order"], want["order"], "order")
    if relevant == []:
        assert (got["mrr"] == 0).all()
    elif relevant != "random":
        assert (got["mrr"][relevant, 2] > 0).all()


def test_mrr_first_maximum_across_warps():
    """Tied maximum labels in different warps' strides of a 2000-item slate: the first in score order wins."""
    S, B = 2000, 6
    yp = torch.arange(S, 0, -1, dtype=torch.float32).expand(B, S).contiguous()   # score order = position order
    yt = torch.zeros(B, S)
    for b, where in enumerate([[300, 700], [1999], [33, 32 + 256, 31], [256, 257, 511], [5, 1000], list(range(S))]):
        yt[b, where] = 3.0
    yt[1, 0] = -1.0
    got = run(yp, yt, [S] * 4, [1, 300, 1000, S], POW2, -1.0, 1.0)
    want = reference(yp, yt, [S] * 4, [1, 300, 1000, S], POW2, -1.0, 1.0)
    assert_same(got["mrr"], want["mrr"], "mrr")
    assert np.allclose(1.0 / got["mrr"][:, 3], [301, 1999, 32, 257, 6, 1])   # (slate 1: the padded item ranks last)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_launch_nothing():
    from allrank_b200 import _lib
    from allrank_b200.metrics import discount_table
    lib, P, st = _lib.lib(), _lib.ptr, _lib.stream_ptr()

    def call(S=8, ats=(1, 2), mrr=(1, 2), yp=True, yt=True, disc=True, scratch=True, B=2, n=None):
        x = torch.zeros(B, S, device="cuda")
        out = torch.full((B, max(len(ats), 1)), NAN, device="cuda")
        sc = torch.zeros(2 * B, device="cuda")
        before = _lib.launch_count()
        rc = lib.arb_rank_metrics(P(x) if yp else None, P(x) if yt else None, B, S,
                                  P(discount_table(S, x.device)) if disc else None, c_ints(list(ats)),
                                  c_ints(list(mrr)), len(ats) if n is None else n, POW2, -1.0, 1.0, P(out), P(out),
                                  P(out), P(out), None, P(sc) if scratch else None, st)
        torch.cuda.synchronize()
        assert _lib.launch_count() == before, "a refused call launched a kernel"
        assert bool(torch.isnan(out).all()), "a refused call wrote an output"
        return rc

    assert call(S=S_MAX + 1, ats=(1,), mrr=(1,)) == E_UNSUPPORTED
    assert call(ats=tuple(range(1, 34)), mrr=tuple(range(1, 34))) == E_INVALID
    assert call(n=-1) == E_INVALID
    assert call(ats=(1, -1)) == E_INVALID
    assert call(ats=(9, 1)) == E_INVALID
    assert call(yp=False) == E_INVALID
    assert call(yt=False) == E_INVALID
    assert call(disc=False) == E_INVALID
    assert call(scratch=False) == E_INVALID
    assert call(S=0) == E_INVALID


def test_longest_slate_is_accepted():
    from allrank_b200 import _lib
    g = torch.Generator().manual_seed(5)
    yp, yt = make_scores("ties", 1, S_MAX, g), make_labels("int", 1, S_MAX, -1.0, g)
    before = _lib.launch_count()
    launch(yp.cuda(), yt.cuda(), [S_MAX], [S_MAX], POW2, -1.0, 1.0)
    assert _lib.launch_count() == before + 2


# ------------------------------------------------------------------------------------------------ the public wrappers
WRAPPER_ATS = [[1, 5, 10], [3, 3, 1, 10_000], [0, 2], [-1, 4], [7, -3, 2, 7], [2, -3]]


@pytest.mark.parametrize("S", [5, 17, 257, 6684])
@pytest.mark.parametrize("ats", WRAPPER_ATS, ids=str)
def test_public_wrappers_against_the_stable_oracle(S, ats):
    """ndcg / dcg / mrr / all_metrics / ranking, cut-offs included: <= 0 count from the end like the reference."""
    from allrank_b200 import metrics as M
    from oracle import metrics_ref as R
    g = torch.Generator().manual_seed(S * 31 + len(ats))
    B = 12
    yp, yt = make_scores("special", B, S, g), make_labels("int", B, S, -1.0, g).clamp(-3.0, 6.0)
    ypd, ytd = yp.cuda(), yt.cuda()
    identity = lambda x: x  # noqa: E731
    assert_same(M.ranking(ypd, ytd).cpu().numpy(), R.ranking(yp, yt, stable=True).to(torch.int32).numpy(), "ranking")
    assert_same(M.mrr(ypd, ytd, ats=ats).cpu().numpy(), R.mrr(yp, yt, ats=ats, stable=True).numpy(), "mrr")
    try:
        want = {"dcg": R.dcg(yp, yt, ats=ats, stable=True), "ndcg": R.ndcg(yp, yt, ats=ats, stable=True),
                "dcg_id": R.dcg(yp, yt, ats=ats, gain_function=identity, stable=True),
                "ndcg_f": R.ndcg(yp, yt, ats=ats, filler_value=0.25, stable=True)}
    except IndexError:
        for fn in (M.dcg, M.ndcg):
            with pytest.raises(IndexError):
                fn(ypd, ytd, ats=ats)
        with pytest.raises(IndexError):
            M.all_metrics(ypd, ytd, ats)
        return
    assert_same(M.dcg(ypd, ytd, ats=ats).cpu().numpy(), want["dcg"].numpy(), "dcg")
    assert_same(M.ndcg(ypd, ytd, ats=ats).cpu().numpy(), want["ndcg"].numpy(), "ndcg")
    assert_same(M.dcg(ypd, ytd, ats=ats, gain_function=identity).cpu().numpy(), want["dcg_id"].numpy(), "dcg id")
    assert_same(M.ndcg(ypd, ytd, ats=ats, filler_value=0.25).cpu().numpy(), want["ndcg_f"].numpy(), "ndcg filler")
    fused = M.all_metrics(ypd, ytd, ats)
    assert_same(fused["dcg"].cpu().numpy(), want["dcg"].numpy(), "fused dcg")
    assert_same(fused["ndcg"].cpu().numpy(), want["ndcg"].numpy(), "fused ndcg")
    assert_same(fused["mrr"].cpu().numpy(), R.mrr(yp, yt, ats=ats, stable=True).numpy(), "fused mrr")


def test_empty_cutoff_lists():
    from allrank_b200 import metrics as M
    yp, yt = torch.randn(3, 5, device="cuda"), torch.ones(3, 5, device="cuda")
    for fn in (M.dcg, M.ndcg):
        with pytest.raises(ValueError):
            fn(yp, yt, ats=[])
    with pytest.raises(ValueError):
        M.all_metrics(yp, yt, [])
    assert M.mrr(yp, yt, ats=[]).shape == (3, 0)


def test_golden_edges_from_the_reference(golden):
    """tests/golden/metrics_edges.npz (tools/make_golden_metrics_edges.py): the unmodified reference's outputs and
    exceptions.  Integer labels bit for bit; fractional ones within fractional_bound."""
    from allrank_b200 import metrics as M
    g = golden("metrics_edges")
    for name in (str(n) for n in g["names"]):
        call = json.loads(str(g[name + ":call"]))
        yp, yt = torch.from_numpy(g[name + ":pred"]), torch.from_numpy(g[name + ":true"])
        kw = {"padding_indicator": call["pad"]}
        gain = IDENTITY if call["gain"] == "identity" else POW2
        if call["fn"] != "mrr":
            kw["gain_function"] = M.identity_gain if gain == IDENTITY else M.pow2_gain
        if call["fn"] == "ndcg":
            kw["filler_value"] = call["filler"]
        fn = getattr(M, call["fn"])
        if call["raises"]:
            with pytest.raises({"IndexError": IndexError, "ValueError": ValueError}[call["raises"]]):
                fn(yp.cuda(), yt.cuda(), ats=call["ats"], **kw)
            continue
        got = fn(yp.cuda(), yt.cuda(), ats=call["ats"], **kw).cpu().numpy()
        want = g[name + ":out"]
        if not call["frac"] or call["fn"] == "mrr":
            assert_same(got, want, name)
            continue
        cut = M.dcg_cutoffs(call["ats"], yt.shape[1])
        exact, zero = fractional_bound(yp, yt, cut, gain, call["pad"])
        if call["fn"] == "ndcg":
            assert_within(got, *exact["ndcg"], name, want, zero, call["filler"])
        else:
            assert_within(got, *exact["dcg"], name, want)


# ------------------------------------------------------------------------------------------------ ranking users
class FixedScorer:
    def __init__(self, scores):
        self.scores = scores

    def score(self, X, mask, indices):
        return self.scores


@pytest.mark.parametrize("S", [16, 17, 300])
def test_rank_batch_gathers_in_the_stable_order(S):
    from allrank_b200 import inference
    g = torch.Generator().manual_seed(S)
    B, F = 9, 5
    scores = make_scores("special", B, S, g)
    yt = make_labels("int", B, S, -1.0, g).clamp(-1.0, 4.0)
    X = torch.randn(B, S, F, generator=g)
    order = scores.masked_fill(yt == -1, -INF).sort(dim=1, descending=True, stable=True).indices
    want_x, want_y = X.gather(1, order[..., None].expand(B, S, F)), yt.gather(1, order)
    x, y = inference.rank_batch(FixedScorer(scores.cuda()), X.cuda(), yt.cuda())
    assert np.array_equal(bits(x.cpu()), bits(want_x)) and np.array_equal(bits(y.cpu()), bits(want_y))
    x2, y2 = inference.reorder_slates(X.cuda(), yt.cuda(), order.cuda())
    assert np.array_equal(bits(x2.cpu()), bits(want_x)) and np.array_equal(bits(y2.cpu()), bits(want_y))


def test_metrics_on_clicked_slates_across_chunks():
    from allrank_b200 import inference
    from oracle import metrics_ref as R
    rng = np.random.RandomState(9)
    ys = [rng.choice([0, 0, 0, 1, -1], size=n).astype(np.int64) for n in [7] * 13 + [3] * 4 + [7, 1]]
    ys[2][:] = 0
    ys[5][:] = -1
    xs = [np.zeros((len(y), 2), dtype=np.float32) for y in ys]
    got = list(inference.metrics_on_clicked_slates((xs, ys), chunk=5))
    for y, row in zip(ys, got):
        yp = torch.arange(len(y), 0, -1, dtype=torch.float32)[None, :]
        yt = torch.tensor(y)[None, :].float()
        assert row["slate_length"] == len(y) and row["no_of_clicks"] == (y > 0).sum()
        assert row["dcg"] == R.dcg(yp, yt, stable=True).item()
        assert row["ndcg"] == R.ndcg(yp, yt, stable=True).item()


def test_report_worst_bound_ratio():
    """Runs last in this module: the worst |kernel - exact| / bound over the fractional-label cases above, and the
    same ratio for torch's fp32 evaluation."""
    print(f"\nworst fractional-label error / bound: kernel {WORST['ratio']:.3f}, torch fp32 {WORST['torch']:.3f}")
    assert WORST["ratio"] <= 1.0 and WORST["torch"] <= 1.0
