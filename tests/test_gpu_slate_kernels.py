"""The slate movers of csrc/slates.cu bit for bit against exact models, through the C ABI.

assemble_slates_kernel: every slate equals oracle/slates_ref.assemble -- the reference's FixLength rules (_pad and
_sample, dataset_loading.py:55-93) driven by HashSource, the host restatement of the kernel's counter hash -- in x, y
and indices, at query lengths around the block size and the sort's powers of two up to the largest accepted (16384),
at slate lengths from 1 to the largest the shared memory takes, at feature counts that take the float4 and the
scalar copy, with misaligned rows, label patterns from the reference's rule golden (tests/golden/slates_rules.npz),
redraws up to the 1024-attempt cap, unknown query numbers, 64-bit seeds and a batch of ~70 000 slates.
gather_slates_kernel: torch.gather, bit for bit.  Every output is prefilled with NaN or a sentinel, every launch runs
twice and must give the same bits and leave its inputs untouched."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import slates_ref

pytestmark = pytest.mark.gpu

SMEM_LIMIT = 200 * 1024
SENTINEL = -0x5A5A5A5A5A5A5A5A


def lib():
    from allrank_b200 import _lib, data, inference  # noqa: F401  (registers the signatures)
    return _lib.lib()


def shifted(n, shift, fill=float("nan")):
    """A float32 device vector of n elements starting `shift` floats into its allocation (shift 1: 4-byte aligned)."""
    base = torch.full((n + 4,), fill, dtype=torch.float32, device="cuda")
    return base[shift:shift + n]


class Corpus:
    def __init__(self, lengths, F, labels=None, seed=0, docs_shift=0):
        rng = np.random.RandomState(seed)
        self.offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        N = int(self.offsets[-1])
        self.X = rng.randn(N, F).astype(np.float32)
        self.y = (rng.randint(0, 5, N) * (rng.rand(N) < 0.3)).astype(np.float32) if labels is None else \
            np.asarray(labels, dtype=np.float32)
        self.F, self.Q, self.max_len = F, len(lengths), int(max(lengths))
        self.docs_x = shifted(N * F, docs_shift)
        self.docs_x.copy_(torch.from_numpy(self.X).reshape(-1))
        self.docs_y = torch.from_numpy(self.y).cuda()
        self.d_off = torch.from_numpy(self.offsets).cuda()


def launch(c, queries, S, seed, x_shift=0, max_len=None):
    """Two launches of arb_assemble_slates into prefilled outputs: (x, y, idx) as numpy, checked for repeatability."""
    from allrank_b200 import _lib
    q = torch.as_tensor(np.asarray(queries, dtype=np.int64)).cuda()
    B, F = q.numel(), c.F
    inputs = [t.clone() for t in (c.docs_x, c.docs_y, c.d_off, q)]
    runs = []
    for _ in range(2):
        x = shifted(B * S * F, x_shift)
        y = torch.full((B, S), float("nan"), device="cuda")
        idx = torch.full((B, S), SENTINEL, dtype=torch.int64, device="cuda")
        rc = lib().arb_assemble_slates(_lib.ptr(c.docs_x), _lib.ptr(c.docs_y), _lib.ptr(c.d_off), c.Q, _lib.ptr(q),
                                       B, S, F, c.max_len if max_len is None else max_len,
                                       ctypes.c_uint64(seed & (2 ** 64 - 1)), _lib.ptr(x), _lib.ptr(y), _lib.ptr(idx),
                                       _lib.stream_ptr())
        _lib.check(rc, "arb_assemble_slates")
        runs.append((x.view(torch.int32).cpu().numpy().reshape(B, S, F), y.view(torch.int32).cpu().numpy(),
                     idx.cpu().numpy()))
    for a, b in zip(*runs):
        assert np.array_equal(a, b)                                        # same bits twice
    for before, t in zip(inputs, (c.docs_x, c.docs_y, c.d_off, q)):
        assert torch.equal(before.view(torch.int32) if before.is_floating_point() else before,
                           t.view(torch.int32) if t.is_floating_point() else t)
    return runs[0]


def check(c, queries, S, seed, **kw):
    x, y, idx = launch(c, queries, S, seed, **kw)
    ex, ey, ei = slates_ref.assemble(c.X, c.y, c.offsets, queries, S, seed)
    bad = np.nonzero((idx != ei).any(axis=1) | (y != ey.view(np.int32)).any(axis=1))[0]
    assert len(bad) == 0, ("slates differ", bad[:8].tolist(), idx[bad[0]][:12].tolist(), ei[bad[0]][:12].tolist())
    assert np.array_equal(x, ex.view(np.int32))
    return ei


LENGTHS = [63, 64, 65, 255, 256, 257, 1023, 1024, 1025, 1251, 8191, 8192, 8193, 16383, 16384]


@pytest.fixture(scope="module")
def long_corpus():
    S_values = (1, 2, 20, 240, 256, 257, 1000)
    lengths = LENGTHS + [s + d for s in S_values for d in (-1, 0, 1) if s + d > 0]
    return Corpus(lengths, F=4, seed=1)


@pytest.mark.parametrize("S", [1, 2, 20, 240, 256, 257, 1000])
def test_query_lengths_around_every_power_of_two(long_corpus, S):
    c = long_corpus
    ei = check(c, np.arange(c.Q), S, seed=0x1234_5678_9ABC + S)
    lengths = np.diff(c.offsets)
    assert ((ei >= 0).sum(axis=1) == np.minimum(lengths, S)).all()


def test_largest_slates_beside_the_largest_query():
    """Beside a 16384-item query the sort takes 128 KB: S = 16384 still samples (192 KB in all); a longer slate needs
    no keys, since no query can be sampled to it, and is refused only above 51200 ints (200 KB)."""
    smem = lib().arb_assemble_slates_smem_bytes
    assert smem(16384, 16384) == 16384 * 12 <= SMEM_LIMIT < smem(16385, 16384)
    assert smem(16384, 51200) == SMEM_LIMIT < smem(16384, 51201)
    c = Corpus([16384, 5, 16383], F=3, seed=2)
    check(c, [0, 2, 0, 1, 2], 16384, seed=8)                                 # sampled at the longest slate that samples
    check(c, [0, 1, 2, 0], 16383, seed=9)
    check(c, [0, 1, 2], 51200, seed=7)                                       # the longest accepted: all padding


RULES = np.load(os.path.join(os.path.dirname(__file__), "golden", "slates_rules.npz"), allow_pickle=False)


@pytest.mark.parametrize("name", [str(n) for n in RULES["names"]])
def test_rule_golden_label_patterns(name):
    """Each pattern of the reference's rule golden as a query, drawn 64 times: the kernel keeps, redraws and appends
    where the reference's rules do (label sums of 0, below 0, NaN and fractional 1, -0.0, S = 1, n == S)."""
    y = RULES[f"{name}:y"].astype(np.float32)
    S = json.loads(str(RULES[f"{name}:call"]))["slate_length"]
    c = Corpus([len(y)], F=5, labels=y, seed=3)
    check(c, np.zeros(64, dtype=np.int64), S, seed=0xC0FFEE ^ len(name))


@pytest.mark.parametrize("n,S", [(1251, 20), (300, 240), (1024, 2)])
def test_rare_relevant_items_force_redraws(n, S):
    y = np.zeros(n, dtype=np.float32)
    y[[n // 3, n - 1]] = [1.0, 1.0]                                         # sum 2: the redraw branch
    c = Corpus([n], F=4, labels=y, seed=4)
    check(c, np.zeros(48, dtype=np.int64), S, seed=99 + n)


class CountingSource(slates_ref.HashSource):
    def choice_n(self, n, k, attempt):
        self.attempts = attempt + 1
        return super().choice_n(n, k, attempt)


def test_the_attempt_cap_and_a_late_success():
    """n = 2048, S = 1, one item of label 2: a slate that misses it 1024 times keeps its last draw; another finds it
    after several draws.  The seed is searched on the host."""
    n = 2048
    y = np.zeros(n, dtype=np.float32)
    y[777] = 2.0
    X = np.zeros((n, 1), dtype=np.float32)
    for seed in range(1, 200):
        srcs = [CountingSource(seed, b) for b in range(2)]
        out = [slates_ref.fix_length(X, y, 1, s)[2][0] for s in srcs]
        if out[0] != 777 and srcs[0].attempts == 1024 and out[1] == 777 and srcs[1].attempts > 1:
            break
    else:
        pytest.fail("no seed found")
    c = Corpus([n], F=2, labels=y, seed=5)
    ei = check(c, [0, 0], 1, seed=seed)
    assert ei[0, 0] != 777 and ei[1, 0] == 777


@pytest.mark.parametrize("F", [1, 3, 4, 46, 136, 137, 700])
def test_feature_counts(F):
    lengths = [1, 17, 40, 63, 64, 65, 100, 257, 30, 64]
    c = Corpus(lengths, F=F, seed=6 + F)
    check(c, [0, 3, 4, 5, 6, 7, 8, 9, 2, 1, 7, 7], 64, seed=F)


@pytest.mark.parametrize("F", [4, 136])
@pytest.mark.parametrize("docs_shift,x_shift", [(1, 0), (0, 1), (1, 1)])
def test_misaligned_rows_take_the_scalar_copy(F, docs_shift, x_shift):
    c = Corpus([10, 64, 200, 65], F=F, seed=7, docs_shift=docs_shift)
    check(c, [0, 1, 2, 3, 2], 64, seed=11, x_shift=x_shift)


def test_repeated_and_unknown_queries_and_64_bit_seeds():
    c = Corpus([30, 70, 12, 300], F=8, seed=8)
    queries = [1, 1, 1, -1, 3, 4, 2 ** 40, 3, 1, 0, -(2 ** 40), 2, 3]
    for seed in (0, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 63 + 5, 2 ** 64 - 1):
        ei = check(c, queries, 20, seed)
        for b in (3, 5, 6, 10):
            assert (ei[b] == -1).all()
    a = launch(c, queries, 20, 2 ** 32 + 7)[2]
    b = launch(c, queries, 20, 7)[2]
    assert not np.array_equal(a, b)                                          # the seed's high half is hashed


def test_a_batch_of_70000_slates():
    rng = np.random.RandomState(9)
    c = Corpus(list(rng.randint(10, 41, 50)), F=3, seed=9)
    check(c, rng.randint(0, 50, 70_003), 20, seed=2 ** 64 - 3)


def test_refusals_launch_nothing():
    from allrank_b200 import _lib
    c = Corpus([16384, 20], F=4, seed=10)
    q = torch.zeros(2, dtype=torch.int64, device="cuda")
    x = torch.empty(2 * 51200 * 4, device="cuda")
    y = torch.empty(2 * 51200, device="cuda")
    idx = torch.empty(2 * 51200, dtype=torch.int64, device="cuda")
    good = dict(docs_x=c.docs_x, docs_y=c.docs_y, offsets=c.d_off, n_queries=2, queries=q, B=2, S=20, F=4,
                max_len=16384, x=x, y=y, idx=idx)

    def call(**kw):
        a = dict(good, **kw)
        p = {k: (_lib.ptr(v) if isinstance(v, torch.Tensor) else v) for k, v in a.items()}
        return lib().arb_assemble_slates(p["docs_x"], p["docs_y"], p["offsets"], p["n_queries"], p["queries"],
                                         p["B"], p["S"], p["F"], p["max_len"], ctypes.c_uint64(1), p["x"], p["y"],
                                         p["idx"], _lib.stream_ptr())

    before = _lib.launch_count()
    for k in ("docs_x", "docs_y", "offsets", "queries", "x", "y", "idx"):
        assert call(**{k: None}) == -1, k
    for k in ("B", "S", "F", "max_len", "n_queries"):
        for v in (0, -1):
            assert call(**{k: v}) == -1, (k, v)
    assert call(max_len=16385) == -2                                         # 32768 keys: 256 KB
    assert call(S=51201) == -2                                               # S ints above 200 KB
    assert call(S=30000, max_len=30000) == -2
    assert _lib.launch_count() == before
    assert call(S=16384) == 0 and call(S=51200) == 0                         # the largest accepted shapes launch
    torch.cuda.synchronize()
    assert _lib.launch_count() == before + 2
    o = torch.zeros(4, dtype=torch.int32, device="cuda")
    for args in ((None, y, o, 1, 2, 2, x, y), (x, None, o, 1, 2, 2, x, y), (x, y, None, 1, 2, 2, x, y),
                 (x, y, o, 1, 2, 2, None, y), (x, y, o, 1, 2, 2, x, None), (x, y, o, 0, 2, 2, x, y),
                 (x, y, o, 1, 0, 2, x, y), (x, y, o, 1, 2, -1, x, y)):
        p = [_lib.ptr(a) if isinstance(a, torch.Tensor) or a is None else a for a in args]
        assert lib().arb_gather_slates(*p, _lib.stream_ptr()) == -1
    assert _lib.launch_count() == before + 2


def gather(x, y, order, x_shift=0):
    from allrank_b200 import _lib
    B, S, F = x.shape
    xs = shifted(B * S * F, x_shift)
    xs.copy_(x.reshape(-1))
    inputs = (xs.clone(), y.clone(), order.clone())
    runs = []
    for _ in range(2):
        xo = shifted(B * S * F, x_shift)
        yo = torch.full((B, S), float("nan"), device="cuda")
        rc = lib().arb_gather_slates(_lib.ptr(xs), _lib.ptr(y), _lib.ptr(order), B, S, F, _lib.ptr(xo), _lib.ptr(yo),
                                     _lib.stream_ptr())
        _lib.check(rc, "arb_gather_slates")
        runs.append((xo.view(torch.int32).reshape(B, S, F).clone(), yo.view(torch.int32).clone()))
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    assert torch.equal(inputs[0].view(torch.int32), xs.view(torch.int32))
    assert torch.equal(inputs[1].view(torch.int32), y.view(torch.int32)) and torch.equal(inputs[2], order)
    return runs[0]


@pytest.mark.parametrize("F", [1, 3, 4, 46, 136, 137, 700])
@pytest.mark.parametrize("repeats", [False, True])
def test_gather_matches_torch_gather(F, repeats):
    g = torch.Generator(device="cuda").manual_seed(F * 2 + repeats)
    B, S = (3, 257) if F >= 136 else (17, 240)
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, S, F), generator=g, device="cuda", dtype=torch.int32)
    x = bits.view(torch.float32)                                             # any bit pattern, NaN payloads included
    y = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, S), generator=g, device="cuda", dtype=torch.int32).view(torch.float32)
    if repeats:
        order = torch.randint(0, S, (B, S), generator=g, device="cuda")
    else:
        order = torch.stack([torch.randperm(S, generator=g, device="cuda") for _ in range(B)])
    order = order.to(torch.int32)
    for x_shift in ((0, 1) if F % 4 == 0 else (0,)):
        xo, yo = gather(x, y, order, x_shift)
        ol = order.long()
        assert torch.equal(xo, torch.gather(bits, 1, ol[..., None].expand(B, S, F)))
        assert torch.equal(yo, torch.gather(y.view(torch.int32), 1, ol))


@pytest.mark.parametrize("F", [3, 4])
def test_gather_at_a_million_rows(F):
    g = torch.Generator(device="cuda").manual_seed(F)
    B, S = 4096, 256
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (B, S, F), generator=g, device="cuda", dtype=torch.int32)
    y = torch.randn(B, S, generator=g, device="cuda")
    order = torch.argsort(torch.rand(B, S, generator=g, device="cuda"), dim=1).to(torch.int32)
    order[::3] = order[::3].flip(1)[:, :1]                                     # every third slate: one row repeated
    xo, yo = gather(bits.view(torch.float32), y, order)
    ol = order.long()
    assert torch.equal(xo, torch.gather(bits, 1, ol[..., None].expand(B, S, F)))
    assert torch.equal(yo, torch.gather(y, 1, ol).view(torch.int32))


@pytest.mark.parametrize("F", [136, 46])
def test_device_loader_end_to_end(F):
    """An MSLR-shaped corpus built here (queries of 1 to 1251 items, labels 0-4, some all-zero and single-relevant
    queries) read by DeviceSlateLoader under torch.manual_seed: every batch is the model's, given the loader's seeds."""
    from allrank_b200.data import DeviceSlateLoader, SlateStore
    rng = np.random.RandomState(F)
    lengths = np.concatenate([rng.randint(1, 1252, 90), [1251, 240, 239, 241]])
    N = int(lengths.sum())
    X = rng.randn(N, F).astype(np.float32)
    y = np.where(rng.rand(N) < 0.1, rng.randint(1, 5, N), 0).astype(np.float32)
    offsets = np.concatenate([[0], np.cumsum(lengths)])
    for q in range(0, 20, 2):
        y[offsets[q]:offsets[q + 1]] = 0.0                                     # no relevant item
        if q % 4 == 0:
            y[offsets[q] + rng.randint(lengths[q])] = 1.0                      # exactly one
    store = SlateStore(X, y, np.repeat(np.arange(len(lengths)), lengths), device="cuda")
    assert np.array_equal(store.offsets_host, offsets)
    S, bs = 240, 32
    torch.manual_seed(17)
    batches = list(DeviceSlateLoader(store, batch_size=bs, slate_length=S, shuffle=True))
    torch.manual_seed(17)                                                      # the loader's draws, replayed
    order = torch.randperm(len(lengths))
    seeds = [int(torch.randint(0, 2 ** 62, (1,)).item()) for _ in range(len(batches))]
    for k, (xb, yb, ib) in enumerate(batches):
        ex, ey, ei = slates_ref.assemble(X, y, offsets, order[k * bs:(k + 1) * bs].numpy(), S, seeds[k])
        assert np.array_equal(ib.cpu().numpy(), ei), k
        assert np.array_equal(yb.cpu().numpy().view(np.int32), ey.view(np.int32))
        assert np.array_equal(xb.cpu().numpy().view(np.int32), ex.view(np.int32))


def test_inclusion_is_uniform_at_mslr_length():
    """A 1251-item query without relevant items sampled to 240, 4096 times: each item is included with probability
    240 / 1251 (a check of the hash's quality at a realistic length)."""
    n, S, trials = 1251, 240, 4096
    c = Corpus([n], F=1, labels=np.zeros(n), seed=12)
    _, _, idx = launch(c, np.zeros(trials, dtype=np.int64), S, seed=31337)
    counts = np.bincount(idx.ravel(), minlength=n)
    p = S / n
    sd = np.sqrt(trials * p * (1 - p))
    assert np.abs(counts - trials * p).max() < 5.5 * sd
    assert abs(np.std(counts) / sd - 1) < 0.1                                # binomial spread, not more, not less
