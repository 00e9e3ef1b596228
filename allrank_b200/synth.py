"""Synthetic MSLR-WEB30K-shaped slates (SURVEY.md section 8d) for benchmarks, smoke and tests.

Shapes and conventions follow the reference's data pipeline
(/root/reference/allrank/data/dataset_loading.py:15-16,29,88-93): features fp32 `[B,S,F]` zeroed on
padded rows, labels fp32 `[B,S]` holding small integers with -1 = padding, indices int64 `[B,S]`
with -1 = padding.  Label marginals approximate MSLR-WEB30K; true slate lengths ~ N(120, 60)
clipped to [1, S].  No dataset is read: the benchmark and the tests need no download.
"""
import torch

LABEL_P = (0.516, 0.322, 0.134, 0.018, 0.010)
PADDED_Y_VALUE = -1
PADDED_INDEX_VALUE = -1


def make_slates(batch, slate_len, n_features=136, seed=1234, device="cpu", mean_len=120.0, std_len=60.0,
                full=False):
    """Return (x [B,S,F] f32, y [B,S] f32, indices [B,S] i64), generated with a CPU generator so the
    same seed gives the same slates on every device."""
    g = torch.Generator().manual_seed(int(seed))
    x = torch.randn(batch, slate_len, n_features, generator=g, dtype=torch.float32)
    y = torch.multinomial(torch.tensor(LABEL_P), batch * slate_len, replacement=True, generator=g)
    y = y.view(batch, slate_len).float()
    if full:
        length = torch.full((batch,), slate_len, dtype=torch.long)
    else:
        length = torch.clamp(torch.round(torch.randn(batch, generator=g) * std_len + mean_len), 1, slate_len).long()
    pos = torch.arange(slate_len)[None, :]
    is_pad = pos >= length[:, None]
    y[is_pad] = PADDED_Y_VALUE
    x[is_pad] = 0.0
    idx = pos.expand(batch, slate_len).clone()
    idx[is_pad] = PADDED_INDEX_VALUE
    return x.to(device), y.to(device), idx.to(device)


def make_scores(batch, slate_len, seed=4321, device="cpu", scale=1.0):
    """Tie-free fp32 scores (ties have measure zero for randn; asserted in tests)."""
    g = torch.Generator().manual_seed(int(seed))
    return (torch.randn(batch, slate_len, generator=g, dtype=torch.float32) * scale).to(device)
