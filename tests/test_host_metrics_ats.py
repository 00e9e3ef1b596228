"""The DCG cut-off rule of allrank_b200.metrics (dcg_cutoffs), without a GPU.

The reference keeps the first max(clipped ats) cumulative DCG columns and reads column `at - 1` of them
(allrank/models/metrics.py:58-75), so a cut-off <= 0 counts from the end.  `kept_columns_rule` restates that indexing
on a tensor of cut-offs 1..S; dcg_cutoffs must name the same cut-off for every list, and raise where it raises.
"""
import json

import pytest
import torch

from allrank_b200.metrics import dcg_cutoffs


def kept_columns_rule(ats, S):
    clipped = [min(a, S) for a in ats]
    columns = torch.arange(1, S + 1)[:max(clipped)]
    return columns[torch.tensor(clipped, dtype=torch.long) - 1].tolist()


ATS_LISTS = [[1], [5], [9], [0, 2], [0, 3], [-1, 4], [-2, 5], [7, 0], [-2], [-4], [2, 2, 0, -1, 5, 1], [5, 1, 3],
             [12, -3, 12, 4], [3, 1, 2, -2]]


@pytest.mark.parametrize("S", [1, 2, 5, 6684])
@pytest.mark.parametrize("ats", ATS_LISTS, ids=str)
def test_cutoffs_follow_the_reference_indexing(ats, S):
    try:
        want = kept_columns_rule(ats, S)
    except IndexError:
        with pytest.raises(IndexError):
            dcg_cutoffs(ats, S)
        return
    got = dcg_cutoffs(ats, S)
    assert got == want
    assert all(1 <= a <= S for a in got)


@pytest.mark.parametrize("ats,S", [([0], 5), ([-5], 5), ([3, -3], 5), ([-1], 1), ([0, -1], 1), ([2, -2], 5)])
def test_cutoffs_before_the_first_column_raise_index_error(ats, S):
    with pytest.raises(IndexError):
        kept_columns_rule(ats, S)
    with pytest.raises(IndexError):
        dcg_cutoffs(ats, S)


def test_empty_list_raises_value_error():
    with pytest.raises(ValueError):
        dcg_cutoffs([], 5)


def test_positive_cutoffs_are_only_clipped():
    assert dcg_cutoffs([1, 5, 10, 5000], 240) == [1, 5, 10, 240]
    assert dcg_cutoffs(range(1, 33), 7) == [min(a, 7) for a in range(1, 33)]


def test_the_reference_raises_what_the_rule_raises(golden):
    """Every exception the unmodified reference raised on a cut-off list in tests/golden/metrics_edges.npz (written by
    tools/make_golden_metrics_edges.py) is the one dcg_cutoffs raises; every list it accepted is accepted."""
    g = golden("metrics_edges")
    seen = 0
    for name in g["names"]:
        call = json.loads(str(g[str(name) + ":call"]))
        if call["fn"] == "mrr" or call["ats"] is None:
            continue
        S = g[str(name) + ":true"].shape[1]
        seen += 1
        if call["raises"]:
            with pytest.raises({"IndexError": IndexError, "ValueError": ValueError}[call["raises"]]):
                dcg_cutoffs(call["ats"], S)
        else:
            assert len(dcg_cutoffs(call["ats"], S)) == g[str(name) + ":out"].shape[1]
    assert seen >= 10
