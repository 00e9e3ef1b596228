import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def golden():
    cache = {}

    def load(name):
        if name not in cache:
            cache[name] = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
        return cache[name]

    return load


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a box without a GPU skips the `gpu`-marked tests instead of failing them."""
    import torch
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture
def dense_rows():
    """Pin the scorer to the dense [B*S] row layout for one test (restored afterwards).  Used by the tests that compare
    EVERY position of the score tensor -- padded items included -- or send a gradient into padded items, i.e. that
    check the kernels against what the reference computes for padded rows; the packed layout (the default) scores those
    items 0 by design (include/allrank_b200.h: arb_set_pack_rows) and is tied to the dense layout bit for bit on the
    real items by tests/test_gpu_pack_rows.py."""
    from allrank_b200 import _lib
    lib = _lib.lib()
    lib.arb_set_pack_rows(0)
    yield
    lib.arb_set_pack_rows(_lib.default_pack_rows())
