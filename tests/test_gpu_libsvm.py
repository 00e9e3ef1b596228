"""The device LibSVM parser (csrc/libsvm.cu) on the GPU against what sklearn's load_svmlight_file + SlateStore store,
bit for bit: the golden arrays of tools/make_golden_libsvm.py, and sklearn itself where it is importable.  Every case
is parsed twice into NaN-filled outputs and must give the same bits both times."""
import hashlib
import io
import os
import warnings

import numpy as np
import pytest
import torch

from allrank_b200 import _lib
from allrank_b200.data import DeviceSlateLoader, LibSVMPlan, SlateStore, read_svm_to_device
from tests import libsvm_cases as C

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SMALL = np.load(os.path.join(GOLDEN, "libsvm_small.npz"))
SMALL_NAMES = sorted({k.rsplit(".", 1)[0] for k in SMALL.files})
try:
    import sklearn  # noqa: F401
    HAVE_SKLEARN = True
except ImportError:
    HAVE_SKLEARN = False


def _parse(text_bytes):
    """Parses text_bytes twice into NaN-filled outputs; returns (docs_x bits, docs_y bits, qids) after checking that
    both runs agree bit for bit and the store built from them has the same offsets."""
    dev = torch.device("cuda", 0)
    runs = []
    for _ in range(2):
        text = read_svm_to_device(io.BytesIO(text_bytes), dev)
        plan = LibSVMPlan(text)
        x = torch.full((plan.n_rows, plan.n_features), float("nan"), device=dev)
        y = torch.full((plan.n_rows,), float("nan"), device=dev)
        q = torch.full((plan.n_rows,), -12345, dtype=torch.int64, device=dev)
        plan.write(x, y, q)
        torch.cuda.synchronize()
        runs.append((x.cpu().numpy().view(np.uint32), y.cpu().numpy().view(np.uint32), q.cpu().numpy()))
    for a, b in zip(*runs):
        assert np.array_equal(a, b)
    return runs[0]


def _store(text_bytes):
    return SlateStore.from_svm_file(io.BytesIO(text_bytes), device="cuda:0", parser="device")


@pytest.mark.parametrize("name", SMALL_NAMES)
def test_small_files_match_sklearn_bit_for_bit(name):
    text = SMALL[name + ".text"].tobytes()
    xb, yb, _ = _parse(text)
    assert np.array_equal(xb, SMALL[name + ".docs_x"])
    assert np.array_equal(yb, SMALL[name + ".docs_y"])
    st = _store(text)
    n_features, longest = SMALL[name + ".meta"].tolist()
    assert np.array_equal(st.offsets_host, SMALL[name + ".offsets"])
    assert np.array_equal(st.offsets.cpu().numpy(), SMALL[name + ".offsets"])
    assert (st.n_features, st.longest_query_length) == (n_features, longest)
    if HAVE_SKLEARN:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            ref = C.reference_arrays(text)
        assert np.array_equal(xb, ref["docs_x"].view(np.uint32))
        assert np.array_equal(yb, ref["docs_y"].view(np.uint32))


def test_mslr_shaped_file_matches_sklearn(tmp_path):
    rows, seed, n_features, longest = np.load(os.path.join(GOLDEN, "libsvm_mslr.npz"))["meta"].tolist()
    golden = np.load(os.path.join(GOLDEN, "libsvm_mslr.npz"))
    text = C.mslr_text(rows, seed=seed)
    path = tmp_path / "train.txt"
    path.write_bytes(text)
    xb, yb, _ = _parse(text)
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    assert sha(xb) == str(golden["docs_x_sha"]) and sha(yb) == str(golden["docs_y_sha"])
    st = SlateStore.from_svm_file(str(path), device="cuda:0", parser="device")   # from a path: chunked reads
    assert sha(st.offsets_host) == str(golden["offsets_sha"])
    assert (st.n_features, st.longest_query_length, st.docs_x.shape[0]) == (n_features, longest, rows)
    assert sha(st.docs_x.cpu().numpy()) == str(golden["docs_x_sha"])


@pytest.mark.parametrize("name", sorted(C.REFUSED_CASES))
def test_refuses_what_sklearn_refuses(name):
    text, exc = C.REFUSED_CASES[name]
    if HAVE_SKLEARN:
        with pytest.raises(exc):
            C.reference_arrays(text)
    dev = torch.device("cuda", 0)
    t = read_svm_to_device(io.BytesIO(text), dev)
    before = _lib.launch_count()
    with pytest.raises(exc) as info:
        LibSVMPlan(t)
    # pass 1 only: newline count + scan, index, summary init, pass 1, row scan -- pass 2 never launches
    assert _lib.launch_count() - before == 6
    if name == "late_error":
        assert "line 51" in str(info.value)
    with pytest.raises(exc):
        _store(text)


def test_argument_refusals_launch_nothing():
    lib = _lib.lib()
    dev = torch.device("cuda", 0)
    text = read_svm_to_device(io.BytesIO(b"1 qid:1 1:2\n"), dev)
    buf = torch.zeros(16, dtype=torch.int64, device=dev)
    p, st = _lib.ptr, _lib.stream_ptr(dev)
    before = _lib.launch_count()
    assert lib.arb_libsvm_count_lines(None, 12, p(buf), st) == -1
    assert lib.arb_libsvm_count_lines(p(text), 0, p(buf), st) == -1
    assert lib.arb_libsvm_count_lines(text[1:].data_ptr(), 11, p(buf), st) == -1                 # misaligned
    assert lib.arb_libsvm_index_lines(p(text), 12, None, p(buf), st) == -1
    assert lib.arb_libsvm_pass1(p(text), 12, p(buf), 1, 3, p(buf), p(buf), p(buf), st) == -1     # n_lines > nl + 1
    assert lib.arb_libsvm_pass1(p(text), 12, None, 1, 1, p(buf), p(buf), p(buf), st) == -1
    assert lib.arb_libsvm_pass2(p(text), 12, p(buf), 1, 1, p(buf), p(buf), 1, 2, 1, p(buf), p(buf), p(buf), st) == -1
    assert lib.arb_libsvm_pass2(p(text), 12, p(buf), 1, 1, p(buf), p(buf), 1, 0, 0, p(buf), p(buf), p(buf), st) == -1
    assert lib.arb_libsvm_pass2(p(text), 12, p(buf), 1, 1, p(buf), p(buf), 2, 0, 1, p(buf), p(buf), p(buf), st) == -1
    assert lib.arb_libsvm_pass2(p(text), 12, p(buf), 1, 1, p(buf), p(buf), 1, 0, 2 ** 31 + 1, p(buf), p(buf), p(buf),
                                st) == -1                                                     # above 2^31 features
    assert _lib.launch_count() == before
    plan = LibSVMPlan(text)
    with pytest.raises(ValueError):
        plan.write(torch.empty((1, 2), device=dev), torch.empty(1, device=dev),
                   torch.empty(1, dtype=torch.int64, device=dev))
    with pytest.raises(ValueError):
        plan.write(torch.empty((1, 1), device=dev), torch.empty(1, device=dev), torch.empty(1, device=dev))


def test_empty_file_gives_sklearn_shape():
    st = _store(b"")
    assert (len(st), st.n_features, st.longest_query_length, tuple(st.docs_x.shape)) == (0, 1, 0, (0, 1))


def test_loader_batches_match_the_sklearn_parsed_store():
    name = "hard_numerals"                         # 416 rows in queries of 10, with inf / nan / -0 values
    text = SMALL[name + ".text"].tobytes()
    dev = torch.device("cuda", 0)
    mine = _store(text)
    ref = SlateStore.__new__(SlateStore)           # what SlateStore(*load_svmlight_file(...)) holds
    ref._init_from_groups(SMALL[name + ".docs_x"].view(np.float32), SMALL[name + ".docs_y"].view(np.float32),
                          SMALL[name + ".offsets"], dev, None)
    for S, shuffle in ((4, True), (mine.longest_query_length, False), (16, False)):
        batches = []
        for st in (mine, ref):
            torch.manual_seed(11)
            batches.append(list(DeviceSlateLoader(st, 8, slate_length=S, shuffle=shuffle)))
        assert len(batches[0]) == len(batches[1]) > 0
        for (xa, ya, ia), (xb, yb, ib) in zip(*batches):
            assert torch.equal(xa.view(torch.int32), xb.view(torch.int32))
            assert torch.equal(ya.view(torch.int32), yb.view(torch.int32))
            assert torch.equal(ia, ib)


@pytest.mark.parametrize("text, n_features, cols", [
    (b"1 qid:1 2147483646:1\n", 2147483646, (2147483645,)),                  # shift 1: F = 2^31 - 2
    (b"1 qid:1 0:3 2147483647:2\n", 2147483648, (0, 2147483647)),            # index INT32_MAX, zero-based: F = 2^31
])
def test_widest_rows_a_c_int_index_allows(text, n_features, cols):
    """The widest rows a C-int index allows: every element written (NaN fill), nothing outside the row."""
    dev = torch.device("cuda", 0)
    plan = LibSVMPlan(read_svm_to_device(io.BytesIO(text), dev))
    assert (plan.n_rows, plan.n_features) == (1, n_features)
    guard = 1 << 20
    buf = torch.full((n_features + 2 * guard,), float("nan"), device=dev)    # NaN guards either side of the row
    x = buf[guard:guard + n_features].view(1, n_features)
    y = torch.full((1,), float("nan"), device=dev)
    q = torch.zeros(1, dtype=torch.int64, device=dev)
    plan.write(x, y, q)
    assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + n_features:]).all()
    assert not torch.isnan(x).any()
    assert int((x != 0).sum()) == len(cols) and all(float(x[0, c]) != 0 for c in cols)
    assert float(y[0]) == 1.0 and int(q[0]) == 1
    del buf, x


def test_compressed_files_and_descriptors(tmp_path):
    """What load_svmlight_file reads besides plain files: GzipFile / BZ2File objects (their fileno is the compressed
    file's), .gz / .bz2 paths (decompressed by suffix) and file descriptors."""
    import bz2
    import gzip
    name = "hard_numerals"
    text = SMALL[name + ".text"].tobytes()
    (tmp_path / "t.txt.gz").write_bytes(gzip.compress(text))
    (tmp_path / "t.txt.bz2").write_bytes(bz2.compress(text))
    (tmp_path / "t.txt").write_bytes(text)
    sources = [str(tmp_path / "t.txt.gz"), tmp_path / "t.txt.bz2"]
    with gzip.open(tmp_path / "t.txt.gz", "rb") as gz, bz2.BZ2File(tmp_path / "t.txt.bz2", "rb") as bz:
        for src in sources + [gz, bz]:
            st = SlateStore.from_svm_file(src, device="cuda:0", parser="device")
            assert np.array_equal(st.docs_x.cpu().numpy().view(np.uint32), SMALL[name + ".docs_x"])
            assert np.array_equal(st.offsets_host, SMALL[name + ".offsets"])
    fd = os.open(tmp_path / "t.txt", os.O_RDONLY)
    try:
        st = SlateStore.from_svm_file(fd, device="cuda:0", parser="device")
        assert np.array_equal(st.docs_y.cpu().numpy().view(np.uint32), SMALL[name + ".docs_y"])
    finally:
        os.close(fd)
    with open(tmp_path / "t.txt", "rb") as fh:         # from the current position, as sklearn reads a stream
        first = fh.readline()
        st = SlateStore.from_svm_file(fh, device="cuda:0", parser="device")
        assert st.docs_x.shape[0] == SMALL[name + ".docs_x"].shape[0] - 1 and first


def test_large_file_crosses_the_pinned_buffers(tmp_path, monkeypatch):
    """Several pieces through the two pinned buffers (small pieces here) give the same bytes as one upload."""
    from allrank_b200 import data
    text = C.mslr_text(2000, seed=3)
    path = tmp_path / "m.txt"
    path.write_bytes(text)
    monkeypatch.setattr(data, "_READ_CHUNK", 4096 + 13)
    got = read_svm_to_device(str(path), "cuda:0").cpu().numpy().tobytes()
    with open(path, "rb") as fh:
        got_stream = read_svm_to_device(io.BytesIO(fh.read()), "cuda:0").cpu().numpy().tobytes()
    assert got == text and got_stream == text
