"""Device-side replacement for allRank's slate pipeline (allrank/data/dataset_loading.py).

The reference keeps the corpus as per-query numpy arrays and builds every slate in Python
(`LibSVMDataset.__getitem__` -> `FixLength` -> `ToTensor`, then DataLoader collation; dataset_loading.py:32-165,
:230-247).  Here the corpus is uploaded once and stays in HBM as query-grouped rows with CSR offsets (MSLR-WEB30K's
train fold is 2.27 M x 136 fp32 = 1.2 GB of the 180 GB), and one kernel launch (csrc/slates.cu,
`arb_assemble_slates`) builds a whole `(x, y, indices)` batch: padding is bit-identical to the reference, sampling
follows the same rules with a counter-hash stream instead of numpy's.

Same call surface as the reference module:

    train_ds, val_ds = load_libsvm_dataset(input_path, slate_length, validation_ds_role)    # :206-217
    n_features = train_ds.shape[-1]                                                         # main.py:63
    train_dl, val_dl = create_data_loaders(train_ds, val_ds, num_workers, batch_size)       # :230-247
    for xb, yb, indices in train_dl: ...                                                    # train_utils.py:93-96

No CPU fallback: the loaders need a CUDA device.
"""
import bz2
import ctypes
import gzip
import io
import os
import stat

import numpy as np
import torch

from . import _lib

PADDED_Y_VALUE = -1        # dataset_loading.py:15
PADDED_INDEX_VALUE = -1    # dataset_loading.py:16

c_p, c_i = ctypes.c_void_p, ctypes.c_int32
_lib.register("arb_assemble_slates_smem_bytes", ctypes.c_size_t, [c_i, c_i])
_lib.register("arb_assemble_slates", c_i, [c_p, c_p, c_p, ctypes.c_int64, c_p, c_i, c_i, c_i, c_i, ctypes.c_uint64, c_p,
                                           c_p, c_p, c_p])
c_i64 = ctypes.c_int64
_lib.register("arb_libsvm_chunks", c_i64, [c_i64])
_lib.register("arb_libsvm_count_lines", c_i, [c_p, c_i64, c_p, c_p])
_lib.register("arb_libsvm_index_lines", c_i, [c_p, c_i64, c_p, c_p, c_p])
_lib.register("arb_libsvm_pass1", c_i, [c_p, c_i64, c_p, c_i64, c_i64, c_p, c_p, c_p, c_p])
_lib.register("arb_libsvm_pass2", c_i, [c_p, c_i64, c_p, c_i64, c_i64, c_p, c_p, c_i64, c_i, c_i64, c_p, c_p, c_p, c_p])
_lib.register("arb_libsvm_pass2_f64", c_i, [c_p, c_i64, c_p, c_i64, c_i64, c_p, c_p, c_i64, c_i, c_i64, c_p, c_p, c_p,
                                            c_p])
_lib.register("arb_libsvm_parse_numerals_host", c_i, [c_p, c_p, c_i64, c_i, c_p, c_p])

PARSERS = ("sklearn", "device")
_READ_CHUNK = 64 << 20      # bytes per pinned buffer; one buffer's upload overlaps the read into the other

# include/allrank_b200.h ARB_LIBSVM_E_*: the exception sklearn raises for the same line, and why
_LIBSVM_ERRORS = {
    1: (ValueError, "could not convert the label to float"),
    2: (ValueError, "invalid qid"),
    3: (OverflowError, "qid out of the int64 range"),
    4: (ValueError, "feature without ':'"),
    5: (ValueError, "invalid feature index"),
    6: (OverflowError, "feature index out of the C int range"),
    7: (ValueError, "Invalid index: negative"),
    8: (ValueError, "Feature indices in SVMlight/LibSVM data file should be sorted and unique"),
    9: (ValueError, "could not convert the feature value to float"),
    10: (ValueError, "numeral beyond the parser's exact range"),
}


def group_offsets(query_ids):
    """CSR offsets of the query groups exactly as LibSVMDataset splits them (dataset_loading.py:106-111): groups are
    taken in order of first appearance and are `count` consecutive rows long."""
    query_ids = np.asarray(query_ids)
    _, first, counts = np.unique(query_ids, return_index=True, return_counts=True)
    ordered = counts[np.argsort(first)]
    return np.concatenate([[0], np.cumsum(ordered)]).astype(np.int64)


class SlateStore:
    """Query-grouped corpus resident on one CUDA device; the counterpart of LibSVMDataset (dataset_loading.py:96-165)."""

    def __init__(self, X, y, query_ids, device=None, slate_length=None):
        if hasattr(X, "toarray"):
            X = X.toarray()                                   # :104 (the reference densifies too)
        X = np.ascontiguousarray(np.asarray(X, dtype=np.float32))
        y = np.ascontiguousarray(np.asarray(y, dtype=np.float32))
        offsets = group_offsets(query_ids)
        if offsets[-1] != X.shape[0] or y.shape[0] != X.shape[0]:
            raise ValueError("X, y and query_ids must have one row per document")
        self._init_from_groups(X, y, offsets, device, slate_length)

    def _init_from_groups(self, X, y, offsets, device, slate_length):
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.type != "cuda":
            raise _lib.ArbError("SlateStore needs a CUDA device (allrank_b200 has no CPU fallback)")
        self.device = device
        self.offsets_host = np.asarray(offsets, dtype=np.int64)
        lengths = np.diff(self.offsets_host)
        self.n_queries = int(lengths.shape[0])
        self.n_features = int(X.shape[1])
        self.longest_query_length = int(lengths.max()) if self.n_queries else 0     # :112
        self.docs_x = torch.as_tensor(X, device=device)      # (device tensors from the device parser stay put)
        self.docs_y = torch.as_tensor(y, device=device)
        self.offsets = torch.from_numpy(self.offsets_host).to(device)
        self.slate_length = slate_length

    @classmethod
    def from_groups(cls, X_by_qid, y_by_qid, device=None, slate_length=None):
        """From per-query arrays (e.g. an allrank LibSVMDataset's X_by_qid / y_by_qid)."""
        self = cls.__new__(cls)
        lengths = [len(v) for v in y_by_qid]
        offsets = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        X = np.ascontiguousarray(np.concatenate([np.asarray(v, dtype=np.float32) for v in X_by_qid], axis=0))
        y = np.ascontiguousarray(np.concatenate([np.asarray(v, dtype=np.float32) for v in y_by_qid], axis=0))
        self._init_from_groups(X, y, offsets, device, slate_length)
        return self

    @classmethod
    def from_svm_file(cls, svm_file_path, device=None, slate_length=None, parser="sklearn"):
        """dataset_loading.py:118-130 (file or file-like object).  parser="sklearn": the reference's parser on the
        host, then one upload.  parser="device": the file's bytes are uploaded and parsed by CUDA kernels
        (csrc/libsvm.cu) into the same arrays, bit for bit, refusing the same inputs with the same exception types."""
        if parser not in PARSERS:
            raise ValueError("parser must be one of {}, got {!r}".format(PARSERS, parser))
        if parser == "device":
            return cls.from_svm_bytes(read_svm_to_device(svm_file_path, device), device=device,
                                      slate_length=slate_length)
        from sklearn.datasets import load_svmlight_file
        x, y, query_ids = load_svmlight_file(svm_file_path, query_id=True)
        return cls(x, y, query_ids, device=device, slate_length=slate_length)

    @classmethod
    def from_svm_bytes(cls, text, device=None, slate_length=None):
        """From LibSVM text already in device memory (`read_svm_to_device`): the device parser's two passes."""
        plan = LibSVMPlan(text)
        docs_x = torch.empty((plan.n_rows, plan.n_features), dtype=torch.float32, device=text.device)
        docs_y = torch.empty((plan.n_rows,), dtype=torch.float32, device=text.device)
        qids = torch.empty((plan.n_rows,), dtype=torch.int64, device=text.device)
        plan.write(docs_x, docs_y, qids)
        self = cls.__new__(cls)
        self._init_from_groups(docs_x, docs_y, group_offsets(qids.cpu().numpy()), text.device, slate_length)
        return self

    def __len__(self):
        return self.n_queries

    @property
    def shape(self):
        """[queries, longest query, features] -- dataset_loading.py:149-165."""
        return [self.n_queries, self.longest_query_length, self.n_features]

    def assemble(self, queries, slate_length=None, seed=0):
        """One batch of slates for the given query numbers: (x [B,S,F] fp32, y [B,S] fp32, indices [B,S] int64)."""
        S = int(slate_length if slate_length is not None else self.slate_length)
        if S <= 0:
            raise ValueError("slate_length must be positive")
        queries = torch.as_tensor(queries, dtype=torch.int64)
        if queries.device.type == "cpu" and queries.numel() and (
                int(queries.min()) < 0 or int(queries.max()) >= self.n_queries):
            raise IndexError("query number out of range")     # (device tensors are range-checked by the kernel)
        queries = queries.to(self.device).contiguous()
        B, F = int(queries.numel()), self.n_features
        x = torch.empty((B, S, F), dtype=torch.float32, device=self.device)
        y = torch.empty((B, S), dtype=torch.float32, device=self.device)
        idx = torch.empty((B, S), dtype=torch.int64, device=self.device)
        if B == 0:
            return x, y, idx
        with torch.cuda.device(self.device):
            rc = _lib.lib().arb_assemble_slates(_lib.ptr(self.docs_x), _lib.ptr(self.docs_y), _lib.ptr(self.offsets),
                                                self.n_queries, _lib.ptr(queries), B, S, F,
                                                self.longest_query_length,
                                                ctypes.c_uint64(int(seed) & (2 ** 64 - 1)), _lib.ptr(x), _lib.ptr(y),
                                                _lib.ptr(idx), _lib.stream_ptr(self.device))
        _lib.check(rc, "arb_assemble_slates")
        return x, y, idx


def open_svm(svm_file):
    """(binary file object, whether the caller must close it) for what load_svmlight_file accepts: a file object
    (read from its current position), a file descriptor, or a path -- ".gz" and ".bz2" paths decompressed, as
    sklearn's _gen_open does."""
    if hasattr(svm_file, "read"):
        return svm_file, False
    if isinstance(svm_file, int):
        return open(svm_file, "rb", closefd=False), True
    path = os.fspath(svm_file)
    ext = os.path.splitext(path)[1]
    if ext == ".gz":
        return gzip.open(path, "rb"), True
    if ext == ".bz2":
        return bz2.BZ2File(path, "rb"), True
    return open(path, "rb"), True


def plain_file_size(f):
    """Bytes left in `f` when it reads a regular file without transformation (io.FileIO, or a BufferedReader over
    one), else None.  A GzipFile or BZ2File has the fileno of its compressed file, so fstat says nothing about it."""
    raw = f.raw if isinstance(f, io.BufferedReader) else f
    if not isinstance(raw, io.FileIO):
        return None
    st = os.fstat(raw.fileno())
    if not stat.S_ISREG(st.st_mode):
        return None
    return max(st.st_size - f.tell(), 0)


def read_svm_to_device(svm_file, device=None):
    """The bytes of a LibSVM file (anything `open_svm` takes) as a uint8 CUDA tensor.  A regular file is read straight
    into two pinned 64 MB buffers in turn, each piece's upload queued before the next read; any other stream (a
    compressed file, an in-memory buffer) is read whole first and uploaded through the same buffers."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise _lib.ArbError("the device parser needs a CUDA device (allrank_b200 has no CPU fallback)")
    f, own = open_svm(svm_file)
    try:
        size = plain_file_size(f)
        data = None
        if size is None:
            data = f.read()
            size = len(data)
        free = torch.cuda.mem_get_info(device)[0]
        if size > free:
            raise _lib.ArbError("the file ({} bytes) does not fit the free device memory ({} bytes)".format(size, free))
        text = torch.empty(size, dtype=torch.uint8, device=device)
        if size == 0:
            return text
        stream = torch.cuda.current_stream(device)
        piece = min(size, _READ_CHUNK)
        ring = [torch.empty(piece, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        uploaded = [None, None]           # the event after each buffer's last upload
        off, k = 0, 0
        while off < size:
            slot = k % 2
            if uploaded[slot] is not None:
                uploaded[slot].synchronize()
            host = ring[slot].numpy()
            want = min(piece, size - off)
            if data is None:
                got = f.readinto(memoryview(host)[:want])
                if not got:
                    break
            else:
                host[:want] = np.frombuffer(data, np.uint8, want, off)
                got = want
            text[off:off + got].copy_(ring[slot][:got], non_blocking=True)
            uploaded[slot] = torch.cuda.Event()
            uploaded[slot].record(stream)
            off, k = off + got, k + 1
        if off != size or (data is None and f.read(1)):
            raise OSError("the file changed while it was read ({} bytes expected)".format(size))
        stream.synchronize()
        return text
    finally:
        if own:
            f.close()


class LibSVMPlan:
    """Pass 1 of the device parser over LibSVM text in device memory (include/allrank_b200.h, arb_libsvm_*): the line
    index, validation and the output shape.  Raises what load_svmlight_file + SlateStore raise for the same text
    (ValueError / OverflowError naming the first failing line) before anything is written.  `write` is pass 2.
    require_qids=False keeps rows without a qid (load_svmlight_file accepts them; only their use fails) and counts
    them in `rows_without_qid`."""

    def __init__(self, text, require_qids=True):
        if not (isinstance(text, torch.Tensor) and text.is_cuda and text.dtype == torch.uint8 and text.dim() == 1
                and text.is_contiguous()):
            raise _lib.ArbError("LibSVM text must be a contiguous 1-D uint8 CUDA tensor")
        self.text = text
        self.n_bytes = n = int(text.numel())
        self.n_rows, self.n_features, self.shift = 0, 1, 0     # sklearn's shape for a file without rows: (0, 1)
        self.rows_without_qid = 0
        if n == 0:
            return
        lib, dev = _lib.lib(), text.device
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            chunks = int(lib.arb_libsvm_chunks(n))
            counts = torch.empty(chunks + 1, dtype=torch.int64, device=dev)
            _lib.check(lib.arb_libsvm_count_lines(_lib.ptr(text), n, _lib.ptr(counts), st), "arb_libsvm_count_lines")
            self.n_newlines = int(counts[chunks])
            self.n_lines = self.n_newlines + int(int(text[n - 1]) != 10)
            need = 8 * (max(self.n_newlines, 1) + 2 * self.n_lines + 8)
            free = torch.cuda.mem_get_info(dev)[0]
            if need > free:
                raise _lib.ArbError("the line index ({} lines) does not fit the free device memory ({} bytes)".format(
                    self.n_lines, free))
            self.line_end = torch.empty(max(self.n_newlines, 1), dtype=torch.int64, device=dev)
            _lib.check(lib.arb_libsvm_index_lines(_lib.ptr(text), n, _lib.ptr(counts), _lib.ptr(self.line_end), st),
                       "arb_libsvm_index_lines")
            del counts
            self.line_row = torch.empty(self.n_lines, dtype=torch.int64, device=dev)
            self.line_qid = torch.empty(self.n_lines, dtype=torch.int64, device=dev)
            summary = torch.empty(8, dtype=torch.int64, device=dev)
            _lib.check(lib.arb_libsvm_pass1(_lib.ptr(text), n, _lib.ptr(self.line_end), self.n_newlines, self.n_lines,
                                            _lib.ptr(self.line_row), _lib.ptr(self.line_qid), _lib.ptr(summary), st),
                       "arb_libsvm_pass1")
            err, lo, hi, rows, no_qid = (int(v) for v in summary[:5].tolist())
        if err != -1:
            exc, why = _LIBSVM_ERRORS[err & 0xFF]
            raise exc("LibSVM line {}: {}".format(err >> 8, why))
        self.rows_without_qid = no_qid
        if no_qid and require_qids:     # load_svmlight_file returns fewer qids than rows; SlateStore refuses that
            raise ValueError("X, y and query_ids must have one row per document "
                             "({} of {} rows have no qid)".format(no_qid, rows))
        self.n_rows = rows
        if hi >= 0:
            self.shift = int(lo > 0)
            self.n_features = hi - self.shift + 1
        need = rows * (4 * self.n_features + 12)     # (the float32 outputs; float64 callers check their own)
        free = torch.cuda.mem_get_info(text.device)[0]
        if need > free:
            raise _lib.ArbError("the dense output ({} rows x {} features) does not fit the free device memory "
                                "({} bytes)".format(rows, self.n_features, free))

    def write(self, docs_x, docs_y, qids):
        """Pass 2: every element of docs_x [n_rows, n_features], docs_y [n_rows] and qids [n_rows] int64.  docs_x and
        docs_y are both fp32 (what SlateStore keeps) or both float64 (load_svmlight_file's X.toarray() and y)."""
        dtype = torch.float64 if docs_x.dtype == torch.float64 else torch.float32
        shapes = ((docs_x, (self.n_rows, self.n_features), dtype), (docs_y, (self.n_rows,), dtype),
                  (qids, (self.n_rows,), torch.int64))
        for t, shape, want in shapes:
            if tuple(t.shape) != shape or t.dtype != want or t.device != self.text.device or not t.is_contiguous():
                raise ValueError("pass 2 outputs must be contiguous {} {} tensors on {}".format(
                    shape, want, self.text.device))
        if self.n_rows == 0:
            return
        name = "arb_libsvm_pass2_f64" if dtype == torch.float64 else "arb_libsvm_pass2"
        with torch.cuda.device(self.text.device):
            rc = getattr(_lib.lib(), name)(_lib.ptr(self.text), self.n_bytes, _lib.ptr(self.line_end),
                                           self.n_newlines, self.n_lines, _lib.ptr(self.line_row),
                                           _lib.ptr(self.line_qid), self.n_rows, self.shift, self.n_features,
                                           _lib.ptr(docs_x), _lib.ptr(docs_y), _lib.ptr(qids),
                                           _lib.stream_ptr(self.text.device))
        _lib.check(rc, name)


class DeviceSlateLoader:
    """Iterates (xb, yb, indices) batches like the reference's DataLoader over a LibSVMDataset (:242-245), built on
    the device.  Shuffling and the per-batch sampling seed come from torch's global CPU generator, so
    torch.manual_seed makes an epoch repeatable."""

    def __init__(self, store, batch_size, slate_length=None, shuffle=False):
        self.dataset = store
        self.batch_size = int(batch_size)
        self.slate_length = int(slate_length if slate_length is not None else store.slate_length)
        self.shuffle = bool(shuffle)
        if self.batch_size <= 0:
            raise ValueError("batch_size must be positive")

    def __len__(self):
        return (len(self.dataset) + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        n = len(self.dataset)
        order = torch.randperm(n) if self.shuffle else torch.arange(n)
        order = order.to(self.dataset.device)
        for start in range(0, n, self.batch_size):
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
            yield self.dataset.assemble(order[start:start + self.batch_size], self.slate_length, seed)


def load_libsvm_role(input_path, role, device=None, parser="sklearn"):
    """dataset_loading.py:168-182 (local files only: the gs:// path is the reference's I/O layer, out of scope).
    parser: "sklearn" (the reference's) or "device" (SlateStore.from_svm_file)."""
    path = os.path.join(input_path, "{}.txt".format(role))
    with open(path, "rb") as stream:
        return SlateStore.from_svm_file(stream, device=device, parser=parser)


def load_libsvm_dataset_role(role, input_path, slate_length, device=None, parser="sklearn"):
    """Train slates are fixed to `slate_length`, every other role to its longest query (:219-227)."""
    ds = load_libsvm_role(input_path, role, device=device, parser=parser)
    ds.slate_length = int(slate_length) if role == "train" else int(ds.longest_query_length)
    return ds


def load_libsvm_dataset(input_path, slate_length, validation_ds_role, device=None, parser="sklearn"):
    """dataset_loading.py:206-217."""
    train_ds = load_libsvm_dataset_role("train", input_path, slate_length, device=device, parser=parser)
    val_ds = load_libsvm_dataset_role(validation_ds_role, input_path, slate_length, device=device, parser=parser)
    return train_ds, val_ds


def _as_store(ds, device=None):
    if isinstance(ds, SlateStore):
        return ds
    # an allrank LibSVMDataset: per-query arrays + Compose([FixLength(dim_given), ToTensor()])
    slate_length = None
    transform = getattr(ds, "transform", None)
    for t in getattr(transform, "transforms", []) or []:
        if hasattr(t, "dim_given"):
            slate_length = int(t.dim_given)
    return SlateStore.from_groups(ds.X_by_qid, ds.y_by_qid, device=device, slate_length=slate_length)


def create_data_loaders(train_ds, val_ds, num_workers, batch_size, device=None):
    """dataset_loading.py:230-247.  Accepts SlateStores or the reference's LibSVMDataset objects (uploaded once).
    `num_workers` is accepted for signature parity and unused (there are no loader processes).  One process drives
    one GPU here, so `batch_size` is the per-process batch (the reference multiplies it by the visible GPU count for
    nn.DataParallel, :237-238)."""
    train_store, val_store = _as_store(train_ds, device), _as_store(val_ds, device)
    train_dl = DeviceSlateLoader(train_store, batch_size, shuffle=True)
    val_dl = DeviceSlateLoader(val_store, batch_size, shuffle=False)
    return train_dl, val_dl


__all__ = ["SlateStore", "DeviceSlateLoader", "LibSVMPlan", "open_svm", "plain_file_size", "read_svm_to_device",
           "group_offsets", "load_libsvm_role", "load_libsvm_dataset_role",
           "load_libsvm_dataset", "create_data_loaders", "PADDED_Y_VALUE", "PADDED_INDEX_VALUE"]
