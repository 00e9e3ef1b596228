"""LibSVM files written on the device: the bytes of sklearn.datasets.dump_svmlight_file, and allRank's
write_to_libsvm_without_masked (allrank/data/dataset_saving.py:9-32) on top of it.  DESIGN.md section 12.

sklearn formats every non-zero value with Python's "%d:%.16g" in a Cython loop, one row at a time.  Here X goes to
the device once (host arrays through two pinned buffers), CUDA kernels (csrc/libsvm_write.cu) turn chunks of rows into
text in a device buffer sized for the chunk's worst case, and the text comes down through two pinned buffers in turn:
each chunk's copy is queued before the previous chunk is written to the file.
"""
import ctypes
import os

import numpy as np
import torch

from . import _lib
from .data import PADDED_Y_VALUE

c_p, c_i, c_i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
_lib.register("arb_svm_write_check", c_i, [c_p, c_i, c_i64, c_p, c_i, c_i64, c_p, c_p])
_lib.register("arb_svm_write_chunk", c_i, [c_p, c_i, c_i64, c_p, c_i, c_p, c_i, c_i64, c_i64, c_p, c_p, c_p])
_lib.register("arb_format_g16", c_i, [c_p, c_i64, c_p, c_p])
_lib.register("arb_format_g16_host", c_i, [c_p, c_i64, c_p])

# include/allrank_b200.h ARB_SVMW_*
_F32, _F64, _I64 = 0, 1, 2
_TEXT_CHUNK = 64 << 20      # bytes of the device text buffer and of each pinned download buffer
_UPLOAD_CHUNK = 64 << 20    # bytes of each pinned upload buffer
FMT_SLOT = 24               # bytes of one arb_format_g16 slot


def worst_row_bytes(n_features, one_based):
    """The longest line a row of n_features values can give: 24 bytes for the label, 25 for " qid:Q", per value a
    space, the index, ':' and 24 bytes, then the trailing space and the newline."""
    return 24 + 25 + n_features * (2 + len(str(n_features - 1 + one_based)) + 24) + 2


def _host(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _is_sparse(a):
    return hasattr(a, "toarray") or (isinstance(a, torch.Tensor) and a.layout != torch.strided)


def _x_kind(dtype):
    """ARB_SVMW_* for an X dtype (numpy or torch) and the dtype it is uploaded as; TypeError where sklearn's dense
    row loop has no signature for it (unsigned, bool, float16)."""
    np_dtype = np.dtype(dtype) if not isinstance(dtype, torch.dtype) else torch.empty(0, dtype=dtype).numpy().dtype
    if np_dtype == np.float32:
        return _F32, torch.float32
    if np_dtype == np.float64:
        return _F64, torch.float64
    if np_dtype.kind == "i":
        return _I64, torch.int64
    raise TypeError("dump_svmlight_file has no row loop for X of dtype {}".format(np_dtype))


def format_g16(values):
    """Python's "%.16g" % v of each double, formatted by the device code (arb_format_g16) when `values` is a CUDA
    tensor and by the same code on the CPU otherwise; a list of bytes."""
    if isinstance(values, torch.Tensor) and values.is_cuda:
        v = values.detach().to(torch.float64).contiguous().reshape(-1)
        n = int(v.numel())
        if n == 0:
            return []
        slots = torch.empty(n * FMT_SLOT, dtype=torch.uint8, device=v.device)
        with torch.cuda.device(v.device):
            _lib.check(_lib.lib().arb_format_g16(_lib.ptr(v), n, _lib.ptr(slots), _lib.stream_ptr(v.device)),
                       "arb_format_g16")
        raw = slots.cpu().numpy()
    else:
        v = np.ascontiguousarray(_host(values), dtype=np.float64).reshape(-1)
        n = int(v.size)
        raw = np.zeros(max(n, 1) * FMT_SLOT, np.uint8)
        _lib.check(_lib.lib().arb_format_g16_host(v.ctypes.data, n, raw.ctypes.data), "arb_format_g16_host")
    return raw[:n * FMT_SLOT].view("S24").tolist()


class DeviceRows:
    """X, y and the qids of a dump_svmlight_file call, checked as sklearn checks them and resident on one device."""

    def __init__(self, X, y, zero_based=True, query_id=None, device=None):
        if _is_sparse(X) or _is_sparse(y):
            raise NotImplementedError("the device writer takes dense X and y only")
        yh = _host(y)
        if yh.ndim != 1:
            raise ValueError("expected y of shape (n_samples,), got {!r}".format(yh.shape))
        if yh.dtype.kind == "i":
            self.y_kind, yh = _I64, yh.astype(np.int64)
        elif yh.dtype.kind in "fub":
            self.y_kind, yh = _F64, yh.astype(np.float64)
        else:
            raise TypeError("y of dtype {} is not numeric".format(yh.dtype))
        xh = None if isinstance(X, torch.Tensor) and X.is_cuda else _host(X)
        shape = tuple(X.shape) if xh is None else xh.shape
        if len(shape) != 2:
            raise ValueError("Expected 2D array, got an array of shape {!r} instead".format(shape))
        self.n_rows, self.n_features = int(shape[0]), int(shape[1])
        if yh.shape[0] == 0 or self.n_rows == 0:
            raise ValueError("Found array with 0 sample(s) while a minimum of 1 is required.")
        if self.n_features == 0:
            raise ValueError("Found array with 0 feature(s) while a minimum of 1 is required.")
        if self.n_rows != yh.shape[0]:
            raise ValueError("X.shape[0] and y.shape[0] should be the same, got {} and {} instead.".format(
                self.n_rows, yh.shape[0]))
        self.qid = None
        if query_id is not None:
            qh = _host(query_id)
            if qh.ndim != 1 or qh.shape[0] != self.n_rows:
                raise ValueError("expected query_id of shape (n_samples,), got {!r}".format(qh.shape))
            if qh.dtype.kind != "i":
                raise TypeError("query_id of dtype {} is not a signed integer".format(qh.dtype))
        self.x_kind, x_dtype = _x_kind(X.dtype if xh is None else xh.dtype)
        if xh is None:
            device = X.device
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.type != "cuda":
            raise _lib.ArbError("the device writer needs a CUDA device (allrank_b200 has no CPU fallback)")
        self.device = device
        if query_id is not None:
            self.qid = torch.from_numpy(np.ascontiguousarray(qh, dtype=np.int64)).to(device)
        self.one_based = int(not zero_based)
        self.y = torch.from_numpy(np.ascontiguousarray(yh)).to(device)
        self.X = X.to(x_dtype).contiguous() if xh is None else self._upload(xh, x_dtype)
        bad = torch.empty(1, dtype=torch.int32, device=device)
        with torch.cuda.device(device):
            _lib.check(_lib.lib().arb_svm_write_check(_lib.ptr(self.X), self.x_kind, self.X.numel(), _lib.ptr(self.y),
                                                      self.y_kind, self.n_rows, _lib.ptr(bad),
                                                      _lib.stream_ptr(device)), "arb_svm_write_check")
        if int(bad.item()):
            raise ValueError("Input contains NaN or infinity.")

    def _upload(self, xh, dtype):
        """Rows of the host array through two pinned buffers in turn, each piece's copy queued before the next is
        staged."""
        out = torch.empty((self.n_rows, self.n_features), dtype=dtype, device=self.device)
        row_bytes = self.n_features * out.element_size()
        step = max(1, min(self.n_rows, _UPLOAD_CHUNK // row_bytes))
        ring = [torch.empty((step, self.n_features), dtype=dtype, pin_memory=True) for _ in range(2)]
        done = [None, None]
        stream = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            for k, r0 in enumerate(range(0, self.n_rows, step)):
                r1, slot = min(self.n_rows, r0 + step), k % 2
                if done[slot] is not None:
                    done[slot].synchronize()
                np.copyto(ring[slot].numpy()[:r1 - r0], xh[r0:r1], casting="unsafe")
                out[r0:r1].copy_(ring[slot][:r1 - r0], non_blocking=True)
                done[slot] = torch.cuda.Event()
                done[slot].record(stream)
            stream.synchronize()
        return out

    def chunk_rows(self):
        return max(1, min(self.n_rows, _TEXT_CHUNK // worst_row_bytes(self.n_features, self.one_based)))

    def chunks(self):
        """Formats chunk after chunk of rows into one device buffer; yields (the buffer, the chunk's byte count)
        after each chunk's kernels are queued.  One 8-byte read per chunk: its byte total."""
        step = self.chunk_rows()
        text = torch.empty(step * worst_row_bytes(self.n_features, self.one_based), dtype=torch.uint8,
                           device=self.device)
        offsets = torch.empty(step + 1, dtype=torch.int64, device=self.device)
        lib = _lib.lib()
        with torch.cuda.device(self.device):
            st = _lib.stream_ptr(self.device)
            args = (_lib.ptr(self.X), self.x_kind, self.n_features, _lib.ptr(self.y), self.y_kind,
                    _lib.ptr(self.qid), self.one_based)
            for r0 in range(0, self.n_rows, step):
                r1 = min(self.n_rows, r0 + step)
                _lib.check(lib.arb_svm_write_chunk(*args, r0, r1, _lib.ptr(offsets), None, st), "arb_svm_write_chunk")
                total = int(offsets[r1 - r0].item())
                _lib.check(lib.arb_svm_write_chunk(*args, r0, r1, _lib.ptr(offsets), _lib.ptr(text), st),
                           "arb_svm_write_chunk")
                yield text, total

    def write_to(self, out):
        """Writes every chunk to the binary file object `out`: each chunk's download goes into one of two pinned
        buffers, queued before the previous chunk is written."""
        cap = self.chunk_rows() * worst_row_bytes(self.n_features, self.one_based)
        ring = [torch.empty(cap, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        stream = torch.cuda.current_stream(self.device)
        pending = None
        for k, (text, total) in enumerate(self.chunks()):
            slot = k % 2
            ring[slot][:total].copy_(text[:total], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(stream)
            if pending is not None:
                self._write_slot(out, ring, *pending)
            pending = (slot, total, ev)
        if pending is not None:
            self._write_slot(out, ring, *pending)

    @staticmethod
    def _write_slot(out, ring, slot, total, ev):
        ev.synchronize()
        out.write(memoryview(ring[slot].numpy())[:total])


def write_svm_file(X, y, f, zero_based=True, query_id=None, comment=None, multilabel=False):
    """sklearn.datasets.dump_svmlight_file(X, y, f, zero_based=zero_based, query_id=query_id), byte for byte, with
    the text formatted on the device.  X: a dense [rows, F] float32, float64 or signed-integer array or tensor (CUDA
    tensors stay where they are); y: 1-D; f: a path or a binary file object.  Refuses what sklearn refuses with the
    same exception types (ValueError for NaN or inf, empty or mismatched inputs) before the file is created or
    truncated; sparse inputs, `multilabel` and `comment` raise NotImplementedError."""
    if multilabel:
        raise NotImplementedError("the device writer does not write multilabel files")
    if comment is not None:
        raise NotImplementedError("the device writer does not write comments (sklearn's header names its version)")
    rows = DeviceRows(X, y, zero_based=zero_based, query_id=query_id)
    if hasattr(f, "write"):
        rows.write_to(f)
        return
    with open(os.fspath(f), "wb") as out:
        rows.write_to(out)


def write_to_libsvm_without_masked(path, X, y):
    """allrank/data/dataset_saving.py:9-32: the slates' rows whose label is not PADDED_Y_VALUE, with the slate's
    ordinal as qid (counted over every slate, including slates left empty), written by `write_svm_file`.  Slates
    held as CUDA tensors are masked and stacked on their device."""
    Xs, ys, qids = [], [], []
    for qid, (xs, yq) in enumerate(zip(X, y)):
        yh = _host(yq)
        mask = yh != PADDED_Y_VALUE
        if isinstance(xs, torch.Tensor) and xs.is_cuda:
            Xs.append(xs[torch.from_numpy(np.asarray(mask)).to(xs.device)])
        else:
            Xs.append(_host(xs)[mask])
        ys.append(yh[mask])
        qids.append(np.repeat(qid, int(np.count_nonzero(mask))))
    if Xs and all(isinstance(x, torch.Tensor) for x in Xs):
        Xs = torch.cat(Xs)
    else:
        Xs = np.vstack([_host(x) for x in Xs])
    write_svm_file(Xs, np.concatenate(ys), path, query_id=np.concatenate(qids))


__all__ = ["write_svm_file", "write_to_libsvm_without_masked", "DeviceRows", "format_g16", "worst_row_bytes"]
