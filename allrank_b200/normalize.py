"""reproducibility/normalize_features.py on the device: LibSVM folds normalised per feature column from file bytes to
written files.  DESIGN.md section 13.

The script loads train.txt, test.txt and vali.txt with sklearn, and for every column of the train role optionally
negates it, takes log(v + 0.01) when every value of all three roles is >= 0, and standardises it with the train
role's np.mean and np.std; then it writes the roles to "{ds_path}_normalized" with dump_svmlight_file.  Here the
files are parsed into dense float64 device tensors (csrc/libsvm.cu, float64 pass 2), transformed in place
(csrc/normalize.cu) and written by writer.DeviceRows.  The statistics follow numpy's pairwise summation bit for bit.
The log is correctly rounded (csrc/log_cr.cuh), so the bytes do not depend on the platform; they are the script's
bytes wherever the host's np.log is correctly rounded on the column's values.

Two deliberate differences from the script: every refusal is raised before the output directory or a file is
created, and the log is correctly rounded.

    python -m allrank_b200.normalize --ds_path <fold> [--features_without_logarithm ...] [--features_negative ...]
"""
import argparse
import ctypes
import os

import numpy as np
import torch

from . import _lib
from .data import LibSVMPlan, read_svm_to_device
from .writer import DeviceRows, worst_row_bytes

c_p, c_i, c_i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
_lib.register("arb_norm_sign_flags", c_i, [c_p, c_i64, c_i64, c_i64, c_p, c_p, c_p])
_lib.register("arb_norm_transform_a", c_i, [c_p, c_i64, c_i64, c_i64, c_p, c_p, c_p, c_p])
_lib.register("arb_norm_column_stats", c_i, [c_p, c_i64, c_i64, c_p, c_i64, c_p, c_p, c_i64, c_p, c_p, c_p, c_p])
_lib.register("arb_norm_transform_b", c_i, [c_p, c_i64, c_i64, c_i64, c_p, c_p, c_p])
_lib.register("arb_log_cr", c_i, [c_p, c_i64, c_p, c_i, c_p, c_p])
_lib.register("arb_log_cr_host", c_i, [c_p, c_i64, c_p, c_i, c_p])
_lib.register("arb_pairwise_sum_host", c_i, [c_p, c_i64, c_i64, c_p])

# the script's defaults (MSLR-WEB30K's feature numbers, zero-based)
FEATURES_WITHOUT_LOGARITHM = [5, 6, 7, 8, 9, 15, 19, 57, 58, 62, 75, 79, 85, 95, 96, 97, 98, 99, 100, 101, 102, 103,
                              104, 121, 122, 127, 129, 130]
FEATURES_NEGATIVE = [110, 111, 112, 113, 114, 115, 116, 117, 118, 119, 120, 123, 124]
ROLES = ("train", "test", "vali")
PW_BLOCK = 128          # numpy's PW_BLOCKSIZE: the largest leaf of its pairwise summation


def unlogged_message(i):
    return "Some values of feature no. {} are still < 0 which is why the feature won't be normalized".format(i)


def _raise_undecided(status, where):
    bits = int(status[1])
    if bits != -1:
        value = np.array([bits], np.int64).view(np.float64)[0]
        raise _lib.ArbError("{}: the log's accurate phase could not round log({!r}) (bits {:#018x})".format(
            where, float(value), bits & (2 ** 64 - 1)))


def log_cr(x, force_accurate=False):
    """(log(x) correctly rounded, how many values took the accurate phase), computed by the device code for a CUDA
    tensor and by the same code on the CPU otherwise.  force_accurate sends every value to the accurate phase."""
    if isinstance(x, torch.Tensor) and x.is_cuda:
        v = x.detach().to(torch.float64).contiguous().reshape(-1)
        y = torch.empty_like(v)
        status = torch.tensor([0, -1], dtype=torch.int64, device=v.device)
        if v.numel():
            with torch.cuda.device(v.device):
                _lib.check(_lib.lib().arb_log_cr(_lib.ptr(v), v.numel(), _lib.ptr(y), int(bool(force_accurate)),
                                                 _lib.ptr(status), _lib.stream_ptr(v.device)), "arb_log_cr")
        status = status.tolist()
    else:
        v = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
        y = np.empty_like(v)
        st = np.array([0, -1], np.int64)
        _lib.check(_lib.lib().arb_log_cr_host(v.ctypes.data, v.size, y.ctypes.data, int(bool(force_accurate)),
                                              st.ctypes.data), "arb_log_cr_host")
        status = st.tolist()
    _raise_undecided(status, "arb_log_cr")
    return y, int(status[0])


def pairwise_sum_host(a):
    """np.add.reduce of a 1-D float64 array (any stride), by the summation the column statistics use."""
    a = np.asarray(a)
    if a.ndim != 1 or a.dtype != np.float64 or a.strides[0] % 8:
        raise ValueError("expected a 1-D float64 array")
    out = np.zeros(1, np.float64)
    _lib.check(_lib.lib().arb_pairwise_sum_host(a.ctypes.data if a.size else None, a.size, a.strides[0] // 8,
                                                out.ctypes.data), "arb_pairwise_sum_host")
    return out[0]


def pairwise_plan(n):
    """numpy's pairwise summation tree over n >= 1 elements: (leaf_start [leaves + 1], children [internal, 2],
    level_counts).  Leaves are numbered left to right from 0, internal nodes from the number of leaves on, level by
    level (a node's children are on lower levels); the last node is the root.  A split of n > 128 elements is at
    n // 2 rounded down to a multiple of 8."""
    starts, internal = [], []           # internal: (left ref, right ref, height); refs ("L" or "I", index)

    def rec(lo, m):
        if m <= PW_BLOCK:
            starts.append(lo)
            return ("L", len(starts) - 1), 0
        m2 = m // 2
        m2 -= m2 % 8
        left, hl = rec(lo, m2)
        right, hr = rec(lo + m2, m - m2)
        internal.append((left, right, 1 + max(hl, hr)))
        return ("I", len(internal) - 1), internal[-1][2]

    rec(0, int(n))
    n_leaves = len(starts)
    order = sorted(range(len(internal)), key=lambda k: internal[k][2])        # stable: by level
    number = {k: n_leaves + j for j, k in enumerate(order)}

    def ref(r):
        return r[1] if r[0] == "L" else number[r[1]]

    children = np.array([[ref(internal[k][0]), ref(internal[k][1])] for k in order], np.int64).reshape(-1, 2)
    heights = [internal[k][2] for k in order]
    level_counts = np.array([heights.count(h) for h in range(1, (max(heights) if heights else 0) + 1)], np.int64)
    return np.array(starts + [int(n)], np.int64), children, level_counts


def _check_roles(roles):
    dev = roles[0].device
    for t in roles:
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.dim() == 2
                and t.is_contiguous() and t.device == dev):
            raise _lib.ArbError("roles must be contiguous 2-D float64 CUDA tensors on one device")
    return dev


def _column_plan(roles, features_without_logarithm, features_negative):
    """(negate mask, log mask, unlogged columns, first column some role lacks or None) over the train role's
    columns.  A column is logged when it is not in features_without_logarithm and every (negated) value of every
    role is >= 0; `unlogged` lists the other columns outside features_without_logarithm, up to the first missing."""
    F = int(roles[0].shape[1])
    dev = roles[0].device
    fwl, fneg = set(int(i) for i in features_without_logarithm), set(int(i) for i in features_negative)
    negate = np.array([i in fneg for i in range(F)], np.uint8)
    short = min([int(t.shape[1]) for t in roles[1:]] + [F])
    neg_dev = torch.from_numpy(negate).to(dev)
    bad = np.zeros(F, bool)
    with torch.cuda.device(dev):
        flags = torch.empty(F, dtype=torch.int32, device=dev)
        for t in roles:
            cols = min(F, int(t.shape[1]))
            if t.shape[0] == 0:
                continue
            _lib.check(_lib.lib().arb_norm_sign_flags(_lib.ptr(t), t.shape[0], t.shape[1], cols, _lib.ptr(neg_dev),
                                                      _lib.ptr(flags), _lib.stream_ptr(dev)), "arb_norm_sign_flags")
            bad[:cols] |= flags[:cols].cpu().numpy() != 0
    wants_log = np.array([i not in fwl for i in range(F)])
    log_mask = (wants_log & ~bad).astype(np.uint8)
    unlogged = [i for i in range(short) if wants_log[i] and bad[i]]
    return negate, log_mask, unlogged, (short if short < F else None)


def _index_error(roles, i):
    size = min(int(t.shape[1]) for t in roles[1:])
    return IndexError("index {} is out of bounds for axis 0 with size {}".format(i, size))


def _transform(roles, negate, log_mask):
    """Transform A on every role, the train role's statistics, then transform B on every role; (mean, std)."""
    train = roles[0]
    dev = train.device
    rows, F = int(train.shape[0]), int(train.shape[1])
    lib = _lib.lib()
    with torch.cuda.device(dev):
        st = _lib.stream_ptr(dev)
        neg_dev, log_dev = torch.from_numpy(negate).to(dev), torch.from_numpy(log_mask).to(dev)
        status = torch.tensor([0, -1], dtype=torch.int64, device=dev)
        for t in roles:
            if t.shape[0]:
                _lib.check(lib.arb_norm_transform_a(_lib.ptr(t), t.shape[0], t.shape[1], F, _lib.ptr(neg_dev),
                                                    _lib.ptr(log_dev), _lib.ptr(status), st), "arb_norm_transform_a")
        _raise_undecided(status.tolist(), "arb_norm_transform_a")
        mean = torch.full((F,), float("nan"), dtype=torch.float64, device=dev)      # np.mean of no rows: nan
        std = torch.full((F,), float("nan"), dtype=torch.float64, device=dev)
        if rows:
            leaf_start, children, level_counts = pairwise_plan(rows)
            n_nodes = len(leaf_start) - 1 + children.shape[0]
            scratch = torch.empty((n_nodes, F), dtype=torch.float64, device=dev)
            ls_dev = torch.from_numpy(leaf_start).to(dev)
            ch_dev = torch.from_numpy(children.reshape(-1)).to(dev) if children.size else None
            _lib.check(lib.arb_norm_column_stats(_lib.ptr(train), rows, F, _lib.ptr(ls_dev), len(leaf_start) - 1,
                                                 _lib.ptr(ch_dev), level_counts.ctypes.data, level_counts.size,
                                                 _lib.ptr(scratch), _lib.ptr(mean), _lib.ptr(std), st),
                       "arb_norm_column_stats")
            del scratch
        for t in roles:
            if t.shape[0]:
                _lib.check(lib.arb_norm_transform_b(_lib.ptr(t), t.shape[0], t.shape[1], F, _lib.ptr(mean),
                                                    _lib.ptr(std), st), "arb_norm_transform_b")
    return mean, std


def normalize_roles(train, others, features_without_logarithm=FEATURES_WITHOUT_LOGARITHM,
                    features_negative=FEATURES_NEGATIVE):
    """The script's column loop on dense float64 CUDA tensors [rows, F], in place: train and every tensor in
    `others` (test and vali).  Returns (log mask [F_train] bool, mean and std [F_train] float64 CUDA tensors, the
    columns outside features_without_logarithm left unlogged because a value is < 0 or NaN).  Columns of `others` at
    or beyond F_train become 0; a role narrower than train raises IndexError, as the script does."""
    roles = [train] + list(others)
    _check_roles(roles)
    negate, log_mask, unlogged, short = _column_plan(roles, features_without_logarithm, features_negative)
    if short is not None:
        raise _index_error(roles, short)
    mean, std = _transform(roles, negate, log_mask)
    return log_mask.astype(bool), mean, std, unlogged


def _load_role(path, device):
    """(X [rows, F] float64, y [rows] float64, qids [rows] int64, rows without a qid) on the device: what
    load_svmlight_file(path, query_id=True) and X.toarray() give.  Raises what they raise."""
    text = read_svm_to_device(path, device)
    plan = LibSVMPlan(text, require_qids=False)
    rows, F = plan.n_rows, plan.n_features
    need = rows * (8 * F + 16)
    free = torch.cuda.mem_get_info(device)[0]
    if need > free:
        raise _lib.ArbError("{}: the dense float64 role ({} rows x {} features) does not fit the free device memory "
                            "({} bytes)".format(path, rows, F, free))
    x = torch.empty((rows, F), dtype=torch.float64, device=device)
    y = torch.empty((rows,), dtype=torch.float64, device=device)
    q = torch.empty((rows,), dtype=torch.int64, device=device)
    plan.write(x, y, q)
    return x, y, q, plan.rows_without_qid


def normalize_features(ds_path, features_without_logarithm=FEATURES_WITHOUT_LOGARITHM,
                       features_negative=FEATURES_NEGATIVE, device=None):
    """reproducibility/normalize_features.py --ds_path ds_path on the device: writes "{ds_path}_normalized/"
    {train,test,vali}.txt and prints the script's lines in the script's order.  Returns the output directory.
    Raises what the script raises first (FileNotFoundError, the parser's ValueError / OverflowError, IndexError for a
    role narrower than train, ValueError for NaN or inf, an empty role or rows without a qid), always before the
    directory or any file is created; ArbError when the roles do not fit the device."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise _lib.ArbError("normalize_features needs a CUDA device (allrank_b200 has no CPU fallback)")
    loaded = [_load_role(os.path.join(ds_path, "{}.txt".format(role)), device) for role in ROLES]
    roles = [x for x, _, _, _ in loaded]
    negate, log_mask, unlogged, short = _column_plan(roles, features_without_logarithm, features_negative)
    for i in unlogged:
        print(unlogged_message(i))
    if short is not None:
        raise _index_error(roles, short)
    _transform(roles, negate, log_mask)
    out = []
    for role, (x, y, q, no_qid) in zip(ROLES, loaded):
        if no_qid and x.shape[0]:
            raise ValueError("expected query_id of shape (n_samples,), got ({},)".format(x.shape[0] - no_qid))
        out.append(DeviceRows(x, y, zero_based=True, query_id=q, device=device))
    text_bytes = max(r.chunk_rows() * worst_row_bytes(r.n_features, r.one_based) for r in out)
    free = torch.cuda.mem_get_info(device)[0]
    if text_bytes > free:
        raise _lib.ArbError("the text buffer ({} bytes) does not fit the free device memory ({} bytes)".format(
            text_bytes, free))
    out_dir = "{}_normalized".format(ds_path)
    os.makedirs(out_dir, exist_ok=True)
    for role, rows in zip(ROLES, out):
        with open(os.path.join(out_dir, "{}.txt".format(role)), "wb") as f:
            rows.write_to(f)
    print("Dataset with normalized features saved here: {}.".format(out_dir))
    return out_dir


def parser():
    """The script's command line."""
    p = argparse.ArgumentParser("Normalize features script")
    p.add_argument("--ds_path", help="location of the dataset", required=True, type=str)
    p.add_argument("--features_without_logarithm",
                   help="indices of features which are to be normalized without being logarithmized", required=False,
                   type=int, nargs="*", default=FEATURES_WITHOUT_LOGARITHM)
    p.add_argument("--features_negative",
                   help="indices of features which are to be normalized with logarithm but their values can be "
                        "negative", required=False, type=int, nargs="*", default=FEATURES_NEGATIVE)
    return p


def main(argv=None):
    args = parser().parse_args(argv)
    normalize_features(args.ds_path, args.features_without_logarithm, args.features_negative)


if __name__ == "__main__":
    main()


__all__ = ["normalize_features", "normalize_roles", "log_cr", "pairwise_sum_host", "pairwise_plan", "parser", "main",
           "FEATURES_WITHOUT_LOGARITHM", "FEATURES_NEGATIVE", "unlogged_message"]
