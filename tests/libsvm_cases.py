"""LibSVM texts for the device parser's tests, each generated from a seed (tools/make_golden_libsvm.py stores what
sklearn's load_svmlight_file + SlateStore make of them under tests/golden/libsvm_*.npz).

This module stays with the tests on purpose: tools/make_golden_libsvm.py and tools/bench_libsvm.py import it, so the
fixtures, the GPU tests and the benchmark all parse the very same generated text."""
import numpy as np

# numerals where decimal -> float64 -> float32 is hard: halfway points, extremes, spellings
HARD_NUMERALS = [
    "1e23", "2.2250738585072011e-308", "2.2250738585072014e-308", "1e-400", "1e400", "-1e400", "-0", "0", ".5", "5.",
    "1E5", "+3", "-3.", "4.9406564584124654e-324", "2.4703282292062327e-324", "2.4703282292062328e-324",
    "1.7976931348623157e308", "1.7976931348623158e308", "1.797693134862315807937289714053e308", "9007199254740993",
    "9007199254740992.5", "0.1", "123456789012345678901234567890", "1_0", "1_000.000_1e1_0", "inf", "-Infinity",
    "nan", "-nan", "NaN", "0e99999999999999999999", "1e-342", "1e-343",
    # float32 halfway points: rn32(rn64(s)) != rn32(s)
    "1.00000005960464477550", "1.000000059604644776", "16777217.000000001", "0.30000001192092895508",
    "3.4028235677973366e38", "3.4028235677973367e38", "1.4012984643248170e-45", "7.0064923216240854e-46",
    "7.00649232162408536e-46",
    # 17 to 40 significant digits around double halfway points
    "9007199254740993.0000000000000000001", "0.500000000000000166533453693773481063544750213623046875",
    "1.0000000000000001110223024625156540423631668090820312500000000001",
    "2.2250738585072012595738e-308", "8.98846567431157953864652595394512366e307",
]


def hard_numerals(seed=0, n=400):
    """HARD_NUMERALS plus n decimal expansions (17 to 40 digits) of random double halfway points, and the
    expansions one digit above and below them."""
    import decimal
    from fractions import Fraction
    rng = np.random.default_rng(seed)
    out = list(HARD_NUMERALS)
    for _ in range(n):
        b = int(rng.integers(0, 0x7fefffffffffffff, dtype=np.uint64))
        lo = Fraction(float(np.uint64(b).view(np.float64)))
        hi = Fraction(float(np.uint64(b + 1).view(np.float64)))
        mid = (lo + hi) / 2
        decimal.getcontext().prec = int(rng.integers(17, 41))
        d = decimal.Decimal(mid.numerator) / decimal.Decimal(mid.denominator)
        out.append(str(d))
        out.append(str(d.next_plus()))
        out.append(str(d.next_minus()))
    return out


def hard_text(seed=0):
    """Rows of three features each, every value from hard_numerals(), labels with decimals."""
    vals = hard_numerals(seed)
    lines = []
    for r in range(0, len(vals), 3):
        feats = " ".join("{}:{}".format(j + 1, v) for j, v in enumerate(vals[r:r + 3]))
        lines.append("{} qid:{} {}".format(vals[r], r // 30, feats))
    return ("\n".join(lines) + "\n").encode()


# layout edge cases: comments, blank lines, tabs, \r\n, no final newline, one row, zero-/one-based, empty rows,
# qids that are not contiguous, labels with decimals
LAYOUT_CASES = {
    "comments": b"# header\n2 qid:1 1:0.5 3:2 # trailing\n\n   \n#\n1 qid:1 2:1.25\n0 qid:2 1:3 #x 4:5\n",
    "tabs_crlf": b"1\tqid:3\t1:1.5\t2:2\r\n0 qid:3 \t 2:7\r\n2 qid:4 1:-1\r\n",
    "no_final_newline": b"1 qid:1 1:1 2:2\n0 qid:1 1:3",
    "one_row": b"3.5 qid:9 4:1e-3",
    "zero_based": b"1 qid:1 0:1 2:2\n0 qid:2 1:3\n",
    "one_based": b"1 qid:1 1:1 3:2\n0 qid:2 2:3\n",
    "no_features": b"1 qid:1\n2 qid:1 5:2\n0 qid:2\n",
    "all_rows_empty": b"1 qid:1\n0 qid:2\n",
    "non_contiguous_qids": b"1 qid:5 1:1\n0 qid:7 1:2\n2 qid:5 1:3\n1 qid:7 1:4\n0 qid:5 1:5\n3 qid:1 1:6\n",
    "decimal_labels": b"0.5 qid:1 1:1\n-1.25 qid:1 1:2\n1e1 qid:2 1:3\n-0 qid:2 1:4\n+.75 qid:2 1:5\n",
    "whitespace_kinds": b"1 qid:1 1:1\x0b2:2\x0c3:3  \n",
    "qid_prefix": b"1 qidx:7 1:1\n0 qid:+8 1:2\n2 qid:0_9 1:3\n",
    "signed_indices": b"1 qid:1 +1:1 1_0:2\n",
    "only_comments": b"# nothing\n\n#\n",
    "nul_in_comment": b"1 qid:1 1:2 #\x00\n",
    # a NUL before the '#': sklearn's strchr stops at the NUL and does not cut the line, so '#:5' is part of the qid
    # token ("qid\x00#:5" starts with "qid": qid 5)
    "nul_before_hash": b"1 qid\x00#:5 1:2\n0 qid:5 1:3 # c\n",
}

# inputs sklearn + SlateStore refuse, and the exception type
REFUSED_CASES = {
    "not_sorted": (b"1 qid:1 2:1 1:2\n", ValueError),
    "duplicate": (b"1 qid:1 2:1 2:2\n", ValueError),
    "bad_value": (b"1 qid:1 1:abc\n", ValueError),
    "bad_label": (b"x qid:1 1:1\n", ValueError),
    "no_qid": (b"1 1:1\n0 1:2\n", ValueError),
    "some_without_qid": (b"1 qid:1 1:1\n0 1:2\n", ValueError),
    "no_colon": (b"1 qid:1 5\n", ValueError),
    "negative_index": (b"1 qid:1 -1:2\n", ValueError),
    "index_overflow": (b"1 qid:1 99999999999:2\n", OverflowError),
    "qid_overflow": (b"1 qid:99999999999999999999 1:2\n", OverflowError),
    "qid_without_colon": (b"1 qid 1:2\n", ValueError),
    "second_qid": (b"1 qid:1 qid:2 1:2\n", ValueError),
    "double_underscore": (b"1 qid:1 1:1__0\n", ValueError),
    "value_with_colon": (b"1 qid:1 1:2:3\n", ValueError),
    "nul_byte": (b"1 qid:1 1:2\n\x00\n", ValueError),
    "hex_value": (b"1 qid:1 1:0x10\n", ValueError),
    "nan_payload": (b"1 qid:1 1:nan(1)\n", ValueError),
    "late_error": (b"1 qid:1 1:1\n" * 50 + b"1 qid:1 3:1 2:2\n", ValueError),
    "nul_then_comment": (b"1 qid:1 1:2 \x00# 3:1\n", ValueError),
}

_POOL = ["0", "1", "2", "3", "4", "0.5", "0.25", "12", "127", "0.333333", "0.666667", "1.5", "-2.75", "42.125",
         "0.0001", "1e-05", "3.14159", "100", "255", "65535", "0.999999", "17.4", "-0", "6e3", "2.5E-2"]


def mslr_text(n_rows, seed=0, n_features=136):
    """An MSLR-WEB30K-shaped file: labels 0-4, qids in runs of 1 to 240 rows, 136 features of which ~3% are absent,
    values from a pool of MSLR-like numerals mixed with random decimals and the hard numerals."""
    rng = np.random.default_rng(seed)
    extra = ["{:.6f}".format(v) for v in rng.random(2000) * 1000] + ["{:.17g}".format(v) for v in
                                                                        rng.standard_normal(2000)] + HARD_NUMERALS[:20]
    pool = np.array(_POOL + extra, dtype=object)
    tok = [[("{}:{}".format(j + 1, v)) for v in pool] for j in range(n_features)]
    choice = rng.integers(0, len(_POOL), (n_rows, n_features))
    rare = rng.random((n_rows, n_features)) < 0.05
    choice[rare] = rng.integers(len(_POOL), len(pool), int(rare.sum()))
    present = rng.random((n_rows, n_features)) >= 0.03
    labels = rng.integers(0, 5, n_rows)
    qids, q, left = np.empty(n_rows, np.int64), 0, 0
    for r in range(n_rows):
        if left == 0:
            q += int(rng.integers(1, 50))
            left = int(rng.integers(1, 241))
        qids[r] = q
        left -= 1
    lines = []
    for r in range(n_rows):
        c, p = choice[r].tolist(), present[r].tolist()
        lines.append("{} qid:{} {}".format(labels[r], qids[r], " ".join(tok[j][c[j]] for j in range(n_features)
                                                                         if p[j])))
    return ("\n".join(lines) + "\n").encode()


def reference_arrays(text):
    """What sklearn's load_svmlight_file + SlateStore store for `text` (host side of SlateStore.__init__)."""
    import io
    from sklearn.datasets import load_svmlight_file
    from allrank_b200.data import group_offsets
    X, y, q = load_svmlight_file(io.BytesIO(text), query_id=True)
    X = np.ascontiguousarray(np.asarray(X.toarray(), dtype=np.float32))
    y = np.ascontiguousarray(np.asarray(y, dtype=np.float32))
    offsets = group_offsets(q)
    if offsets[-1] != X.shape[0]:
        raise ValueError("X, y and query_ids must have one row per document")
    lengths = np.diff(offsets)
    return {"docs_x": X, "docs_y": y, "offsets": offsets, "n_features": X.shape[1],
            "longest_query_length": int(lengths.max()) if len(lengths) else 0}
