"""The device LibSVM parser without a GPU: its numeral conversion (the same __host__ __device__ code the kernels run,
called through arb_libsvm_parse_numerals_host) against Python's float(), np.float32(float()), int() and np.int64()
over 10^6 random and adversarial numerals, and the refusals of the Python layer."""
import inspect

import numpy as np
import pytest
import torch

from allrank_b200 import _lib, data, integration

RNG_SEED = 20261017


def _convert(tokens, kind):
    lib = _lib.lib()
    text = b"".join(tokens)
    offsets = np.zeros(len(tokens) + 1, np.int64)
    offsets[1:] = np.cumsum([len(t) for t in tokens])
    buf = np.frombuffer(text, np.uint8) if text else np.zeros(1, np.uint8)
    out = np.zeros(len(tokens), np.uint64)
    status = np.zeros(len(tokens), np.int32)
    rc = lib.arb_libsvm_parse_numerals_host(buf.ctypes.data, offsets.ctypes.data, len(tokens), kind,
                                            out.ctypes.data, status.ctypes.data)
    assert rc == 0
    return out, status


def _halfway_numerals(rng, n):
    """Decimal expansions of double halfway points, cut to 17-40 significant digits, exactly and +- one unit."""
    out = []
    for b in rng.integers(0, 0x7fefffffffffffff, n, dtype=np.uint64).tolist():
        ex, fr = b >> 52, b & ((1 << 52) - 1)
        m, e = (fr | (1 << 52), ex - 1075) if ex else (fr, -1074)
        num, p2 = 2 * m + 1, e - 1                          # midpoint = num * 2^p2
        if p2 >= 0:
            digits, point = str(num << p2), 0
        else:
            digits, point = str(num * 5 ** -p2), -p2        # value = digits * 10^-point
        keep = int(rng.integers(17, 41))
        if len(digits) > keep:
            point -= len(digits) - keep
            digits = digits[:keep]
        delta = int(rng.integers(-1, 2))
        digits = str(max(int(digits) + delta, 1))
        out.append("{}e{}".format(digits, -point).encode())
    return out


def _numerals(n_total):
    rng = np.random.default_rng(RNG_SEED)
    toks = [s.encode() for s in (
        "1e23", "2.2250738585072011e-308", "1e-400", "1e400", "-0", ".5", "5.", "1E5", "+3", "inf", "-inf",
        "Infinity", "-INFINITY", "nan", "-nan", "NaN", "1_0", "1__0", "_1", "1_", "1_.5", "1._5", "1e1_0", "1e_1",
        "infinit", "nan(1)", "0x10", "1.5f", "1d5", ".", "e5", ".e5", "5.e", "1e", "1e+", "+.5", "-.5e-3", "",
        "+", "-", "++1", "1e+-1", "0e999999999999999999999", "1e-999999999999999999999", "4.9406564584124654e-324",
        "2.4703282292062327e-324", "2.4703282292062328e-324", "1.7976931348623157e308", "1.7976931348623158e308",
        "1.797693134862315807937289714053e308", "9007199254740993", "1" * 800, "0." + "0" * 400 + "1" * 900,
        "1" + "0" * 5000 + "e-5000", "1.00000005960464477550", "3.4028235677973366e38", "7.0064923216240854e-46")]
    n_rest = (n_total - len(toks)) // 5
    bits = rng.integers(0, 1 << 64, n_rest, dtype=np.uint64).view(np.float64)
    toks += [repr(float(v)).encode() for v in bits]
    vals = rng.standard_normal(n_rest) * 10.0 ** rng.integers(-300, 300, n_rest)
    prec = rng.integers(0, 40, n_rest)
    toks += [("%.*e" % (int(p), v)).encode() for p, v in zip(prec.tolist(), vals.tolist())]
    toks += _halfway_numerals(rng, n_rest)
    digits = rng.integers(0, 10, (n_rest, 24)).astype(np.uint8) + ord("0")
    lens = rng.integers(1, 25, n_rest)
    dots = rng.integers(0, 26, n_rest)
    exps = rng.integers(-400, 400, n_rest)
    for row, k, d, e in zip(digits, lens.tolist(), dots.tolist(), exps.tolist()):
        s = row[:k].tobytes()
        if d <= k:
            s = s[:d] + b"." + s[d:]
        toks.append(s + (b"e%d" % e if e % 3 else b""))
    alphabet = np.frombuffer(b"0123456789._eE+-nif", np.uint8)   # (tokens never hold whitespace)
    junk = rng.choice(alphabet, (n_total - len(toks), 8))
    junk_len = rng.integers(1, 9, len(junk))
    toks += [r[:k].tobytes() for r, k in zip(junk, junk_len.tolist())]
    return toks


def _py(fn, t):
    try:
        return 0, fn(t)
    except ValueError:
        return 1, None
    except OverflowError:
        return 2, None


def test_float_conversion_matches_python_bit_for_bit():
    toks = _numerals(1_000_000)
    assert len(toks) >= 1_000_000
    f64, st64 = _convert(toks, 0)
    f32, st32 = _convert(toks, 1)
    assert (st64 == st32).all()
    n_ok = 0
    for i, t in enumerate(toks):
        status, v = _py(float, t)
        assert st64[i] == status, (t[:80], st64[i], status)
        if status:
            continue
        n_ok += 1
        want64 = np.float64(v).view(np.uint64)
        with np.errstate(over="ignore"):
            want32 = np.float32(v).view(np.uint32)
        assert f64[i] == want64, (t[:80], hex(int(f64[i])), hex(int(want64)))
        assert f32[i] == want32, (t[:80], hex(int(f32[i])), hex(int(want32)))
    assert n_ok > 800_000


@pytest.mark.parametrize("kind, lo, hi, fn", [(2, -2 ** 31, 2 ** 31 - 1, int), (3, -2 ** 63, 2 ** 63 - 1, np.int64)])
def test_integer_conversion_matches_python(kind, lo, hi, fn):
    rng = np.random.default_rng(RNG_SEED + kind)
    toks = [b"0", b"+1", b"-1", b"007", b"1_0", b"1__0", b"_1", b"1_", b"", b"+", b"1.0", b"1e3", b"0x1",
            str(hi).encode(), str(hi + 1).encode(), str(lo).encode(), str(lo - 1).encode(), b"9" * 40, b"-" + b"9" * 40,
            b"1" * 4300, b"1" * 4301]
    toks += [str(int(v)).encode() for v in rng.integers(-2 ** 62, 2 ** 62, 20000)]
    toks += [bytes(rng.choice(np.frombuffer(b"0123456789_+-", np.uint8), int(rng.integers(1, 12))))
             for _ in range(20000)]
    out, st = _convert(toks, kind)
    for t, o, s in zip(toks, out.view(np.int64).tolist(), st.tolist()):
        status, v = _py(int, t)
        if status == 0 and not lo <= v <= hi:
            status = 2                          # a C int / int64 cannot hold it: OverflowError
        if kind == 3 and status == 0:
            assert int(fn(t)) == v
        assert s == status, (t[:60], s, status)
        if status == 0:
            assert o == v, t


def test_parse_numerals_host_refuses_bad_arguments():
    lib = _lib.lib()
    out = np.zeros(1, np.uint64)
    st = np.zeros(1, np.int32)
    off = np.zeros(2, np.int64)
    buf = np.zeros(1, np.uint8)
    assert lib.arb_libsvm_parse_numerals_host(None, off.ctypes.data, 1, 0, out.ctypes.data, st.ctypes.data) == -1
    assert lib.arb_libsvm_parse_numerals_host(buf.ctypes.data, off.ctypes.data, 1, 4, out.ctypes.data,
                                              st.ctypes.data) == -1
    assert b"kind" in lib.arb_last_error()


def test_python_layer_refusals():
    with pytest.raises(ValueError, match="parser"):
        data.SlateStore.from_svm_file("does-not-matter.txt", parser="gpu")
    with pytest.raises(ValueError, match="data_parser"):
        integration.patch_allrank(data_parser="cuda")
    with pytest.raises(_lib.ArbError):
        data.LibSVMPlan(torch.zeros(4, dtype=torch.uint8))
    with pytest.raises(_lib.ArbError):
        data.read_svm_to_device(__file__, device="cpu")


def test_only_regular_files_are_sized_by_fstat(tmp_path):
    import bz2
    import gzip
    text = b"1 qid:1 1:2\n" * 1000
    (tmp_path / "t.txt").write_bytes(text)
    (tmp_path / "t.txt.gz").write_bytes(gzip.compress(text))
    (tmp_path / "t.txt.bz2").write_bytes(bz2.compress(text))
    with open(tmp_path / "t.txt", "rb") as fh:
        assert data.plain_file_size(fh) == len(text)
        fh.read(5)
        assert data.plain_file_size(fh) == len(text) - 5
    with open(tmp_path / "t.txt", "rb", buffering=0) as fh:
        assert data.plain_file_size(fh) == len(text)
    for name in ("t.txt.gz", "t.txt.bz2"):             # decompressed by suffix, as sklearn does
        f, own = data.open_svm(tmp_path / name)
        with f:
            assert own and data.plain_file_size(f) is None and f.read() == text
    with gzip.open(tmp_path / "t.txt.gz", "rb") as gz:  # fileno() is the compressed file's
        assert data.plain_file_size(gz) is None
    assert data.plain_file_size(__import__("io").BytesIO(text)) is None


def test_numeral_header_builds_with_gxx(tmp_path):
    """libsvm_numeral.cuh compiles as plain C++ with standard headers included after it."""
    import os
    import shutil
    import subprocess
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    csrc = os.path.join(os.path.dirname(data.__file__), "csrc")
    src = tmp_path / "t.cpp"
    src.write_text('#include "libsvm_numeral.cuh"\n#include <cstdio>\n#include <memory>\n#include <vector>\n'
                   'int main() { double v = 0; const char* s = "2.2250738585072011e-308";\n'
                   '  int st = arb::svm::parse_py_float(reinterpret_cast<const uint8_t*>(s), 23, &v);\n'
                   '  std::vector<int> k{1}; std::printf("%d %a\\n", st, v); return k[0] - 1; }\n')
    exe = tmp_path / "t"
    r = subprocess.run([gxx, "-std=c++17", "-O1", "-I", csrc, str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert out[0] == "0" and float.fromhex(out[1]) == float("2.2250738585072011e-308")


def test_loaders_take_the_parser_keyword():
    for fn in (data.load_libsvm_role, data.load_libsvm_dataset_role, data.load_libsvm_dataset,
               data.SlateStore.from_svm_file):
        p = inspect.signature(fn).parameters["parser"]
        assert p.default == "sklearn"
    assert inspect.signature(integration.patch_allrank).parameters["data_parser"].default == "sklearn"
