"""The GEMM (csrc/gemm_tf32.cu) through its whole launch descriptor (arb_gemm_launch), against exact host references.

Every launch the scorer issues is reachable here: the epilogues (bias, ReLU, dropout, residual, ReLU mask from an aux
tile or from bit words, column sums), pitched and 4-D batched views, device-side row counts, split-K, bf16.  The
operands come in three kinds:

  a. rounding: one operand one-hot, so that C is the other operand after the kernel's fp32 -> tf32 rounding, bit for
     bit; planted ties (low 13 bits 0x1000, tf32 LSB even and odd), +-0 and values just below a power of two tell
     nearest-even from truncation, from ties-away and from rounding one operand twice;
  b. accumulation: random operands against the fp64 product of the host-rounded operands, within
     TAU * ceil(K / 8) * 2^-24 * sum |a~ b~| (one rounding per k8 step of the tensor core; the worst observed ratio is
     printed at the end of the module);
  c. epilogues and indexing: small-integer operands, whose products are exact in any order, so the expected output is
     computed on the host in float32 in the kernel's order and compared bit for bit.

Every case runs twice and must give the same bits, on NaN-prefilled outputs (bit words: -1), on both the one-tile and
the persistent kernel where the shape allows both, at block_n 32 / 64 / 128."""
import contextlib
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from tests.dropout_masks import M32, _mix32, _site
from tests.test_gpu_attn_bwd_order import det_reduce

pytestmark = pytest.mark.gpu

BIAS, RELU, ADD_AUX, MASK_AUX, ATOMIC, DROPOUT, COLSUM, RELU_BITS, MASK_BITS = 1, 2, 4, 8, 16, 32, 64, 128, 256
E_INVALID_ARG, E_UNSUPPORTED = -1, -2
F32 = np.float32
NAN = float("nan")
BIG_M = 2 ** 17 + 37          # 1025 row tiles: the persistent kernel walks several per CTA, DetParts runs two levels
TAU = 2.0                     # accumulation bound constant (b)
RATIOS = {}                   # worst error / bound per product kind (b)

i32, i64, u32, vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32, ctypes.c_void_p


class View(ctypes.Structure):
    _fields_ = [("ptr", vp), ("dim", i64 * 4), ("stride", i64 * 4), ("bf16", i32)]


class Desc(ctypes.Structure):
    _fields_ = ([(n, i32) for n in ("M", "N", "K", "a_mn", "b_mn", "b_tf32", "dgrad")]
                + [(n, View) for n in ("A", "B", "C", "aux")]
                + [(n, i32) for n in ("nb2", "nb3", "a_b2", "a_b3", "b_b2", "b_b3", "c_b2", "c_b3", "block_n",
                                      "split_k", "flags")]
                + [("alpha", ctypes.c_float), ("bias", vp), ("atomic_out", vp), ("atomic_ld", i64),
                   ("drop_seed", u32), ("drop_thresh", u32), ("drop_scale", ctypes.c_float), ("drop_key", u32),
                   ("drop_call_seed", vp), ("colsum_out", vp), ("bits", vp), ("rows_dev", vp)])


@pytest.fixture(scope="module")
def lib():
    from allrank_b200 import _lib
    _lib.register("arb_gemm_launch", i32, [ctypes.POINTER(Desc), vp])
    _lib.register("arb_set_gemm_persistent", None, [i32])
    _lib.register("arb_set_tf32_round_on_load", None, [i32])
    yield _lib
    for name, worst in sorted(RATIOS.items()):
        print(f"gemm: worst error / bound of {name}: {worst:.3g}")


def _ptr(t):
    return None if t is None else t.data_ptr()


def view(t, dims, strides, off=0):
    v = View()
    v.ptr = t.data_ptr() + off * t.element_size()
    for i in range(4):
        v.dim[i] = dims[i] if i < len(dims) else 1
        v.stride[i] = strides[i] if i < len(strides) else 0
    v.bf16 = int(t.dtype == torch.bfloat16)
    return v


def mat(t, cols, off=0):
    """[rows, cols] view of a 2-D buffer with its own row pitch, starting at column `off`."""
    return view(t, (cols, t.shape[0]), (1, t.stride(0)), off)


def padded(x, fill=NAN):
    """x in a buffer whose row pitch is wider than the row, the tail filled with `fill` (nothing past a view's dim[0]
    may be read or written)."""
    per16 = 16 // x.element_size()
    pitch = (x.shape[1] + per16 - 1) // per16 * per16 + per16
    buf = torch.full((x.shape[0], pitch), fill, dtype=x.dtype, device="cuda")
    buf[:, :x.shape[1]] = x
    return buf


def operand(x, mn):
    """The logical operand x [rows, K] stored K-major (x itself) or MN-major (its transpose): (buffer, view)."""
    buf = padded(x.t() if mn else x)
    return buf, mat(buf, x.shape[0] if mn else x.shape[1])


def out_buf(M, N, dtype=torch.float32):
    return padded(torch.full((M, N), NAN, dtype=dtype, device="cuda"))


def desc(M, N, K, A, B, C, a_mn=0, b_mn=0, block_n=64, flags=0, alpha=1.0, aux=None, bias=None, b_tf32=0,
         atomic_out=None, split_k=1, drop=None, colsum=None, bits=None, rows_dev=None):
    d = Desc()
    d.M, d.N, d.K, d.a_mn, d.b_mn, d.b_tf32 = M, N, K, a_mn, b_mn, b_tf32
    d.A, d.B = A, B
    if C is not None:
        d.C = C
    if aux is not None:
        d.aux = aux
    d.nb2 = d.nb3 = 1
    d.block_n, d.split_k, d.flags, d.alpha = block_n, split_k, flags, alpha
    d.bias = _ptr(bias)
    if atomic_out is not None:
        d.atomic_out, d.atomic_ld = atomic_out.data_ptr(), atomic_out.stride(0)
    d.drop_scale = 1.0
    if drop is not None:
        d.drop_seed, d.drop_thresh, d.drop_scale, d.drop_key = drop["seed"], drop["thresh"], drop["scale"], drop["key"]
        d.drop_call_seed = _ptr(drop.get("call_seed"))
    d.colsum_out, d.bits, d.rows_dev = _ptr(colsum), _ptr(bits), _ptr(rows_dev)
    return d


def launch(lib, d):
    return lib.lib().arb_gemm_launch(ctypes.byref(d), lib.stream_ptr())


def run(lib, d):
    lib.check(launch(lib, d), "arb_gemm_launch")
    torch.cuda.synchronize()


@contextlib.contextmanager
def gemm_kernel(lib, persistent):
    lib.lib().arb_set_gemm_persistent(persistent)
    try:
        yield
    finally:
        lib.lib().arb_set_gemm_persistent(int(os.environ.get("ARB_GEMM_PERSISTENT", 2)))


def kernels(a_mn, b_mn, bf16=False):
    """persistent settings that reach distinct kernels: fp32 pairs both MN-major and bf16 have the one-tile kernel only"""
    return (0,) if bf16 or (a_mn and b_mn) else (0, 1)


def bits_of(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def twice(fn):
    """fn() -> tuple of outputs; run it twice on fresh buffers and require the same bits."""
    first, second = fn(), fn()
    for x, y in zip(first, second):
        assert torch.equal(bits_of(x), bits_of(y)), "two identical launches gave different bits"
    return first


def assert_exact(got, want, what):
    got = got.float().cpu()
    want = torch.as_tensor(want).float().cpu()
    ok = (got == want) | (torch.isnan(got) & torch.isnan(want))
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} of {ok.numel()} elements differ, first at {i}: "
                             f"got {float(got[i])!r} want {float(want[i])!r}")


def sentinel_kept(buf, cols, what):
    tail = buf[:, cols:]
    if tail.dtype == torch.int32:
        assert bool((tail == -1).all()), f"{what}: the kernel wrote past the view"
    else:
        assert bool(torch.isnan(tail.float()).all()), f"{what}: the kernel wrote past the view"


# ---- host restatements ---------------------------------------------------------------------------------------------
def tf32(x, nearest=True):
    """fp32 -> tf32: round to nearest even (cvt.rn.tf32.f32), or truncate (what the tensor core does to raw fp32)."""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    if nearest:
        b = b + 0xFFF + ((b >> 13) & 1)
    b = b & 0xFFFFE000
    return torch.where(b >= 2 ** 31, b - 2 ** 32, b).to(torch.int32).view(torch.float32)


def keep_mask(M, N, seed, thresh):
    """drop_keep (csrc/dropout.cuh) at element m * N + n."""
    idx = np.arange(M * N, dtype=np.uint64)
    h = _mix32((idx & M32) ^ np.uint64(seed))
    h = _mix32((h + (idx >> np.uint64(32)) * np.uint64(0x9e3779b1) + np.uint64(0x7f4a7c15)) & M32)
    return (h >= np.uint64(thresh)).reshape(M, N)


def drop_site(p, call_seed=None, seed=0x2545F491):
    """The launch's dropout site for rate p (p = None: thresh 1), with the seed given directly or through a device
    call-seed word (make_drop_site's derivation, restated by tests/dropout_masks.py)."""
    if p is None:
        thresh, scale = 1, F32(1.0)
    else:
        thresh = max(1, min(int(float(F32(p)) * 4294967296.0), 0xFFFFFFFF))
        scale = F32(1.0) / (F32(1.0) - F32(p))
    d = dict(seed=seed, thresh=thresh, scale=float(scale), key=0)
    if call_seed is not None:
        layer, site = 1, 3
        d["key"] = layer * 8 + site + 1
        d["call_seed"] = torch.tensor([call_seed], dtype=torch.int64, device="cuda")
        d["host_seed"] = int(_site(call_seed, layer, site, 0.5)[0])
        d["seed"] = 0                        # must not be used
    else:
        d["host_seed"] = seed
    return d


def epilogue(acc, flags, alpha=1.0, bias=None, aux=None, drop=None, word_mask=None, fused_aux=False):
    """The epilogue in the kernel's order, float32: acc*alpha, + bias, ReLU, keep ? x*scale : 0, + aux / mask.
    fused_aux: the kept x*scale + aux as one rounding (ptxas may contract the two into an FFMA)."""
    M, N = acc.shape
    x = acc.astype(F32) * F32(alpha)
    if flags & BIAS:
        x = x + bias[None, :]
    if flags & RELU:
        x = np.maximum(x, F32(0))
    if flags & DROPOUT:
        keep = keep_mask(M, N, drop["host_seed"], drop["thresh"])
        if fused_aux and flags & ADD_AUX:
            f = (x.astype(np.float64) * np.float64(F32(drop["scale"])) + aux.astype(np.float64)).astype(F32)
            return np.where(keep, f, aux)
        x = np.where(keep, x * F32(drop["scale"]), F32(0))
    if flags & ADD_AUX:
        x = x + aux
    if flags & MASK_AUX:
        x = np.where(aux > 0, x, F32(0))
    if flags & MASK_BITS:
        x = np.where(word_mask, x, F32(0))
    return x.astype(F32)


def pack_bits(mask):
    """[M, N] bool -> [M, N / 32] int32 words, bit j of word w = mask[:, 32 w + j]."""
    M, N = mask.shape
    w = (mask.reshape(M, N // 32, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1)
    return w.astype(np.uint32).view(np.int32)


def unpack_bits(words, N):
    w = words.view(np.uint32).astype(np.uint64)
    return ((w[:, :, None] >> np.arange(32, dtype=np.uint64)) & 1).astype(bool).reshape(w.shape[0], N)


def tile_sums(C, persistent):
    """Per 128-row tile and column, the kernel's column sum over its stored C (rows past M are zeros): the one-tile
    kernel adds the 128 rows in order from 0.f; the persistent one adds four 32-row runs so and combines them by two
    shuffles, (s0 + s1) + (s2 + s3)."""
    M, N = C.shape
    T = (M + 127) // 128
    Cp = np.zeros((T * 128, N), F32)
    Cp[:M] = C
    Cp = Cp.reshape(T, 128, N)
    runs = []
    for r0, r1 in ([(0, 32), (32, 64), (64, 96), (96, 128)] if persistent else [(0, 128)]):
        t = np.zeros((T, N), F32)
        for r in range(r0, r1):
            t = t + Cp[:, r]
        runs.append(t)
    return (runs[0] + runs[1]) + (runs[2] + runs[3]) if persistent else runs[0]


def colsum_expect(C, persistent, col0, live_tiles=None):
    slots = tile_sums(C, persistent)
    if live_tiles is not None:
        slots[live_tiles:] = 0
    return col0 + det_reduce(slots)


def small_ints(shape, lo, hi, gen, dtype=torch.float32):
    return torch.randint(lo, hi + 1, shape, generator=gen).to(dtype).cuda()


# ---- a. rounding, bit-exact ----------------------------------------------------------------------------------------
def planted(shape, gen):
    """fp32 values whose tf32 rounding is delicate: exact ties (low 13 bits 0x1000) with the tf32 LSB even and odd,
    one ulp either side of a tie, +-0, the largest values below a power of two, and plain random ones."""
    b = torch.randn(shape, generator=gen).view(torch.int32)
    kind = torch.randint(0, 8, shape, generator=gen)
    b = torch.where(kind == 1, (b & ~0x3FFF) | 0x1000, b)           # tie, tf32 LSB even
    b = torch.where(kind == 2, (b & ~0x3FFF) | 0x3000, b)           # tie, tf32 LSB odd
    b = torch.where(kind == 3, (b & ~0x1FFF) | 0x1001, b)           # just above a tie
    b = torch.where(kind == 4, (b & ~0x1FFF) | 0x0FFF, b)           # just below a tie
    b = torch.where(kind == 5, (b & ~0x7FFFFF) - 1, b)              # just below a power of two: rounds up a binade
    b = torch.where(kind == 6, b & -2 ** 31, b)                     # +-0
    return b.view(torch.float32)


ROUND_PATHS = {"wgmma": (0, 0), "k-major rewrite": (1, 1), "mma.sync A mn": (1, 0), "mma.sync B mn": (0, 1)}


@pytest.mark.parametrize("M,N,K", [(300, 136, 136), (129, 36, 36)])
@pytest.mark.parametrize("side", ["A", "B"])
@pytest.mark.parametrize("nearest", [1, 0], ids=["rn", "truncate"])
@pytest.mark.parametrize("path", list(ROUND_PATHS))
def test_operand_rounding_is_bit_exact(lib, path, nearest, side, M, N, K):
    """C = one operand after the kernel's rounding: A side with a one-hot B (wgmma: A rounded in registers), B side with
    a one-hot A (wgmma: the B stage rounded in shared memory, rnd_b).  With a pre-rounded B, b_tf32 = 1 gives the bits
    of b_tf32 = 0."""
    a_mn, b_mn = ROUND_PATHS[path]
    gen = torch.Generator().manual_seed(M + K + 2 * nearest + (side == "B"))
    if side == "A":
        A = planted((M, K), gen)
        B = (torch.arange(K)[None, :] == (torch.arange(N) % K)[:, None]).float()
        want = tf32(A, nearest)[:, torch.arange(N) % K]
    else:
        B = planted((N, K), gen)
        A = (torch.arange(K)[None, :] == (torch.arange(M) % K)[:, None]).float()
        want = tf32(B, nearest)[:, torch.arange(M) % K].t()
    Ab, Av = operand(A.cuda(), a_mn)
    variants = [(B, 0)] + ([(tf32(B), 1), (tf32(B), 0)] if nearest else [])
    try:
        lib.lib().arb_set_tf32_round_on_load(nearest)
        for Bx, b_tf32 in variants:
            Bb, Bv = operand(Bx.cuda(), b_mn)
            for persistent in kernels(a_mn, b_mn):
                for block_n in (32, 64, 128):
                    def go():
                        C = out_buf(M, N)
                        with gemm_kernel(lib, persistent):
                            run(lib, desc(M, N, K, Av, Bv, mat(C, N), a_mn, b_mn, block_n, b_tf32=b_tf32))
                        return (C,)
                    C, = twice(go)
                    what = f"{path} {side} side b_tf32={b_tf32} persistent={persistent} block_n={block_n}"
                    assert_exact(C[:, :N], want, what)
                    sentinel_kept(C, N, what)
    finally:
        lib.lib().arb_set_tf32_round_on_load(1)


@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_bf16_operands_and_output_rounding_are_bit_exact(lib, a_mn, b_mn):
    """bf16 operands reach the fp32 accumulator exactly (one-hot products); a bf16 output (K-major A or B: with both
    operands MN-major the GEMM refuses it, test_refusals_launch_nothing) is rounded to nearest even
    (ties planted through the bias: column n holds values of one binade 2^e_n, and the bias 2^(e_n - 8) is half a bf16
    ulp of them, so one-hot product + bias lies halfway between two bf16 numbers, their last bit even or odd)."""
    M, N, K = 300, 136, 136
    gen = torch.Generator().manual_seed(5 + 2 * a_mn + b_mn)
    e = torch.randint(-3, 4, (K,), generator=gen).float()
    mant = 1 + torch.randint(0, 128, (M, K), generator=gen).float() / 128
    sign = torch.randint(0, 2, (M, K), generator=gen).float() * 2 - 1
    A = (sign * mant * torch.exp2(e)[None, :]).to(torch.bfloat16)
    A[torch.rand(M, K, generator=gen) < 0.05] = 0.0
    B = (torch.arange(K)[None, :] == torch.arange(N)[:, None]).to(torch.bfloat16)
    Ab, Av = operand(A.cuda(), a_mn)
    Bb, Bv = operand(B.cuda(), b_mn)
    a32 = A[:, :N].float()
    bias = torch.exp2(e[:N] - 8).contiguous()
    for block_n in (64, 128):
        def go():
            C32 = out_buf(M, N)
            run(lib, desc(M, N, K, Av, Bv, mat(C32, N), a_mn, b_mn, block_n))
            C16 = out_buf(M, N, torch.bfloat16)
            if not (a_mn and b_mn):
                run(lib, desc(M, N, K, Av, Bv, mat(C16, N), a_mn, b_mn, block_n, flags=BIAS, bias=bias.cuda()))
            return C32, C16
        C32, C16 = twice(go)
        assert_exact(C32[:, :N], a32, f"bf16 operands block_n={block_n}")
        sentinel_kept(C32, N, "bf16 operands")
        if a_mn and b_mn:
            continue
        want16 = (a32 + bias[None, :]).to(torch.bfloat16)
        assert_exact(C16[:, :N], want16.float(), f"bf16 output block_n={block_n}")
        sentinel_kept(C16, N, "bf16 output")


# ---- b. accumulation, bounded --------------------------------------------------------------------------------------
def check_bound(got, ref, scale, K, alpha, name):
    """|got - ref| <= TAU * (ceil(K/8) + 1) * 2^-24 * |alpha| * sum |a~ b~| (+1: the rounding of acc * alpha)."""
    bound = TAU * (math.ceil(K / 8) + 1) * 2.0 ** -24 * abs(alpha) * scale + 1e-30
    err = (got.double() - ref).abs()
    r = err / bound
    worst = float(r.max()) if r.numel() else 0.0
    RATIOS[name] = max(RATIOS.get(name, 0.0), worst)
    assert bool(torch.isfinite(got).all()), f"{name}: non-finite outputs"
    assert worst <= 1.0, f"{name}: worst error / bound {worst:.3g}"


@pytest.mark.parametrize("M,N,K", [(1, 4, 4), (127, 36, 1000), (129, 200, 4013), (300, 96, 136), (BIG_M, 136, 36)])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_accumulation_within_the_depth_bound(lib, a_mn, b_mn, M, N, K):
    gen = torch.Generator().manual_seed(M + N + K + 2 * a_mn + b_mn)
    A = torch.randn(M, K, generator=gen).cuda()
    B = torch.randn(N, K, generator=gen).cuda()
    Ar, Br = tf32(A), tf32(B)
    ref = Ar.double() @ Br.double().t()
    scale = Ar.double().abs() @ Br.double().abs().t()
    Ab, Av = operand(A, a_mn)
    Bb, Bv = operand(B, b_mn)
    outs = []
    for persistent in kernels(a_mn, b_mn):
        for block_n in (32, 64, 128):
            def go():
                C = out_buf(M, N)
                with gemm_kernel(lib, persistent):
                    run(lib, desc(M, N, K, Av, Bv, mat(C, N), a_mn, b_mn, block_n))
                return (C,)
            C, = twice(go)
            sentinel_kept(C, N, "accumulation")
            check_bound(C[:, :N], ref, scale, K, 1.0, f"product a_mn={a_mn} b_mn={b_mn}")
            outs.append(C)
    # wgmma: same instruction shapes and k order in both kernels and at every tile width, so the same bits
    if a_mn == b_mn == 0:
        for C in outs[1:]:
            assert torch.equal(bits_of(C), bits_of(outs[0]))


# ---- c. epilogues and indexing, bit-exact --------------------------------------------------------------------------
FWD = [BIAS, BIAS | RELU, BIAS | RELU | DROPOUT, BIAS | DROPOUT, BIAS | ADD_AUX, BIAS | ADD_AUX | DROPOUT,
       BIAS | RELU | RELU_BITS]
DGRAD = [0, COLSUM, MASK_AUX | COLSUM, MASK_BITS | COLSUM]
SHAPES = [(1, 36, 4), (129, 96, 36), (300, 136, 136), (127, 200, 1000)]
BITS_SHAPES = [(1, 32, 4), (129, 96, 36), (300, 128, 136), (127, 32, 1000)]


def flag_id(f):
    names = [(BIAS, "bias"), (RELU, "relu"), (ADD_AUX, "add"), (MASK_AUX, "mask"), (DROPOUT, "drop"),
             (COLSUM, "colsum"), (RELU_BITS, "relubits"), (MASK_BITS, "maskbits")]
    return "+".join(n for b, n in names if f & b) or "plain"


def run_epilogue_case(lib, flags, M, N, K, b_mn=0, in_place=False, seed=0, alpha=None, drop=None, block_ns=(32, 64, 128),
                      persistents=None):
    gen = torch.Generator().manual_seed(seed + 1000 * M + N + K + flags)
    A = small_ints((M, K), -8, 8, gen)
    B = small_ints((N, K), -8, 8, gen)
    bias = small_ints((N,), -64, 64, gen) / 4
    aux = small_ints((M, N), -8, 8, gen) / 2
    col0 = torch.randn(N, generator=gen).cuda()
    acc = (A.double() @ B.double().t()).cpu().numpy()
    if alpha is None:
        alpha = 0.5 if flags & BIAS else (float(F32(1) / F32(0.9)) if flags & MASK_AUX else 1.0)
    if flags & DROPOUT and drop is None:
        drop = drop_site(0.1)
    word_mask = (aux.cpu().numpy() > 0) if flags & MASK_BITS else None
    words_in = torch.from_numpy(pack_bits(word_mask)).cuda() if flags & MASK_BITS else None
    Ab, Av = operand(A, 0)
    Bb, Bv = operand(B, b_mn)
    aux_np = aux.cpu().numpy()
    want = epilogue(acc, flags, alpha, bias.cpu().numpy(), aux_np, drop, word_mask)
    want_fused = epilogue(acc, flags, alpha, bias.cpu().numpy(), aux_np, drop, word_mask, fused_aux=True)
    for persistent in persistents or kernels(0, b_mn):
        for block_n in block_ns:
            def go():
                C = padded(aux) if in_place else out_buf(M, N)
                X = C if in_place else padded(aux)
                bits = torch.full((M, N // 32), -1, dtype=torch.int32, device="cuda") if flags & RELU_BITS else None
                cs = col0.clone() if flags & COLSUM else None
                d = desc(M, N, K, Av, Bv, mat(C, N), 0, b_mn, block_n, flags, alpha, bias=bias,
                         aux=mat(X, N) if flags & (ADD_AUX | MASK_AUX) else None, drop=drop, colsum=cs,
                         bits=words_in if flags & MASK_BITS else bits)
                with gemm_kernel(lib, persistent):
                    run(lib, d)
                return tuple(t for t in (C, bits, cs) if t is not None)
            outs = twice(go)
            C = outs[0]
            what = f"{flag_id(flags)} M={M} N={N} K={K} b_mn={b_mn} persistent={persistent} block_n={block_n}"
            got = C[:, :N].cpu().numpy()
            if flags & DROPOUT and flags & ADD_AUX:
                # the kept x * scale + aux: two roundings, or one where ptxas contracts them (either, consistently)
                if not np.array_equal(got, want_fused):
                    assert_exact(C[:, :N], want, what)
            else:
                assert_exact(C[:, :N], want, what)
            sentinel_kept(C, N, what)
            k = 1
            if flags & RELU_BITS:
                assert torch.equal(outs[k].cpu(), torch.from_numpy(pack_bits(got > 0))), what + " bit words"
                k += 1
            if flags & COLSUM:
                want_cs = colsum_expect(got, persistent, col0.cpu().numpy())
                assert np.array_equal(outs[k].cpu().numpy().view(np.int32), want_cs.view(np.int32)), \
                    what + " column sums"


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("flags", [f for f in FWD if not f & RELU_BITS], ids=flag_id)
def test_forward_epilogues(lib, flags, M, N, K):
    run_epilogue_case(lib, flags, M, N, K)


@pytest.mark.parametrize("M,N,K", BITS_SHAPES)
@pytest.mark.parametrize("flags", [BIAS | RELU | RELU_BITS, MASK_BITS | COLSUM, MASK_BITS], ids=flag_id)
def test_relu_bit_words(lib, flags, M, N, K):
    """EPI_RELU_BITS words are pack(C > 0); EPI_MASK_BITS masks as EPI_MASK_AUX does with an aux tile carrying the
    same mask (N = 96 at block_n 64: a half-filled tile; N = 32: one word per row)."""
    run_epilogue_case(lib, flags, M, N, K)
    if flags & MASK_BITS:
        run_epilogue_case(lib, flags & ~MASK_BITS | MASK_AUX, M, N, K, alpha=1.0)


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("b_mn", [0, 1])
@pytest.mark.parametrize("flags", [f for f in DGRAD if not f & MASK_BITS], ids=flag_id)
def test_input_gradient_epilogues(lib, flags, b_mn, M, N, K):
    run_epilogue_case(lib, flags, M, N, K, b_mn=b_mn)


@pytest.mark.parametrize("M,N,K", SHAPES[1:])
def test_residual_in_place(lib, M, N, K):
    """aux aliasing C: the residual stream updated in place (the attention-output and FFN-output linears)."""
    run_epilogue_case(lib, BIAS | ADD_AUX, M, N, K, in_place=True)
    run_epilogue_case(lib, BIAS | ADD_AUX | DROPOUT, M, N, K, in_place=True)


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9, None], ids=["p0.1", "p0.5", "p0.9", "thresh1"])
@pytest.mark.parametrize("source", ["seed", "call_seed"])
@pytest.mark.parametrize("flags", [BIAS | RELU | DROPOUT, BIAS | DROPOUT, BIAS | ADD_AUX | DROPOUT], ids=flag_id)
def test_dropout_sites(lib, flags, source, p):
    """The zeros of C are the host drop_keep at m N + n, kept elements the scaled value; the seed given directly or
    derived in the kernel from the device call-seed word and the site key."""
    drop = drop_site(p, call_seed=0x0123456789ABCDEF if source == "call_seed" else None)
    run_epilogue_case(lib, flags, 300, 136, 136, drop=drop)


@pytest.mark.parametrize("flags", [BIAS | RELU | DROPOUT, BIAS | ADD_AUX | DROPOUT], ids=flag_id)
def test_dropout_with_thresh_zero_is_no_dropout(lib, flags):
    M, N, K = 129, 96, 36
    gen = torch.Generator().manual_seed(11)
    A, B = small_ints((M, K), -8, 8, gen), small_ints((N, K), -8, 8, gen)
    bias, aux = small_ints((N,), -8, 8, gen), small_ints((M, N), -8, 8, gen)
    Ab, Av = operand(A, 0)
    Bb, Bv = operand(B, 0)
    Xb = padded(aux)
    off = dict(seed=77, thresh=0, scale=3.0, key=0)
    for persistent in (0, 1):
        outs = []
        for f, drop in ((flags, off), (flags & ~DROPOUT, None)):
            C = out_buf(M, N)
            with gemm_kernel(lib, persistent):
                run(lib, desc(M, N, K, Av, Bv, mat(C, N), 0, 0, 64, f, 0.5, aux=mat(Xb, N), bias=bias, drop=drop))
            outs.append(C)
        assert torch.equal(bits_of(outs[0]), bits_of(outs[1]))


@pytest.mark.parametrize("split_k", [1, 7, 37, 1000])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_weight_gradient_accumulates(lib, dtype, split_k):
    """dW += dY^T X, split-K over the rows (both operands MN-major), into a non-zero dW; the splits' slots are summed
    by DetParts.  split_k beyond the number of k-blocks leaves no split empty-handed: it is clamped."""
    R, out_f, in_f = 1700, 96, 136
    gen = torch.Generator().manual_seed(split_k)
    lo = -8 if dtype == torch.float32 else -4
    dY = small_ints((R, out_f), lo, -lo, gen, dtype)
    X = small_ints((R, in_f), lo, -lo, gen, dtype)
    dW0 = small_ints((out_f, in_f), -100, 100, gen)
    want = dW0.double() + dY.double().t() @ X.double()
    Ab, Av = operand(dY.t(), 1)
    Bb, Bv = operand(X.t(), 1)
    for block_n in ((32, 64, 128) if dtype == torch.float32 else (64, 128)):
        def go():
            dW = padded(dW0)
            run(lib, desc(out_f, in_f, R, Av, Bv, None, 1, 1, block_n, ATOMIC, atomic_out=dW, split_k=split_k))
            return (dW,)
        dW, = twice(go)
        assert_exact(dW[:, :in_f], want, f"weight gradient {dtype} split_k={split_k} block_n={block_n}")
        sentinel_kept(dW, in_f, "weight gradient")


@pytest.mark.parametrize("flags", [BIAS | RELU, BIAS | RELU | DROPOUT, BIAS | ADD_AUX, BIAS | ADD_AUX | DROPOUT,
                                   MASK_AUX | COLSUM], ids=flag_id)
def test_bf16_epilogues(lib, flags):
    """bf16 mode: BIAS|RELU(|DROPOUT) into bf16, BIAS|ADD_AUX(|DROPOUT) into fp32, MASK_AUX|COLSUM into bf16 with
    alpha (the column sums add the bf16-rounded terms in fp32)."""
    M, N, K = 300, 136, 1000
    out16 = not flags & ADD_AUX
    gen = torch.Generator().manual_seed(flags)
    A = small_ints((M, K), -4, 4, gen, torch.bfloat16)
    B = small_ints((N, K), -4, 4, gen, torch.bfloat16)
    bias = small_ints((N,), -64, 64, gen) / 4
    aux = small_ints((M, N), -8, 8, gen) / 2
    col0 = torch.randn(N, generator=gen).cuda()
    alpha = 0.5 if flags & BIAS else float(F32(1) / F32(0.9))
    drop = drop_site(0.1) if flags & DROPOUT else None
    acc = (A.double() @ B.double().t()).cpu().numpy()
    aux_np = aux.to(torch.bfloat16 if out16 else torch.float32).float().cpu().numpy()
    for b_mn in ((0, 1) if not flags & DROPOUT else (0,)):
        Ab, Av = operand(A, 0)
        Bb, Bv = operand(B, b_mn)
        for block_n in (64, 128):
            def go():
                C = out_buf(M, N, torch.bfloat16 if out16 else torch.float32)
                X = padded(aux.to(C.dtype))
                cs = col0.clone() if flags & COLSUM else None
                run(lib, desc(M, N, K, Av, Bv, mat(C, N), 0, b_mn, block_n, flags, alpha, aux=mat(X, N), bias=bias,
                              drop=drop, colsum=cs))
                return tuple(t for t in (C, cs) if t is not None)
            outs = twice(go)
            C = outs[0]
            what = f"bf16 {flag_id(flags)} b_mn={b_mn} block_n={block_n}"
            want = epilogue(acc, flags, alpha, bias.cpu().numpy(), aux_np, drop)
            want_fused = epilogue(acc, flags, alpha, bias.cpu().numpy(), aux_np, drop, fused_aux=True)
            if out16:
                want = torch.from_numpy(want).to(torch.bfloat16).float().numpy()
            got = C[:, :N].float().cpu().numpy()
            if flags & DROPOUT and flags & ADD_AUX and np.array_equal(got, want_fused):
                pass
            else:
                assert_exact(C[:, :N], want, what)
            sentinel_kept(C, N, what)
            if flags & COLSUM:
                want_cs = colsum_expect(got, False, col0.cpu().numpy())
                assert np.array_equal(outs[1].cpu().numpy().view(np.int32), want_cs.view(np.int32)), what


# ---- column sums over many tiles -----------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 8192, 8193, BIG_M], ids=["1-slot", "64-slots", "65-slots", "1025-slots"])
@pytest.mark.parametrize("flags", [COLSUM, MASK_AUX | COLSUM, MASK_BITS | COLSUM], ids=flag_id)
def test_column_sums_follow_the_kernel_order(lib, flags, M):
    """Random operands: the b1 / FC-bias gradient equals, bit for bit, the kernel's order over its own stored C (one
    tile slot per 128 rows), reduced by DetParts and added to a non-zero incoming vector."""
    N, K = 96, 36
    gen = torch.Generator().manual_seed(M + flags)
    A = torch.randn(M, K, generator=gen).cuda()
    B = torch.randn(N, K, generator=gen).cuda()
    aux = torch.randn(M, N, generator=gen).cuda()
    col0 = torch.randn(N, generator=gen).cuda()
    words = torch.from_numpy(pack_bits(aux.cpu().numpy() > 0)).cuda()
    Ab, Av = operand(A, 0)
    Bb, Bv = operand(B, 0)
    Xb = padded(aux)
    for persistent in (0, 1):
        for block_n in ((32, 64, 128) if M < BIG_M else (64,)):
            def go():
                C = out_buf(M, N)
                cs = col0.clone()
                with gemm_kernel(lib, persistent):
                    run(lib, desc(M, N, K, Av, Bv, mat(C, N), 0, 0, block_n, flags, 2.0, aux=mat(Xb, N),
                                  bits=words if flags & MASK_BITS else None, colsum=cs))
                return C, cs
            C, cs = twice(go)
            got = C[:, :N].cpu().numpy()
            want = colsum_expect(got, persistent, col0.cpu().numpy())
            diff = np.nonzero(cs.cpu().numpy().view(np.int32) != want.view(np.int32))[0]
            assert diff.size == 0, f"{flag_id(flags)} M={M} persistent={persistent} block_n={block_n}: " \
                                   f"{diff.size} columns differ from the emulated order, first {diff[:4].tolist()}"


# ---- device-side row counts ----------------------------------------------------------------------------------------
M_LIVE = 1700
LIVES = [0, 128, 1536, M_LIVE // 128 * 128, 2 * M_LIVE]


@pytest.mark.parametrize("live", LIVES)
@pytest.mark.parametrize("flags", [BIAS | RELU | RELU_BITS, MASK_BITS | COLSUM, BIAS | ADD_AUX, BIAS | DROPOUT],
                         ids=flag_id)
def test_device_row_count_bounds_the_rows(lib, flags, live):
    """Rows at or past the live count hold NaN in the operand; below it the outputs equal the full launch's bits; from
    the first dead tile on, C, the bit words and the column-sum slots are untouched."""
    M, N, K = M_LIVE, 96, 136
    gen = torch.Generator().manual_seed(live + flags)
    A = torch.randn(M, K, generator=gen).cuda()
    B = torch.randn(N, K, generator=gen).cuda()
    bias = torch.randn(N, generator=gen).cuda()
    aux = torch.randn(M, N, generator=gen).cuda()
    col0 = torch.randn(N, generator=gen).cuda()
    words = torch.from_numpy(pack_bits(aux.cpu().numpy() > 0)).cuda()
    A_dead = A.clone()
    A_dead[live:] = NAN
    rows = torch.tensor([live], dtype=torch.int32, device="cuda")
    drop = drop_site(0.1)
    Bb, Bv = operand(B, 0)
    Xb = padded(aux)
    n_live = min(live, M)
    for persistent in (0, 1):
        for block_n in (32, 64, 128):
            outs = {}
            for name, Ax, rd in (("full", A, None), ("live", A_dead, rows)):
                Ab, Av = operand(Ax, 0)

                def go():
                    C = out_buf(M, N)
                    bits = torch.full((M, N // 32), -1, dtype=torch.int32, device="cuda")
                    cs = col0.clone()
                    d = desc(M, N, K, Av, Bv, mat(C, N), 0, 0, block_n, flags, 1.0, aux=mat(Xb, N), bias=bias,
                             drop=drop, colsum=cs if flags & COLSUM else None, rows_dev=rd,
                             bits=words if flags & MASK_BITS else (bits if flags & RELU_BITS else None))
                    with gemm_kernel(lib, persistent):
                        run(lib, d)
                    return C, bits, cs
                outs[name] = twice(go)
            (Cf, bf, _), (Cl, bl, csl) = outs["full"], outs["live"]
            what = f"{flag_id(flags)} live={live} persistent={persistent} block_n={block_n}"
            assert torch.equal(bits_of(Cl[:n_live]), bits_of(Cf[:n_live])), what
            assert bool(torch.isnan(Cl[n_live:]).all()), what + ": C written past the live rows"
            assert torch.equal(bl[:n_live], bf[:n_live]), what
            assert bool((bl[n_live:] == -1).all()), what + ": bit words written past the live rows"
            if flags & COLSUM:
                got = Cf[:, :N].cpu().numpy()
                want = colsum_expect(got, persistent, col0.cpu().numpy(), live_tiles=(n_live + 127) // 128)
                assert np.array_equal(csl.cpu().numpy().view(np.int32), want.view(np.int32)), what + " column sums"


@pytest.mark.parametrize("live", LIVES)
@pytest.mark.parametrize("split_k", [1, 7, 37, 1000])
def test_device_row_count_bounds_the_weight_gradient(lib, split_k, live):
    """Split-K weight gradients under a device row count reduce over the live rows only (the k-blocks redistributed
    over the grid's splits, some splits empty); rows past it hold NaN."""
    R, out_f, in_f = M_LIVE, 96, 136
    gen = torch.Generator().manual_seed(live * 3 + split_k)
    for dtype in (torch.float32, torch.bfloat16):
        lo = -8 if dtype == torch.float32 else -4
        dY = small_ints((R, out_f), lo, -lo, gen, dtype)
        X = small_ints((R, in_f), lo, -lo, gen, dtype)
        dW0 = small_ints((out_f, in_f), -100, 100, gen)
        n_live = min(live, R)
        want = dW0.double() + dY[:n_live].double().t() @ X[:n_live].double()
        dY[n_live:] = NAN
        X[n_live:] = NAN
        Ab, Av = operand(dY.t(), 1)
        Bb, Bv = operand(X.t(), 1)
        rows = torch.tensor([live], dtype=torch.int32, device="cuda")
        for block_n in ((32, 128) if dtype == torch.float32 else (64, 128)):
            def go():
                dW = padded(dW0)
                run(lib, desc(out_f, in_f, R, Av, Bv, None, 1, 1, block_n, ATOMIC, atomic_out=dW, split_k=split_k,
                              rows_dev=rows))
                return (dW,)
            dW, = twice(go)
            assert_exact(dW[:, :in_f], want, f"{dtype} live={live} split_k={split_k} block_n={block_n}")


# ---- views ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("part", [0, 1, 2], ids=["q", "k", "v"])
def test_pitched_views(lib, part):
    """A read from a [R, 3d] buffer at column offset part * d (pitch 3d); C and the residual written into column
    slices of wider buffers, whose neighbouring columns keep their sentinels."""
    R, d, N, off = 300, 64, 96, 32
    gen = torch.Generator().manual_seed(part)
    qkv = small_ints((R, 3 * d), -8, 8, gen)
    W = small_ints((N, d), -8, 8, gen)
    bias = small_ints((N,), -8, 8, gen)
    res = small_ints((R, N), -8, 8, gen)
    want = epilogue((qkv[:, part * d:(part + 1) * d].double() @ W.double().t()).cpu().numpy(), BIAS | ADD_AUX, 1.0,
                    bias.cpu().numpy(), res.cpu().numpy())
    Wb, Wv = operand(W, 0)
    for persistent in (0, 1):
        for block_n in (32, 64, 128):
            def go():
                C = torch.full((R, N + 64), NAN, device="cuda")
                X = torch.full((R, N + 96), NAN, device="cuda")
                X[:, 64:64 + N] = res
                run_d = desc(R, N, d, mat(qkv, d, part * d), Wv, mat(C, N, off), 0, 0, block_n, BIAS | ADD_AUX,
                             aux=mat(X, N, 64), bias=bias)
                with gemm_kernel(lib, persistent):
                    run(lib, run_d)
                return C, X
            C, X = twice(go)
            what = f"part={part} persistent={persistent} block_n={block_n}"
            assert_exact(C[:, off:off + N], want, what)
            assert bool(torch.isnan(C[:, :off]).all() and torch.isnan(C[:, off + N:]).all()), what
            assert bool(torch.isnan(X[:, :64]).all() and torch.isnan(X[:, 64 + N:]).all()), what
            assert torch.equal(X[:, 64:64 + N], res), what


def head_view(t, off, dk, S, h, B, pitch):
    return view(t, (dk, S, h, B), (1, pitch, dk, S * pitch), off)


def prob_view(t, S, Sp, h, B):
    return view(t, (S, S, h, B), (1, Sp, S * Sp, h * S * Sp))


def batched(M, N, K, A, B, C, a_mn, b_mn, block_n, alpha, h, nB):
    d = desc(M, N, K, A, B, C, a_mn, b_mn, block_n, 0, alpha)
    d.nb2, d.nb3 = h, nB
    d.a_b2 = d.a_b3 = d.b_b2 = d.b_b3 = d.c_b2 = d.c_b3 = 1
    return d


@pytest.mark.parametrize("h,nB", [(1, 1), (3, 1), (1, 5), (3, 5)])
@pytest.mark.parametrize("dk", [8, 24, 64, 96])
@pytest.mark.parametrize("S", [1, 37, 240, 257])
def test_unfused_attention_products(lib, S, dk, h, nB):
    """The products of the unfused attention path on head_view / prob_view, built as the scorer builds them
    (csrc/scorer.cu: the forward's Q K^T and P V, the backward's dP~, dV, dQ and dK), against fp64 per (slate, head)."""
    d = h * dk
    Sp = (S + 3) // 4 * 4 + 4
    alpha = 1.0 / math.sqrt(dk)
    pick = 32 if dk <= 32 else (64 if dk < 128 else 128)
    gen = torch.Generator().manual_seed(S * 7 + dk + 100 * h + nB)
    qkv = torch.randn(nB * S, 3 * d, generator=gen).cuda()
    dctx = torch.randn(nB * S, d, generator=gen).cuda()
    P = torch.full((nB, h, S, Sp), NAN, device="cuda")
    P[..., :S] = torch.rand(nB, h, S, S, generator=gen).cuda()
    dS = torch.full((nB, h, S, Sp), NAN, device="cuda")
    dS[..., :S] = torch.randn(nB, h, S, S, generator=gen).cuda()
    # fp64 per (slate, head) of the tf32-rounded operands: [B, h, S, dk]
    heads = lambda x, part, w: x.view(nB, S, w // d, h, dk)[:, :, part].permute(0, 2, 1, 3).double()  # noqa: E731
    Q, Kh, V = (heads(tf32(qkv), j, 3 * d) for j in range(3))
    dC = heads(tf32(dctx), 0, d)
    Pr, dSr = tf32(P[..., :S].contiguous()).double(), tf32(dS[..., :S].contiguous()).double()
    absd = lambda x: x.abs()  # noqa: E731
    cases = {
        # name: (M, N, K, A view, B view, a_mn, b_mn, block_n, alpha, (out, out view, reader), ref, scale)
        "QK^T": (S, S, dk, head_view(qkv, 0, dk, S, h, nB, 3 * d), head_view(qkv, d, dk, S, h, nB, 3 * d), 0, 0, 64,
                 alpha, "prob", Q @ Kh.transpose(-1, -2) * alpha, absd(Q) @ absd(Kh).transpose(-1, -2)),
        "PV": (S, dk, S, prob_view(P, S, Sp, h, nB), head_view(qkv, 2 * d, dk, S, h, nB, 3 * d), 0, 1, pick, 1.0,
               "ctx", Pr @ V, absd(Pr) @ absd(V)),
        "dP": (S, S, dk, head_view(dctx, 0, dk, S, h, nB, d), head_view(qkv, 2 * d, dk, S, h, nB, 3 * d), 0, 0, 64,
               1.0, "prob", dC @ V.transpose(-1, -2), absd(dC) @ absd(V).transpose(-1, -2)),
        "dV": (S, dk, S, prob_view(P, S, Sp, h, nB), head_view(dctx, 0, dk, S, h, nB, d), 1, 1, pick, 1.0,
               ("dqkv", 2), Pr.transpose(-1, -2) @ dC, absd(Pr).transpose(-1, -2) @ absd(dC)),
        "dQ": (S, dk, S, prob_view(dS, S, Sp, h, nB), head_view(qkv, d, dk, S, h, nB, 3 * d), 0, 1, pick, alpha,
               ("dqkv", 0), dSr @ Kh * alpha, absd(dSr) @ absd(Kh)),
        "dK": (S, dk, S, prob_view(dS, S, Sp, h, nB), head_view(qkv, 0, dk, S, h, nB, 3 * d), 1, 1, pick, alpha,
               ("dqkv", 1), dSr.transpose(-1, -2) @ Q * alpha, absd(dSr).transpose(-1, -2) @ absd(Q)),
    }
    for name, (M, N, K, Av, Bv, a_mn, b_mn, block_n, al, out, ref, scale) in cases.items():
        def go():
            if out == "prob":
                buf = torch.full((nB, h, S, Sp), NAN, device="cuda")
                Cv = prob_view(buf, S, Sp, h, nB)
            elif out == "ctx":
                buf = torch.full((nB * S, d), NAN, device="cuda")
                Cv = head_view(buf, 0, dk, S, h, nB, d)
            else:
                buf = torch.full((nB * S, 3 * d), NAN, device="cuda")
                Cv = head_view(buf, out[1] * d, dk, S, h, nB, 3 * d)
            run(lib, batched(M, N, K, Av, Bv, Cv, a_mn, b_mn, block_n, al, h, nB))
            return (buf,)
        buf, = twice(go)
        if out == "prob":
            # the TMA store writes whole 16-byte granules: a row's last granule may be zero-filled past S (the scorer's
            # pitch is S rounded up to 4); the columns beyond it must keep their sentinels
            got = buf[..., :S]
            assert bool(torch.isnan(buf[..., (S + 3) // 4 * 4:]).all()), f"{name}: padding columns of the Sp pitch written"
        elif out == "ctx":
            got = heads(buf, 0, d)
        else:
            got = heads(buf, out[1], 3 * d)
            others = torch.ones(3, dtype=torch.bool)
            others[out[1]] = False
            rest = buf.view(nB, S, 3, d)[:, :, others]
            assert bool(torch.isnan(rest).all()), f"{name}: wrote outside its third of the [R, 3d] buffer"
        check_bound(got.float(), ref, scale, K, al, f"attention {name}")


# ---- refusals ------------------------------------------------------------------------------------------------------
def refusal_cases():
    """(name, expected code, descriptor overrides) -- each breaks one rule of launch_gemm_tf32"""
    return [
        ("relu bits with an aux tile", E_INVALID_ARG, dict(flags=BIAS | RELU | RELU_BITS | ADD_AUX, bits=1, aux=1)),
        ("relu bits with dropout", E_INVALID_ARG, dict(flags=BIAS | RELU | RELU_BITS | DROPOUT, bits=1, drop=1)),
        ("relu bits into bf16", E_INVALID_ARG, dict(flags=BIAS | RELU | RELU_BITS, bits=1, bf16_in=1, bf16_out=1)),
        ("relu bits with N % 32", E_INVALID_ARG, dict(flags=BIAS | RELU | RELU_BITS, bits=1, N=36)),
        ("mask bits with split-K", E_INVALID_ARG, dict(flags=MASK_BITS | ATOMIC, bits=1, atomic=1, a_mn=1, b_mn=1)),
        ("mask bits with an aux tile", E_INVALID_ARG, dict(flags=MASK_BITS | MASK_AUX, bits=1, aux=1)),
        ("relu bits without relu", E_INVALID_ARG, dict(flags=BIAS | RELU_BITS, bits=1)),
        ("bit words missing", E_INVALID_ARG, dict(flags=MASK_BITS)),
        ("bit words in a batched launch", E_INVALID_ARG, dict(flags=MASK_BITS, bits=1, nb2=2)),
        ("dropout with A mn-major", E_UNSUPPORTED, dict(flags=BIAS | DROPOUT, drop=1, a_mn=1)),
        ("dropout with B mn-major", E_UNSUPPORTED, dict(flags=BIAS | DROPOUT, drop=1, b_mn=1)),
        ("dropout bf16 with B mn-major", E_UNSUPPORTED, dict(flags=BIAS | DROPOUT, drop=1, b_mn=1, bf16_in=1)),
        ("column sums with split-K", E_INVALID_ARG, dict(flags=COLSUM | ATOMIC, colsum=1, atomic=1, a_mn=1, b_mn=1)),
        ("column sums missing", E_INVALID_ARG, dict(flags=COLSUM)),
        ("row count in a batched launch", E_INVALID_ARG, dict(rows=1, nb2=2)),
        ("bf16 output at block_n 32", E_INVALID_ARG, dict(bf16_in=1, bf16_out=1, block_n=32)),
        ("bf16 operands at block_n 32", E_INVALID_ARG, dict(bf16_in=1, block_n=32)),
        ("bf16 output from fp32 operands", E_INVALID_ARG, dict(bf16_out=1)),
        ("bf16 output, both operands mn-major", E_UNSUPPORTED, dict(bf16_in=1, bf16_out=1, a_mn=1, b_mn=1)),
        ("bf16 A with fp32 B", E_INVALID_ARG, dict(bf16_a_only=1)),
        ("bf16 aux into fp32", E_INVALID_ARG, dict(flags=ADD_AUX, aux=1, bf16_aux=1)),
        ("fp32 aux into bf16", E_INVALID_ARG, dict(flags=MASK_AUX, aux=1, bf16_in=1, bf16_out=1)),
        ("bf16 batched", E_UNSUPPORTED, dict(bf16_in=1, nb2=2)),
        ("split_k without split", E_INVALID_ARG, dict(split_k=4)),
        ("split-K batched", E_INVALID_ARG, dict(flags=ATOMIC, atomic=1, nb2=2, a_mn=1, b_mn=1)),
        ("split-K without atomic_out", E_INVALID_ARG, dict(flags=ATOMIC, a_mn=1, b_mn=1)),
        ("block_n 96", E_INVALID_ARG, dict(block_n=96)),
        ("M = 0", E_INVALID_ARG, dict(M=0)),
    ]


@pytest.mark.parametrize("persistent", [0, 1])
@pytest.mark.parametrize("name,code,o", refusal_cases(), ids=[c[0].replace(" ", "-") for c in refusal_cases()])
def test_refusals_launch_nothing(lib, name, code, o, persistent):
    M, N, K = o.get("M", 128), o.get("N", 128), 128
    in16 = torch.bfloat16 if o.get("bf16_in") else torch.float32
    A = torch.zeros(M if M else 1, K, dtype=torch.bfloat16 if o.get("bf16_a_only") else in16, device="cuda")
    B = torch.zeros(N, K, dtype=in16, device="cuda")
    C = torch.full((max(M, 1), N), NAN, dtype=torch.bfloat16 if o.get("bf16_out") else torch.float32, device="cuda")
    X = torch.zeros(max(M, 1), N, dtype=torch.bfloat16 if o.get("bf16_aux") else torch.float32, device="cuda")
    bits = torch.full((max(M, 1), max(N // 32, 1)), -1, dtype=torch.int32, device="cuda")
    cs = torch.zeros(N, device="cuda")
    dW = torch.zeros(M if M else 1, N, device="cuda")
    rows = torch.tensor([64], dtype=torch.int32, device="cuda")
    a_mn, b_mn = o.get("a_mn", 0), o.get("b_mn", 0)
    Av = mat(A.t().contiguous() if a_mn else A, max(M, 1) if a_mn else K)
    Bv = mat(B.t().contiguous() if b_mn else B, N if b_mn else K)
    d = desc(M, N, K, Av, Bv, mat(C, N), a_mn, b_mn, o.get("block_n", 64), o.get("flags", 0), 1.0,
             aux=mat(X, N) if o.get("aux") else None, bias=torch.zeros(N, device="cuda"),
             atomic_out=dW if o.get("atomic") else None, split_k=o.get("split_k", 1),
             drop=drop_site(0.1) if o.get("drop") else None, colsum=cs if o.get("colsum") else None,
             bits=bits if o.get("bits") else None, rows_dev=rows if o.get("rows") else None)
    if o.get("nb2"):
        d.nb2 = o["nb2"]
    torch.cuda.synchronize()
    before = lib.launch_count()
    with gemm_kernel(lib, persistent):
        rc = launch(lib, d)
    torch.cuda.synchronize()
    assert rc == code, (name, rc, lib.lib().arb_last_error())
    assert lib.launch_count() == before, f"{name}: refused, but launched a kernel"
    assert bool(torch.isnan(C.float()).all()) and bool((bits == -1).all()) and bool((cs == 0).all())
