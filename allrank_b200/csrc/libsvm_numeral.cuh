// Numerals of a LibSVM file, read exactly as sklearn.datasets.load_svmlight_file reads them: labels and feature
// values with Python's float(), feature indices with int() into a C int, qids with numpy.int64().  Every function is
// __host__ __device__: the kernels of libsvm.cu call them per token, and arb_libsvm_parse_numerals_host runs the same
// code on the CPU so that it can be compared with Python without a GPU.
//
// Grammar of float() on bytes (CPython 3.12; anything else is refused):
//   [+-] ( digits [ "." [digits] ] | "." digits ) [ (e|E) [+-] digits ]      digits = [0-9] ( "_"? [0-9] )*
//   [+-] ( "inf" | "infinity" | "nan" )                                       ASCII case-insensitive
// A "_" sits between two digits.  -nan is a NaN with its sign bit set, as CPython makes it.
// Grammar of int() / numpy.int64(): [+-] digits, at most 4300 digits (CPython's limit for str -> int).
//
// Decimal -> binary64 is correctly rounded (round half to even), for any number of digits:
//   1. Clinger: mantissa below 2^53 and |exponent| <= 22 -- one exact IEEE multiplication or division.
//   2. Eisel-Lemire: the first 19 significant digits times a 128-bit power of five (libsvm_pow5.h); accepted only
//      when those bits decide the rounding, and with more than 19 digits only when the 19-digit prefix w and w + 1
//      round to the same double.
//   3. Otherwise exact: the candidate is moved one ulp at a time until the value lies between the halfway points
//      on either side of it, each comparison done on big integers (value digits x 10^E against halfway x 2^F).
//      Digits after the 768th only matter as "nonzero or not" (no halfway point has more than 768 significant
//      digits: (2^54 - 1) * 5^1075 is about 10^767.65), so they are replaced by a single 1 when any is nonzero.
#pragma once
#include <cstdint>

// A plain C++ build (g++) sees the CUDA qualifiers as nothing.  The no-inline attribute gets a name of its own:
// libstdc++ spells `__attribute__((__noinline__))`, which a `__noinline__` macro would break.
#ifdef __CUDACC__
#define ARB_SVM_NOINLINE __noinline__
#else
#define __host__
#define __device__
#define __forceinline__ inline
#define ARB_SVM_NOINLINE __attribute__((noinline))
#endif

#include "libsvm_pow5.h"

namespace arb {
namespace svm {

#ifdef __CUDACC__
__device__ const uint64_t kPow5Dev[ARB_POW5_Q_MAX - ARB_POW5_Q_MIN + 1][2] = ARB_POW5_ROWS;
#endif
static const uint64_t kPow5Host[ARB_POW5_Q_MAX - ARB_POW5_Q_MIN + 1][2] = ARB_POW5_ROWS;

__host__ __device__ __forceinline__ const uint64_t* pow5_row(int q) {
#ifdef __CUDA_ARCH__
  return kPow5Dev[q - ARB_POW5_Q_MIN];
#else
  return kPow5Host[q - ARB_POW5_Q_MIN];
#endif
}

// status of a numeral
enum { NUM_OK = 0, NUM_SYNTAX = 1, NUM_OVERFLOW = 2 };

constexpr int kPyIntMaxDigits = 4300;
constexpr int kMaxDigits = 768;                 // kept significant digits of the exact path (+ 1 sticky digit)
constexpr int kBigLimbs = 96;                   // 3072 bits: > 10^769 * 2^55 and > 2^55 * 5^1100
constexpr uint64_t kInfBits = 0x7ff0000000000000ull;
constexpr uint64_t kSignBit = 0x8000000000000000ull;

__host__ __device__ __forceinline__ bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
__host__ __device__ __forceinline__ uint8_t lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? c + 32 : c; }

__host__ __device__ __forceinline__ int clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
  return __clzll(static_cast<long long>(x));
#else
  return __builtin_clzll(x);
#endif
}

__host__ __device__ __forceinline__ void mul128(uint64_t a, uint64_t b, uint64_t* hi, uint64_t* lo) {
#ifdef __CUDA_ARCH__
  *lo = a * b;
  *hi = __umul64hi(a, b);
#else
  const unsigned __int128 p = static_cast<unsigned __int128>(a) * b;
  *lo = static_cast<uint64_t>(p);
  *hi = static_cast<uint64_t>(p >> 64);
#endif
}

__host__ __device__ __forceinline__ double bits_to_double(uint64_t b) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(static_cast<long long>(b));
#else
  double d;
  __builtin_memcpy(&d, &b, 8);
  return d;
#endif
}

// Consumes digits ( "_"? digits )* at s[*i]; returns how many digits (0 = none).  `fn(d)` sees each digit.
template <class Fn>
__host__ __device__ __forceinline__ int64_t scan_digits(const uint8_t* s, int64_t n, int64_t* i, Fn fn) {
  int64_t k = *i, cnt = 0;
  while (k < n) {
    if (is_digit(s[k])) {
      fn(s[k] - '0');
      ++cnt;
      ++k;
    } else if (s[k] == '_' && cnt > 0 && k + 1 < n && is_digit(s[k + 1])) {
      ++k;
    } else {
      break;
    }
  }
  *i = k;
  return cnt;
}

// int() / numpy.int64() of s[0, n): NUM_OK with *out set, NUM_SYNTAX, or NUM_OVERFLOW when the value is outside
// [lo, hi] (a C int for feature indices, int64 for qids).
__host__ __device__ __forceinline__ int parse_py_int(const uint8_t* s, int64_t n, int64_t lo, int64_t hi,
                                                     int64_t* out) {
  int64_t i = 0;
  bool neg = false;
  if (i < n && (s[i] == '+' || s[i] == '-')) neg = s[i++] == '-';
  uint64_t mag = 0;
  bool big = false;
  const uint64_t lim = neg ? static_cast<uint64_t>(-(lo + 1)) + 1 : static_cast<uint64_t>(hi);
  const int64_t nd = scan_digits(s, n, &i, [&](int d) {
    if (!big) {
      if (mag > (lim - d) / 10) big = true;
      else mag = mag * 10 + d;
    }
  });
  if (nd == 0 || i != n || nd > kPyIntMaxDigits) return NUM_SYNTAX;
  if (big) return NUM_OVERFLOW;
  *out = neg ? static_cast<int64_t>(0 - mag) : static_cast<int64_t>(mag);
  return NUM_OK;
}

// ---- exact path: little-endian 32-bit-limb big integers ---------------------------------------------------------
struct Big {
  uint32_t v[kBigLimbs];
  int n;
  bool overflow;
};

__host__ __device__ __forceinline__ void big_set(Big& b, uint64_t x) {
  b.n = 0;
  b.overflow = false;
  while (x) { b.v[b.n++] = static_cast<uint32_t>(x); x >>= 32; }
}

__host__ __device__ __forceinline__ void big_mul_add(Big& b, uint32_t m, uint32_t a) {
  uint64_t carry = a;
  for (int k = 0; k < b.n; ++k) {
    const uint64_t t = uint64_t(b.v[k]) * m + carry;
    b.v[k] = static_cast<uint32_t>(t);
    carry = t >> 32;
  }
  if (carry) {
    if (b.n < kBigLimbs) b.v[b.n++] = static_cast<uint32_t>(carry);
    else b.overflow = true;
  }
}

__host__ __device__ __forceinline__ void big_mul_pow5(Big& b, int64_t k) {
  for (; k >= 13; k -= 13) big_mul_add(b, 1220703125u, 0);     // 5^13
  uint32_t m = 1;
  for (; k > 0; --k) m *= 5;
  if (m != 1) big_mul_add(b, m, 0);
}

__host__ __device__ __forceinline__ void big_shl(Big& b, int64_t bits) {
  if (b.n == 0 || bits <= 0) return;
  const int64_t words = bits >> 5;
  const int sh = static_cast<int>(bits & 31);
  if (b.n + words + 1 > kBigLimbs) { b.overflow = true; return; }
  int n = b.n + static_cast<int>(words);
  b.v[n] = 0;
  for (int k = b.n - 1; k >= 0; --k) {
    const uint32_t x = b.v[k];
    if (sh) b.v[k + words + 1] |= x >> (32 - sh);
    b.v[k + words] = sh ? x << sh : x;
  }
  for (int k = 0; k < words; ++k) b.v[k] = 0;
  b.n = n + 1;
  while (b.n && b.v[b.n - 1] == 0) --b.n;
}

__host__ __device__ __forceinline__ int big_cmp(const Big& a, const Big& b) {
  if (a.n != b.n) return a.n < b.n ? -1 : 1;
  for (int k = a.n - 1; k >= 0; --k)
    if (a.v[k] != b.v[k]) return a.v[k] < b.v[k] ? -1 : 1;
  return 0;
}

// A parsed finite numeral: value = (its significant digits, read as an integer) * 10^e_last, where the digits are
// the digit characters of s[mant_beg, mant_end) after the leading zeros.
struct Decimal {
  uint64_t w;          // the first min(nd, 19) significant digits
  int64_t e10;         // exponent of w's last digit: value ~ w * 10^e10
  int64_t nd;          // significant digits
  bool truncated;      // a nonzero digit follows the first 19
  int64_t mant_beg, mant_end;
};

// the significant digits as a big integer D (at most kMaxDigits + 1 of them), value = D * 10^(*e_out)
__host__ __device__ __forceinline__ void big_from_digits(Big& D, const uint8_t* s, const Decimal& dec,
                                                         int64_t* e_out) {
  big_set(D, 0);
  int64_t kept = 0;
  bool started = false, sticky = false;
  uint32_t chunk = 0, scale = 1;
  for (int64_t k = dec.mant_beg; k < dec.mant_end; ++k) {
    if (!is_digit(s[k])) continue;
    const int d = s[k] - '0';
    if (!started && d == 0) continue;
    started = true;
    if (kept == kMaxDigits) { if (d) { sticky = true; break; } continue; }
    chunk = chunk * 10 + d;
    scale *= 10;
    ++kept;
    if (scale == 1000000000u) { big_mul_add(D, scale, chunk); chunk = 0; scale = 1; }
  }
  if (sticky) { chunk = chunk * 10 + 1; scale *= 10; }
  if (scale != 1) big_mul_add(D, scale, chunk);
  // dec.e10 is the exponent of the 19th digit (or of the last one when nd <= 19)
  const int64_t last_digit_exp = dec.e10 + (dec.nd > 19 ? 19 : dec.nd) - dec.nd;   // exponent of digit nd
  *e_out = last_digit_exp + (dec.nd - kept) - (sticky ? 1 : 0);
}

// halfway point between the adjacent doubles with bit patterns b and b + 1 (b < kInfBits): H * 2^F
__host__ __device__ __forceinline__ void halfway(uint64_t b, uint64_t* H, int64_t* F) {
  uint64_t m[2];
  int64_t e[2];
  for (int j = 0; j < 2; ++j) {
    const uint64_t x = b + j;
    const uint64_t ex = x >> 52, fr = x & ((1ull << 52) - 1);
    m[j] = ex ? (fr | (1ull << 52)) : fr;
    e[j] = ex ? int64_t(ex) - 1075 : -1074;
  }
  const int64_t lo = e[0] < e[1] ? e[0] : e[1];
  *H = (m[0] << (e[0] - lo)) + (m[1] << (e[1] - lo));
  *F = lo - 1;
}

// sign of (value - H * 2^F); *bad on big-integer overflow (never expected within the documented limits)
__host__ __device__ __forceinline__ int cmp_halfway(const uint8_t* s, const Decimal& dec, uint64_t H, int64_t F,
                                                    bool* bad) {
  Big L, R;
  int64_t E;
  big_from_digits(L, s, dec, &E);
  big_set(R, H);
  if (E >= 0) big_mul_pow5(L, E);
  else big_mul_pow5(R, -E);
  if (E - F >= 0) big_shl(L, E - F);
  else big_shl(R, F - E);
  if (L.overflow || R.overflow) *bad = true;
  return big_cmp(L, R);
}

// exact rounding starting from the candidate bit pattern b (magnitude); returns the correctly rounded pattern
static __host__ __device__ ARB_SVM_NOINLINE uint64_t exact_round(const uint8_t* s, const Decimal& dec, uint64_t b,
                                                                 bool* bad) {
  for (int iter = 0; iter < 64; ++iter) {
    uint64_t H;
    int64_t F;
    if (b < kInfBits) {
      halfway(b, &H, &F);
      const int c = cmp_halfway(s, dec, H, F, bad);
      if (c > 0 || (c == 0 && (b & 1))) { ++b; continue; }
    }
    if (b > 0) {
      halfway(b - 1, &H, &F);
      const int c = cmp_halfway(s, dec, H, F, bad);
      if (c < 0 || (c == 0 && (b & 1))) { --b; continue; }
    }
    return b;
  }
  *bad = true;
  return b;
}

// Eisel-Lemire for w * 10^q (w > 0): the bit pattern of a candidate, and whether the 128-bit product decides it.
__host__ __device__ __forceinline__ bool eisel_lemire(int64_t q, uint64_t w, uint64_t* bits) {
  if (q < ARB_POW5_Q_MIN) { *bits = 0; return true; }         // w * 10^q < 2^-1075: rounds to 0
  if (q > ARB_POW5_Q_MAX) { *bits = kInfBits; return true; }  // >= 10^309
  const int lz = clz64(w);
  w <<= lz;
  const uint64_t* t = pow5_row(static_cast<int>(q));
  uint64_t hi, lo;
  mul128(w, t[0], &hi, &lo);
  bool sure = true;
  if ((hi & 0x1FF) == 0x1FF) {          // the low word of the power of five may carry into the kept bits
    uint64_t hi2, lo2;
    mul128(w, t[1], &hi2, &lo2);
    lo += hi2;
    if (lo < hi2) ++hi;
    if ((hi & 0x1FF) == 0x1FF && lo == ~0ull) sure = false;
  }
  const int upper = static_cast<int>(hi >> 63);
  const int shift = upper + 9;
  uint64_t mant = hi >> shift;
  int64_t power2 = ((int64_t(152170 + 65536) * q) >> 16) + 63 + upper - lz + 1023;
  if (lo <= 1 && (mant << shift) == hi && (mant & 3) == 1) sure = false;   // at or next to a halfway point
  if (power2 <= 0) {                                                      // subnormal: confirmed exactly
    if (-power2 + 1 >= 64) { *bits = 0; return false; }
    mant >>= -power2 + 1;
    mant += mant & 1;
    mant >>= 1;
    *bits = mant;                       // (a carry into bit 52 is the smallest normal's pattern)
    return false;
  }
  mant += mant & 1;
  mant >>= 1;
  if (mant >= (2ull << 52)) { mant = 1ull << 52; ++power2; }
  mant &= ~(1ull << 52);
  if (power2 >= 0x7FF) { *bits = kInfBits; return false; }             // overflow: confirmed exactly
  *bits = (uint64_t(power2) << 52) | mant;
  return sure;
}

// float() of s[0, n): NUM_OK with *out set, or NUM_SYNTAX (NUM_OVERFLOW when the exact path ran out of room,
// which the documented limits rule out).
__host__ __device__ __forceinline__ int parse_py_float(const uint8_t* s, int64_t n, double* out) {
  int64_t i = 0;
  bool neg = false;
  if (i < n && (s[i] == '+' || s[i] == '-')) neg = s[i++] == '-';
  const uint64_t sign = neg ? kSignBit : 0;
  const int64_t rest = n - i;
  if (rest == 3 || rest == 8) {
    const char* names[3] = {"inf", "infinity", "nan"};
    for (int k = 0; k < 3; ++k) {
      int64_t len = 0;
      while (names[k][len]) ++len;
      if (len != rest) continue;
      bool eq = true;
      for (int64_t j = 0; j < len && eq; ++j) eq = lower(s[i + j]) == uint8_t(names[k][j]);
      if (eq) {
        *out = bits_to_double(sign | (k == 2 ? 0x7ff8000000000000ull : kInfBits));
        return NUM_OK;
      }
    }
  }
  Decimal dec;
  dec.w = 0;
  dec.nd = 0;
  dec.truncated = false;
  dec.mant_beg = i;
  auto digit = [&](int d) {
    if (dec.nd == 0 && d == 0) return;           // leading zeros
    if (dec.nd < 19) dec.w = dec.w * 10 + d;
    else if (d) dec.truncated = true;
    ++dec.nd;
  };
  const int64_t nint = scan_digits(s, n, &i, digit);
  int64_t nfrac = 0;
  if (i < n && s[i] == '.') {
    ++i;
    nfrac = scan_digits(s, n, &i, digit);
  }
  if (nint + nfrac == 0) return NUM_SYNTAX;
  dec.mant_end = i;
  int64_t exp = 0;
  if (i < n && (s[i] == 'e' || s[i] == 'E')) {
    ++i;
    bool eneg = false;
    if (i < n && (s[i] == '+' || s[i] == '-')) eneg = s[i++] == '-';
    // saturates: 10^12 already puts every value with fewer than 10^11 digits at 0 or inf
    const int64_t ne = scan_digits(s, n, &i, [&](int d) { if (exp < 1000000000000ll) exp = exp * 10 + d; });
    if (ne == 0) return NUM_SYNTAX;
    if (eneg) exp = -exp;
  }
  if (i != n) return NUM_SYNTAX;
  if (dec.w == 0) { *out = bits_to_double(sign); return NUM_OK; }
  dec.e10 = exp - nfrac + (dec.nd - (dec.nd < 19 ? dec.nd : 19));
  if (!dec.truncated && dec.w <= (1ull << 53) && dec.e10 >= -22 && dec.e10 <= 22) {   // Clinger
    const double p10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                            1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
    const double m = static_cast<double>(dec.w);
    double v;
#ifdef __CUDA_ARCH__
    v = dec.e10 >= 0 ? __dmul_rn(m, p10[dec.e10]) : __ddiv_rn(m, p10[-dec.e10]);
#else
    v = dec.e10 >= 0 ? m * p10[dec.e10] : m / p10[-dec.e10];
#endif
    *out = neg ? -v : v;
    return NUM_OK;
  }
  uint64_t b;
  bool sure = eisel_lemire(dec.e10, dec.w, &b);
  if (sure && dec.truncated) {
    uint64_t b1;
    sure = eisel_lemire(dec.e10, dec.w + 1, &b1) && b1 == b;
  }
  if (!sure) {
    bool bad = false;
    b = exact_round(s, dec, b, &bad);
    if (bad) return NUM_OVERFLOW;
  }
  *out = bits_to_double(sign | b);
  return NUM_OK;
}

// The float32 that sklearn + SlateStore store for a numeral: float32(float64(token)) -- rounded twice, first to
// float64 by float(), then to float32 by np.asarray(..., dtype=np.float32), which is not always the float32 nearest
// to the decimal value.  A NaN becomes the quiet float32 NaN with the same sign (x86 cvtsd2ss).  `densified`:
// feature values pass through scipy's toarray(), which adds them into a zero-filled array, so -0.0 becomes +0.0
// (labels are not densified and keep -0.0).
__host__ __device__ __forceinline__ uint32_t sklearn_f32_bits(double v, bool densified) {
  uint64_t b;
#ifdef __CUDA_ARCH__
  b = static_cast<uint64_t>(__double_as_longlong(v));
#else
  __builtin_memcpy(&b, &v, 8);
#endif
  const uint32_t sign = static_cast<uint32_t>(b >> 32) & 0x80000000u;
  if ((b & ~kSignBit) > kInfBits) return sign | 0x7fc00000u;      // NaN
  if ((b & ~kSignBit) == 0) return densified ? 0u : sign;          // +-0
  float f;
#ifdef __CUDA_ARCH__
  f = __double2float_rn(v);
  return static_cast<uint32_t>(__float_as_uint(f));
#else
  f = static_cast<float>(v);
  uint32_t r;
  __builtin_memcpy(&r, &f, 4);
  return r;
#endif
}

}  // namespace svm
}  // namespace arb
