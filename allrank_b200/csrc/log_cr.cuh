// Correctly rounded natural logarithm of a double (round to nearest, ties to even), __host__ __device__: the
// normalisation kernels (normalize.cu) call it per value and arb_log_cr_host runs the same code on the CPU.
// DESIGN.md section 13 gives the error bounds in full.
//
// Reduction: x = 2^e * m with m in [sqrt(1/2), sqrt(2)], m = M * 2^-52 or M * 2^-53 for the 53-bit integer M of x
// (subnormals are first scaled by 2^54).  log x = e * ln2 + 2 atanh(s) with s = (m - 1) / (m + 1), |s| < 0.1716:
//   2 atanh(s) = 2 s * T(u),  T(u) = sum_k u^k / (2k + 1),  u = s^2 < 0.0295.
// Ziv's scheme:
//   fast phase      double-double: s by one correction of the quotient, T by Horner over double-double constants
//                   (K = 20 terms), then e * ln2 added from a three-part ln2.  Relative error < 2^-100.7; the
//                   result is returned when the interval yh + yl +- 2^-94 |yh| rounds to yh.
//   accurate phase  two's-complement fixed point with 256 fraction bits: s and 1/(2k+1) by exact long division,
//                   T by Horner with as many terms as u needs, ln2 to 256 bits.  Absolute error < 2^-237.9, so
//                   relative < 2^-183 (|log x| >= 2^-53.0 for x != 1).  The result is the common rounding of
//                   Y - 2^-236 and Y + 2^-236; if they differ, `path` reports LOG_CR_FAILED.
// Every floating-point operation is spelled __dadd_rn / __dmul_rn / __fma_rn on the device, so nvcc's contraction
// cannot change a bit between the device build and the host build.
#pragma once
#include <cmath>
#include <cstdint>

namespace arb {
namespace lcr {

enum { LOG_CR_FAST = 0, LOG_CR_ACCURATE = 1, LOG_CR_FAILED = 2 };

__host__ __device__ __forceinline__ double add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ double mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ double fma_rn(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rn(a, b, c);
#else
  return std::fma(a, b, c);
#endif
}
__host__ __device__ __forceinline__ uint64_t bits_of(double x) {
#ifdef __CUDA_ARCH__
  return static_cast<uint64_t>(__double_as_longlong(x));
#else
  uint64_t b;
  __builtin_memcpy(&b, &x, 8);
  return b;
#endif
}
__host__ __device__ __forceinline__ double from_bits(uint64_t b) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double(static_cast<long long>(b));
#else
  double x;
  __builtin_memcpy(&x, &b, 8);
  return x;
#endif
}
__host__ __device__ __forceinline__ uint64_t mulhi64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return static_cast<uint64_t>((static_cast<unsigned __int128>(a) * b) >> 64);
#endif
}
// 2^k for k in [-1022, 1023], exactly
__host__ __device__ __forceinline__ double pow2(int k) { return from_bits(static_cast<uint64_t>(k + 1023) << 52); }

// ---- double-double -------------------------------------------------------------------------------------------------
struct DD { double h, l; };

__host__ __device__ __forceinline__ DD fast_two_sum(double a, double b) {   // |a| >= |b| or a == 0
  const double s = add(a, b);
  return {s, sub(b, sub(s, a))};
}
__host__ __device__ __forceinline__ DD two_sum(double a, double b) {
  const double s = add(a, b), bb = sub(s, a);
  return {s, add(sub(a, sub(s, bb)), sub(b, bb))};
}
// AccurateDWPlusDW: relative error <= 3 * 2^-106
__host__ __device__ __forceinline__ DD dd_add(DD a, DD b) {
  DD s = two_sum(a.h, b.h);
  const DD t = two_sum(a.l, b.l);
  s = fast_two_sum(s.h, add(s.l, t.h));
  return fast_two_sum(s.h, add(s.l, t.l));
}
// DWTimesDW with FMA: relative error <= 7 * 2^-106
__host__ __device__ __forceinline__ DD dd_mul(DD a, DD b) {
  const double p = mul(a.h, b.h);
  double e = fma_rn(a.h, b.h, -p);
  e = fma_rn(a.h, b.l, e);
  e = fma_rn(a.l, b.h, e);
  return fast_two_sum(p, e);
}

// 1/(2k+1) for k = 1..20 as double-doubles (hi = RN(c), lo = RN(c - hi))
#define ARB_LOG_CR_COEFFS                                                                                     \
  {{0x1.5555555555555p-2, 0x1.5555555555555p-56},  {0x1.999999999999ap-3, -0x1.999999999999ap-57},            \
   {0x1.2492492492492p-3, 0x1.2492492492492p-57},  {0x1.c71c71c71c71cp-4, 0x1.c71c71c71c71cp-58},              \
   {0x1.745d1745d1746p-4, -0x1.745d1745d1746p-59}, {0x1.3b13b13b13b14p-4, -0x1.3b13b13b13b14p-58},             \
   {0x1.1111111111111p-4, 0x1.1111111111111p-60},  {0x1.e1e1e1e1e1e1ep-5, 0x1.e1e1e1e1e1e1ep-61},              \
   {0x1.af286bca1af28p-5, 0x1.af286bca1af28p-59},  {0x1.8618618618618p-5, 0x1.8618618618618p-59},              \
   {0x1.642c8590b2164p-5, 0x1.642c8590b2164p-60},  {0x1.47ae147ae147bp-5, -0x1.eb851eb851eb8p-61},             \
   {0x1.2f684bda12f68p-5, 0x1.2f684bda12f68p-59},  {0x1.1a7b9611a7b96p-5, 0x1.1a7b9611a7b96p-61},              \
   {0x1.0842108421084p-5, 0x1.0842108421084p-60},  {0x1.f07c1f07c1f08p-6, -0x1.f07c1f07c1f08p-61},             \
   {0x1.d41d41d41d41dp-6, 0x1.0750750750750p-60},  {0x1.bacf914c1bad0p-6, -0x1.bacf914c1bad0p-60},             \
   {0x1.a41a41a41a41ap-6, 0x1.0690690690690p-60},  {0x1.8f9c18f9c18fap-6, -0x1.f3831f3831f38p-61}}
constexpr int kFastTerms = 20;
#ifdef __CUDACC__
__device__ const double kCoeffDev[kFastTerms][2] = ARB_LOG_CR_COEFFS;
#endif
static const double kCoeffHost[kFastTerms][2] = ARB_LOG_CR_COEFFS;

// ln2 = kLn2Hi + kLn2Mid + kLn2Lo + O(2^-156); kLn2Hi has 42 significant bits, so e * kLn2Hi is exact for |e| < 2^11
constexpr double kLn2Hi = 0x1.62e42fefa3800p-1;
constexpr double kLn2Mid = 0x1.ef35793c76730p-45;
constexpr double kLn2Lo = 0x1.f97b57a079a19p-103;
constexpr uint64_t kSqrt2M = 0x16a09e667f3bccull;        // floor(sqrt(2) * 2^52): m = M * 2^-52 when M <= this

// ---- 256-bit fixed point (accurate phase) ------------------------------------------------------------------------
// Value = (w[4] w[3] w[2] w[1] w[0] as a two's-complement 320-bit integer) * 2^-256; w[4] holds the integer part.
struct Fx { uint64_t w[5]; };

__host__ __device__ __forceinline__ Fx fx_zero() { return Fx{{0, 0, 0, 0, 0}}; }

__host__ __device__ inline Fx fx_add(const Fx& a, const Fx& b) {
  Fx r;
  uint64_t c = 0;
  for (int i = 0; i < 5; ++i) {
    const uint64_t s = a.w[i] + b.w[i];
    const uint64_t t = s + c;
    c = (s < a.w[i]) | (t < s);
    r.w[i] = t;
  }
  return r;
}

__host__ __device__ inline Fx fx_neg(const Fx& a) {
  Fx r;
  uint64_t c = 1;
  for (int i = 0; i < 5; ++i) {
    r.w[i] = ~a.w[i] + c;
    c = c && r.w[i] == 0;
  }
  return r;
}

// num / den truncated to 256 fraction bits (0 < den < 2^55, num < 2^64)
__host__ __device__ inline Fx fx_div(uint64_t num, uint64_t den) {
  Fx r = fx_zero();
  r.w[4] = num / den;
  uint64_t rem = num % den;
  const bool small = den < (1ull << 32);
  const int step = small ? 32 : 8;
  for (int bit = 256 - step; bit >= 0; bit -= step) {
    rem <<= step;
    const uint64_t q = rem / den;
    rem -= q * den;
    r.w[bit >> 6] |= q << (bit & 63);
  }
  return r;
}

// a * b truncated to 256 fraction bits, for a, b >= 0
__host__ __device__ inline Fx fx_mul(const Fx& a, const Fx& b) {
  uint64_t p[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 5; ++i) {
    uint64_t carry = 0;
    for (int j = 0; j < 5; ++j) {
      const uint64_t lo = a.w[i] * b.w[j], hi = mulhi64(a.w[i], b.w[j]);
      uint64_t s = p[i + j] + lo;
      uint64_t c1 = s < lo;
      const uint64_t s2 = s + carry;
      c1 += s2 < s;
      p[i + j] = s2;
      carry = hi + c1;
    }
    for (int k = i + 5; k < 10 && carry; ++k) {
      p[k] += carry;
      carry = p[k] < carry;
    }
  }
  return Fx{{p[4], p[5], p[6], p[7], p[8]}};
}

// a * k exactly, for a >= 0 and 0 <= k < 2^32
__host__ __device__ inline Fx fx_mul_small(const Fx& a, uint64_t k) {
  Fx r;
  uint64_t carry = 0;
  for (int i = 0; i < 5; ++i) {
    const uint64_t lo = a.w[i] * k, hi = mulhi64(a.w[i], k);
    const uint64_t s = lo + carry;
    r.w[i] = s;
    carry = hi + (s < lo);
  }
  return r;
}

// bits [pos, pos + 64) of a non-negative Fx as an integer (bits above 319 read as 0)
__host__ __device__ __forceinline__ uint64_t fx_bits(const Fx& a, int pos) {
  const int i = pos >> 6, o = pos & 63;
  const uint64_t lo = i < 5 ? a.w[i] : 0, hi = i + 1 < 5 ? a.w[i + 1] : 0;
  return o ? (lo >> o) | (hi << (64 - o)) : lo;
}

// round-to-nearest-even of a, for 2^-60 <= |a| < 2^62
__host__ __device__ inline double fx_to_double(Fx a) {
  const bool negative = a.w[4] >> 63;
  if (negative) a = fx_neg(a);
  int top = 4;
  while (top > 0 && a.w[top] == 0) --top;
  int hb = 64 * top + 63;
  while (!((a.w[top] >> (hb & 63)) & 1u)) --hb;
  const int shift = hb - 52;                                 // >= 256 - 60 - 52 > 0
  uint64_t mant = fx_bits(a, shift) & ((1ull << 53) - 1);
  const bool round = (fx_bits(a, shift - 1) & 1u) != 0;
  bool sticky = false;
  for (int b = 0; b < shift - 1; b += 64) {
    const int n = shift - 1 - b < 64 ? shift - 1 - b : 64;
    sticky |= (fx_bits(a, b) & (n == 64 ? ~0ull : (1ull << n) - 1)) != 0;
  }
  if (round && (sticky || (mant & 1u))) ++mant;
  const double v = mul(static_cast<double>(mant), pow2(shift - 256));   // exact: mant <= 2^53, no under/overflow
  return negative ? -v : v;
}

__host__ __device__ inline double log_accurate(uint64_t M, int e, bool halve, int* path) {
  const uint64_t unit = halve ? (1ull << 53) : (1ull << 52);
  const bool neg_s = M < unit;
  const Fx s = fx_div(neg_s ? unit - M : M - unit, M + unit);        // |s|
  const Fx u = fx_mul(s, s);
  // terms: with u < 2^-z, u^(K+1) / (1 - u) < 2^-238 once z (K + 1) >= 239
  int z = 0;
  for (int bit = 255; bit >= 0 && !((u.w[bit >> 6] >> (bit & 63)) & 1u); --bit) ++z;
  int K = z >= 239 ? 0 : (239 + z - 1) / z - 1;
  Fx T = fx_div(1, 2 * K + 1);
  for (int k = K - 1; k >= 0; --k) T = fx_add(fx_div(1, 2 * k + 1), fx_mul(u, T));
  Fx L = fx_mul(s, T);
  L = fx_add(L, L);
  if (neg_s) L = fx_neg(L);
  if (e) {
    const Fx ln2 = Fx{{0x8a0d175b8baafa2bull, 0x40f343267298b62dull, 0xc9e3b39803f2f6afull, 0xb17217f7d1cf79abull,
                       0}};                                          // floor(ln2 * 2^256)
    const Fx eln2 = fx_mul_small(ln2, static_cast<uint64_t>(e < 0 ? -e : e));
    L = fx_add(L, e < 0 ? fx_neg(eln2) : eln2);
  }
  Fx d = fx_zero();
  d.w[0] = 1ull << 20;                                               // 2^-236
  const double lo = fx_to_double(fx_add(L, fx_neg(d))), hi = fx_to_double(fx_add(L, d));
  *path = lo == hi ? LOG_CR_ACCURATE : LOG_CR_FAILED;
  return hi;
}

// log(x) correctly rounded; *path = LOG_CR_FAST, LOG_CR_ACCURATE or LOG_CR_FAILED (the accurate phase could not
// decide the rounding: never observed, and the caller must not use the result)
__host__ __device__ inline double log_cr(double x, bool force_accurate, int* path) {
  *path = LOG_CR_FAST;
  uint64_t b = bits_of(x);
  if (x != x) return x;                                              // NaN (quiet, as the operand)
  if (x == 0.0) return -INFINITY;
  if (b >> 63) return from_bits(0x7ff8000000000000ull);              // negative: NaN
  if (b == 0x7ff0000000000000ull) return x;                          // +inf
  if (x == 1.0) return 0.0;
  int E;
  if ((b >> 52) == 0) {                                              // subnormal: scale by 2^54
    b = bits_of(mul(x, 0x1p54));
    E = static_cast<int>(b >> 52) - 1075 - 54;
  } else {
    E = static_cast<int>(b >> 52) - 1075;
  }
  const uint64_t M = (b & ((1ull << 52) - 1)) | (1ull << 52);
  const bool halve = M > kSqrt2M;
  const int e = E + 52 + halve;
  if (force_accurate) return log_accurate(M, e, halve, path);

  const double m = mul(static_cast<double>(M), halve ? 0x1p-53 : 0x1p-52);
  const double num = sub(m, 1.0);                                    // exact (Sterbenz)
  const DD den = two_sum(m, 1.0);                                    // exact
  const double sh = div(num, den.h);
  const double r = fma_rn(-sh, den.h, num);                          // exact remainder
  const DD s = fast_two_sum(sh, div(fma_rn(-sh, den.l, r), den.h));
  const DD u = dd_mul(s, s);
#ifdef __CUDA_ARCH__
  const double(*C)[2] = kCoeffDev;
#else
  const double(*C)[2] = kCoeffHost;
#endif
  DD T = {C[kFastTerms - 1][0], C[kFastTerms - 1][1]};
  for (int k = kFastTerms - 2; k >= 0; --k) T = dd_add(DD{C[k][0], C[k][1]}, dd_mul(u, T));
  T = dd_add(DD{1.0, 0.0}, dd_mul(u, T));
  DD y = dd_mul(s, T);
  y = {mul(y.h, 2.0), mul(y.l, 2.0)};
  if (e) {
    const double ed = static_cast<double>(e);
    const double p = mul(ed, kLn2Mid);
    const double pe = fma_rn(ed, kLn2Mid, -p);
    y = dd_add(y, DD{add(pe, mul(ed, kLn2Lo)), 0.0});
    y = dd_add(y, DD{p, 0.0});
    y = dd_add(y, DD{mul(ed, kLn2Hi), 0.0});                         // exact product
  }
  // y.h is the rounding of every value within |y.l| + 2^-95 |y.h| of y.h + y.l when that reach stays inside the
  // half-gap to the neighbour on y.l's side (a quarter ulp below a power of two)
  const uint64_t yb = bits_of(y.h) & 0x7fffffffffffffffull;
  const double ulp = pow2(static_cast<int>(yb >> 52) - 1023 - 52);
  const bool toward_zero = (y.l < 0) != (y.h < 0) && y.l != 0.0;
  const double gap = toward_zero && (yb & ((1ull << 52) - 1)) == 0 ? mul(ulp, 0.25) : mul(ulp, 0.5);
  const double reach = add(fabs(y.l), mul(fabs(y.h), 0x1p-94));   // 2^-94 |y.h| > 2^-100.7 |y|
  if (reach < gap) return y.h;
  return log_accurate(M, e, halve, path);
}

}  // namespace lcr
}  // namespace arb
