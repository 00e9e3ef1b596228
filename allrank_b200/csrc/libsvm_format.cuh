// Numbers as sklearn.datasets.dump_svmlight_file writes them: Python's "%.16g" of a double and "%d" of an int64.
// Every function is __host__ __device__: the kernels of libsvm_write.cu call them per value, and arb_format_g16_host
// runs the same code on the CPU.  DESIGN.md section 12 states the exactness argument in full.
//
// "%.16g" (CPython: David Gay's dtoa, mode 2, 16 digits):
//   digits   D = v * 10^q rounded to an integer, half to even on the exact binary value, with q = 15 - E chosen so
//            that 10^15 <= D < 10^16 (E = the decimal exponent of the first digit); D = 10^16 after rounding is
//            10^15 with E + 1.
//   notation -4 <= E < 16: fixed, otherwise d.ddd e[+-]XX with at least two exponent digits; trailing zeros and a
//            trailing '.' are stripped.  -0.0 is "-0"; inf, -inf and nan (any sign) as Python prints them.
//
// Digit generation is integer-only.  v = m * 2^e (m < 2^53).  A 128-bit power of five T ~ 5^q * 2^s
// (libsvm_pow5.h) gives the 192-bit product X = m * T, and v * 10^q = X * 2^-(s - e - q): the integer part is D, the
// next 64 bits are the fraction F.
//   q in [0, 55]  5^q < 2^128, so T is exact and so is F: ties are decided on the exact product (the fast path is
//                 exact for every double from 1e-40 to 1e16, every float32 normal among them).
//   otherwise     T is within one unit of its last bit, so X is within m < 2^53 of m * 5^q * 2^s and F within
//                 2^-73 of the true fraction (s - e - q >= 71 + bitlen(m)).  The rounding is taken from F unless
//                 |F - 1/2| <= 2^-56; then exact_half compares v * 10^q with D + 1/2 on big integers.
// A misplaced E (the estimate from the binary exponent can be one too small) shows as D >= 10^16 and is redone with
// E + 1.  A product within 2^-73 of 10^15 or 10^16 can put D on the wrong side of the boundary, but rounding there
// gives the same 16 digits and exponent either way.
#pragma once
#include "libsvm_numeral.cuh"

namespace arb {
namespace svm {

constexpr int kFmtSlot = 24;                  // bytes that hold any output of format_g16 / format_i64
constexpr uint64_t kTen15 = 1000000000000000ull;
constexpr uint64_t kTen16 = 10000000000000000ull;

#ifdef __CUDACC__
__device__ const uint64_t kPow5ExtDev[ARB_POW5_EXT_Q_MAX - ARB_POW5_Q_MAX][2] = ARB_POW5_EXT_ROWS;
#endif
static const uint64_t kPow5ExtHost[ARB_POW5_EXT_Q_MAX - ARB_POW5_Q_MAX][2] = ARB_POW5_EXT_ROWS;

// the table row of 5^q for q in [ARB_POW5_Q_MIN, ARB_POW5_EXT_Q_MAX]
__host__ __device__ __forceinline__ const uint64_t* fmt_pow5_row(int q) {
  if (q <= ARB_POW5_Q_MAX) return pow5_row(q);
#ifdef __CUDA_ARCH__
  return kPow5ExtDev[q - ARB_POW5_Q_MAX - 1];
#else
  return kPow5ExtHost[q - ARB_POW5_Q_MAX - 1];
#endif
}

// bits [pos, pos + 64) of the 192-bit x2:x1:x0 (0 < pos < 192)
__host__ __device__ __forceinline__ uint64_t bits192(uint64_t x2, uint64_t x1, uint64_t x0, int pos) {
  if (pos >= 128) return x2 >> (pos - 128);
  if (pos >= 64) return pos == 64 ? x1 : (x1 >> (pos - 64)) | (x2 << (128 - pos));
  return (x0 >> pos) | (x1 << (64 - pos));
}

// sign of m * 2^e * 10^q - (D + 1/2), on big integers: m * 5^q * 2^(e+q+1) against 2D + 1
static __host__ __device__ ARB_SVM_NOINLINE int exact_half(uint64_t m, int e, int q, uint64_t D) {
  Big L, R;
  big_set(L, m);
  big_set(R, 2 * D + 1);
  if (q >= 0) big_mul_pow5(L, q);
  else big_mul_pow5(R, -q);
  const int k = e + q + 1;
  if (k >= 0) big_shl(L, k);
  else big_shl(R, -k);
  return big_cmp(L, R);
}

// 16 significant digits of finite v > 0 (bit pattern b): *D in [10^15, 10^16), *E the decimal exponent of its first
// digit
__host__ __device__ __forceinline__ void digits16(uint64_t b, uint64_t* D_out, int* E_out) {
  const int ex = static_cast<int>(b >> 52);
  const uint64_t fr = b & ((1ull << 52) - 1);
  const uint64_t m = ex ? fr | (1ull << 52) : fr;
  const int e = ex ? ex - 1075 : -1074;
  const int p2 = e + 63 - clz64(m);                    // floor(log2 v)
  int E = (p2 * 78913) >> 18;                          // floor(p2 * log10 2): the exponent, or one below it
  for (;;) {
    const int q = 15 - E;
    const uint64_t* T = fmt_pow5_row(q);
    const int s = 127 - ((((152170 + 65536) * q) >> 16) - q);    // T ~ 5^q * 2^s, 2^127 <= T < 2^128
    uint64_t h0, x0, h1, l1;
    mul128(m, T[1], &h0, &x0);
    mul128(m, T[0], &h1, &l1);
    const uint64_t x1 = l1 + h0;
    const uint64_t x2 = h1 + (x1 < l1);
    const int sh = s - e - q;                          // in [72, 131]
    uint64_t D = bits192(x2, x1, x0, sh);
    if (D >= kTen16) { ++E; continue; }
    const uint64_t F = bits192(x2, x1, x0, sh - 64);
    bool up;
    if (q >= 0 && q <= 55) {                           // exact product
      const int low = sh - 64;                         // bits below F
      const bool rest = low >= 128 ? (x0 | x1 | (x2 & ((1ull << (low - 128)) - 1))) != 0
                                   : low >= 64 ? (x0 | (x1 & ((1ull << (low - 64)) - 1))) != 0
                                               : (x0 & ((1ull << low) - 1)) != 0;
      const uint64_t half = 1ull << 63;
      up = F > half || (F == half && (rest || (D & 1)));
    } else {
      const uint64_t half = 1ull << 63;
      const uint64_t dist = F > half ? F - half : half - F;
      if (dist <= 256) {
        const int c = exact_half(m, e, q, D);
        up = c > 0 || (c == 0 && (D & 1));
      } else {
        up = F > half;
      }
    }
    D += up;
    if (D == kTen16) { D = kTen15; ++E; }
    *D_out = D;
    *E_out = E;
    return;
  }
}

// "%d" of an unsigned magnitude into out; returns the length
__host__ __device__ __forceinline__ int format_u64(uint64_t u, char* out) {
  char t[20];
  int n = 0;
  do { t[n++] = static_cast<char>('0' + u % 10); u /= 10; } while (u);
  for (int k = 0; k < n; ++k) out[k] = t[n - 1 - k];
  return n;
}

// "%d" of an int64 into out (at most 20 bytes); returns the length
__host__ __device__ __forceinline__ int format_i64(int64_t v, char* out) {
  if (v < 0) {
    out[0] = '-';
    return 1 + format_u64(0 - static_cast<uint64_t>(v), out + 1);
  }
  return format_u64(static_cast<uint64_t>(v), out);
}

// Python's "%.16g" % v into out (at most 23 bytes); returns the length
__host__ __device__ __forceinline__ int format_g16(double v, char* out) {
  uint64_t b;
#ifdef __CUDA_ARCH__
  b = static_cast<uint64_t>(__double_as_longlong(v));
#else
  __builtin_memcpy(&b, &v, 8);
#endif
  int n = 0;
  const uint64_t mag = b & ~kSignBit;
  if (mag > kInfBits) { out[0] = 'n'; out[1] = 'a'; out[2] = 'n'; return 3; }
  if (b >> 63) out[n++] = '-';
  if (mag == kInfBits) { out[n] = 'i'; out[n + 1] = 'n'; out[n + 2] = 'f'; return n + 3; }
  if (mag == 0) { out[n] = '0'; return n + 1; }
  uint64_t D;
  int E;
  digits16(mag, &D, &E);
  char d[16];
  for (int k = 15; k >= 0; --k) { d[k] = static_cast<char>('0' + D % 10); D /= 10; }
  int nd = 16;
  while (nd > 1 && d[nd - 1] == '0') --nd;
  if (E >= 0 && E < 16) {
    for (int k = 0; k <= E; ++k) out[n++] = d[k];
    if (nd > E + 1) {
      out[n++] = '.';
      for (int k = E + 1; k < nd; ++k) out[n++] = d[k];
    }
  } else if (E < 0 && E >= -4) {
    out[n++] = '0';
    out[n++] = '.';
    for (int k = 0; k < -E - 1; ++k) out[n++] = '0';
    for (int k = 0; k < nd; ++k) out[n++] = d[k];
  } else {
    out[n++] = d[0];
    if (nd > 1) {
      out[n++] = '.';
      for (int k = 1; k < nd; ++k) out[n++] = d[k];
    }
    out[n++] = 'e';
    out[n++] = E < 0 ? '-' : '+';
    const int a = E < 0 ? -E : E;
    if (a >= 100) out[n++] = static_cast<char>('0' + a / 100);
    out[n++] = static_cast<char>('0' + a / 10 % 10);
    out[n++] = static_cast<char>('0' + a % 10);
  }
  return n;
}

}  // namespace svm
}  // namespace arb
