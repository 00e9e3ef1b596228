// Dense rows -> the LibSVM text sklearn.datasets.dump_svmlight_file(X, y, f, zero_based, query_id) writes, on the
// device.  DESIGN.md section 12.
//
//   check_kernel           any NaN or +-inf in X or y sets *bad (every writer stores the same 1)
//   length_kernel          one warp per row, lanes over columns: the bytes of the row's line
//   exclusive_scan_kernel  (libsvm_scan.cuh) one block: the lengths become row offsets inside the chunk, and the
//                          chunk's byte total
//   emit_kernel            one warp per row: the label, the qid and, lane by lane, " j:v" for every non-zero value
//                          at the offsets of a warp scan of the token lengths, then the '\n'
// A line is  label[ qid:Q] j:v j:v ...\n  with exactly one space after the label (or the qid) even when the row has
// no non-zero value: sklearn writes "%s qid:%d %s\n" with the joined tokens as the last %s.  Numbers are formatted by
// libsvm_format.cuh.  Where each byte goes follows from the lengths and the scan alone.
#include <cstdint>
#include <cuda_runtime.h>

#include "common.h"
#include "libsvm_format.cuh"
#include "libsvm_scan.cuh"

namespace arb {

constexpr int WR_WARPS = 8;             // warps per block of the row kernels

// X element k of a row as the formatter sees it: "%.16g" of the value widened to double, or "%d"
struct XVal {
  double f;
  long long i;
};

__device__ __forceinline__ bool x_nonzero(const void* X, int kind, long long at, XVal* v) {
  if (kind == ARB_SVMW_F32) {
    const float x = static_cast<const float*>(X)[at];
    v->f = x;
    return x != 0.f;
  }
  if (kind == ARB_SVMW_F64) {
    v->f = static_cast<const double*>(X)[at];
    return v->f != 0.0;
  }
  v->i = static_cast<const long long*>(X)[at];
  return v->i != 0;
}

// " j:v" into t; returns its length (at most 1 + 20 + 1 + 24 bytes)
__device__ __forceinline__ int format_token(long long j, int kind, const XVal& v, char* t) {
  t[0] = ' ';
  int n = 1 + svm::format_i64(j, t + 1);
  t[n++] = ':';
  n += kind == ARB_SVMW_I64 ? svm::format_i64(v.i, t + n) : svm::format_g16(v.f, t + n);
  return n;
}

// label and " qid:Q" into t; returns the length (at most 24 + 25 bytes)
__device__ __forceinline__ int format_head(const void* y, int y_kind, const long long* qid, long long row, char* t) {
  int n = y_kind == ARB_SVMW_I64 ? svm::format_i64(static_cast<const long long*>(y)[row], t)
                                 : svm::format_g16(static_cast<const double*>(y)[row], t);
  if (qid) {
    t[n++] = ' '; t[n++] = 'q'; t[n++] = 'i'; t[n++] = 'd'; t[n++] = ':';
    n += svm::format_i64(qid[row], t + n);
  }
  return n;
}

__global__ void check_kernel(const void* __restrict__ X, int x_kind, long long n_x, const void* __restrict__ y,
                             int y_kind, long long n_y, int* __restrict__ bad) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  bool b = false;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x_kind == ARB_SVMW_F32)
    for (long long k = t0; k < n_x; k += stride) b |= !isfinite(static_cast<const float*>(X)[k]);
  else if (x_kind == ARB_SVMW_F64)
    for (long long k = t0; k < n_x; k += stride) b |= !isfinite(static_cast<const double*>(X)[k]);
  if (y_kind == ARB_SVMW_F64)
    for (long long k = t0; k < n_y; k += stride) b |= !isfinite(static_cast<const double*>(y)[k]);
  if (b) *bad = 1;
}

// len[r - r0] = bytes of row r's line, r in [r0, r1)
__global__ void __launch_bounds__(WR_WARPS * 32) length_kernel(const void* __restrict__ X, int x_kind, long long F,
                                                               const void* __restrict__ y, int y_kind,
                                                               const long long* __restrict__ qid, int one_based,
                                                               long long r0, long long r1,
                                                               long long* __restrict__ len) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * WR_WARPS;
  for (long long row = r0 + (long long)blockIdx.x * WR_WARPS + (threadIdx.x >> 5); row < r1; row += warps) {
    long long bytes = 0;
    int ntok = 0;
    for (long long k = lane; k < F; k += 32) {
      XVal v;
      if (!x_nonzero(X, x_kind, row * F + k, &v)) continue;
      char t[48];
      bytes += format_token(k + one_based, x_kind, v, t);
      ++ntok;
    }
    for (int o = 16; o; o >>= 1) {
      bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
      ntok += __shfl_xor_sync(0xffffffffu, ntok, o);
    }
    if (lane == 0) {
      char t[56];
      len[row - r0] = format_head(y, y_kind, qid, row, t) + bytes + (ntok == 0) + 1;
    }
  }
}

__global__ void __launch_bounds__(WR_WARPS * 32) emit_kernel(const void* __restrict__ X, int x_kind, long long F,
                                                             const void* __restrict__ y, int y_kind,
                                                             const long long* __restrict__ qid, int one_based,
                                                             long long r0, long long r1,
                                                             const long long* __restrict__ off,
                                                             uint8_t* __restrict__ text) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * WR_WARPS;
  for (long long row = r0 + (long long)blockIdx.x * WR_WARPS + (threadIdx.x >> 5); row < r1; row += warps) {
    uint8_t* out = text + off[row - r0];
    long long pos;
    {
      char t[56];
      const int n = format_head(y, y_kind, qid, row, t);     // every lane: the same length
      if (lane == 0)
        for (int k = 0; k < n; ++k) out[k] = t[k];
      pos = n;
    }
    bool any = false;
    for (long long k0 = 0; k0 < F; k0 += 32) {
      const long long k = k0 + lane;
      char t[48];
      int n = 0;
      XVal v;
      if (k < F && x_nonzero(X, x_kind, row * F + k, &v)) n = format_token(k + one_based, x_kind, v, t);
      int incl = n;
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
      }
      for (int b = 0; b < n; ++b) out[pos + incl - n + b] = t[b];
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      any |= total != 0;
      pos += total;
    }
    if (lane == 0) {
      if (!any) out[pos++] = ' ';
      out[pos] = '\n';
    }
  }
}

__global__ void format_g16_kernel(const double* __restrict__ v, long long n, char* __restrict__ slots) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    char t[svm::kFmtSlot];
    const int len = svm::format_g16(v[i], t);
    char* s = slots + i * svm::kFmtSlot;
    for (int k = 0; k < svm::kFmtSlot; ++k) s[k] = k < len ? t[k] : 0;
  }
}

}  // namespace arb

using namespace arb;

static int row_grid(long long rows) {
  const long long want = (rows + WR_WARPS - 1) / WR_WARPS;
  const long long cap = (long long)sm_count() * 16;
  return int(want < cap ? (want > 0 ? want : 1) : cap);
}

static bool bad_kinds(int x_kind, int y_kind) {
  return (x_kind != ARB_SVMW_F32 && x_kind != ARB_SVMW_F64 && x_kind != ARB_SVMW_I64) ||
         (y_kind != ARB_SVMW_F64 && y_kind != ARB_SVMW_I64);
}

extern "C" int32_t arb_svm_write_check(const void* X, int32_t x_kind, int64_t n_x, const void* y, int32_t y_kind,
                                       int64_t n_y, int32_t* bad, void* stream) {
  if (!X || !y || !bad || n_x < 0 || n_y < 0 || bad_kinds(x_kind, y_kind)) {
    arb_set_error("arb_svm_write_check: null pointer, negative size or unknown dtype");
    return ARB_E_INVALID_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(bad, 0, sizeof(int32_t), st) != cudaSuccess) {
    cudaGetLastError();
    arb_set_error("arb_svm_write_check: cudaMemsetAsync failed");
    return ARB_E_CUDA;
  }
  const long long n = n_x > n_y ? n_x : n_y;
  const long long want = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  const int grid = int(want < cap ? (want > 0 ? want : 1) : cap);
  return launch(check_kernel, dim3(grid), dim3(256), 0, st, false, X, (int)x_kind, (long long)n_x, y, (int)y_kind,
                (long long)n_y, reinterpret_cast<int*>(bad));
}

extern "C" int32_t arb_svm_write_chunk(const void* X, int32_t x_kind, int64_t n_features, const void* y,
                                       int32_t y_kind, const int64_t* qid, int32_t one_based, int64_t r0, int64_t r1,
                                       int64_t* offsets, uint8_t* text, void* stream) {
  if (!X || !y || !offsets || n_features <= 0 || r0 < 0 || r1 <= r0 || (one_based != 0 && one_based != 1) ||
      bad_kinds(x_kind, y_kind)) {
    arb_set_error("arb_svm_write_chunk: null pointer, empty chunk, n_features <= 0 or unknown dtype");
    return ARB_E_INVALID_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* q = reinterpret_cast<const long long*>(qid);
  long long* off = reinterpret_cast<long long*>(offsets);
  const int grid = row_grid(r1 - r0);
  if (!text) {
    if (int rc = launch(length_kernel, dim3(grid), dim3(WR_WARPS * 32), 0, st, false, X, (int)x_kind,
                        (long long)n_features, y, (int)y_kind, q, (int)one_based, (long long)r0, (long long)r1, off))
      return rc;
    return launch(exclusive_scan_kernel, dim3(1), dim3(SCAN_THREADS), 0, st, false, off, (long long)(r1 - r0),
                  off + (r1 - r0));
  }
  return launch(emit_kernel, dim3(grid), dim3(WR_WARPS * 32), 0, st, false, X, (int)x_kind, (long long)n_features, y,
                (int)y_kind, q, (int)one_based, (long long)r0, (long long)r1, static_cast<const long long*>(off), text);
}

extern "C" int32_t arb_format_g16(const double* values, int64_t n, char* slots, void* stream) {
  if (!values || !slots || n <= 0) {
    arb_set_error("arb_format_g16: null pointer or n <= 0");
    return ARB_E_INVALID_ARG;
  }
  const long long want = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  const int grid = int(want < cap ? want : cap);
  return launch(format_g16_kernel, dim3(grid), dim3(256), 0, static_cast<cudaStream_t>(stream), false, values,
                (long long)n, slots);
}

extern "C" int32_t arb_format_g16_host(const double* values, int64_t n, char* slots) {
  if (!values || !slots || n < 0) {
    arb_set_error("arb_format_g16_host: null pointer or n < 0");
    return ARB_E_INVALID_ARG;
  }
  for (int64_t i = 0; i < n; ++i) {
    char* s = slots + i * svm::kFmtSlot;
    const int len = svm::format_g16(values[i], s);
    for (int k = len; k < svm::kFmtSlot; ++k) s[k] = 0;
  }
  return ARB_OK;
}
