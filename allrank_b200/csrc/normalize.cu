// reproducibility/normalize_features.py on the device: per column of a dense row-major float64 role [rows, F],
// optional negation, log(v + 0.01) correctly rounded (log_cr.cuh), and standardisation with the train role's
// np.mean / np.std, bit for bit as numpy computes them.  DESIGN.md section 13.
//
//   sign_flags_kernel   per column: does any (negated) value fail v >= 0?  Integer atomicOr: order-free.
//   transform_a_kernel  in place: negate, then log_cr(v + 0.01), per column mask.
//   leaf_kernel         numpy's pairwise_sum leaves (8 to 128 rows, or the whole column below 8) for every column,
//                       lanes across columns so that a warp reads 32 consecutive doubles of a row; SQUARES sums
//                       (v - mean)^2 with both operations rounded on their own.
//   combine_kernel      one level of the fixed combination tree: node = left + right.
//   finish_kernel       0.0 + root (np.add.reduce's start), / n, and sqrt for the std.
//   transform_b_kernel  in place: (v - mean) / (std + 1e-6) below the train role's width, 0 beyond it.
// The tree (leaves, then internal nodes level by level, root last) is numpy's recursion, laid out by the caller; the
// result does not depend on the grid.
#include <cstdint>
#include <cuda_runtime.h>

#include "common.h"
#include "log_cr.cuh"

namespace arb {

constexpr int NZ_COLS = 32;     // lanes across columns
constexpr int NZ_ROWS = 8;      // rows (or leaves) per block step

// numpy's pairwise_sum of n <= 128 elements get(0 .. n-1) (n < 8: in order from -0.0; else eight accumulators)
template <class Get>
__host__ __device__ __forceinline__ double pairwise_leaf(const Get& get, long long n) {
  if (n < 8) {
    double res = -0.0;
    for (long long i = 0; i < n; ++i) res = lcr::add(res, get(i));
    return res;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = get(j);
  long long i = 8;
  for (; i < n - (n % 8); i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = lcr::add(r[j], get(i + j));
  }
  double res = lcr::add(lcr::add(lcr::add(r[0], r[1]), lcr::add(r[2], r[3])),
                        lcr::add(lcr::add(r[4], r[5]), lcr::add(r[6], r[7])));
  for (; i < n; ++i) res = lcr::add(res, get(i));
  return res;
}

struct StridedGet {
  const double* a;
  long long stride;
  __host__ __device__ double operator()(long long i) const { return a[i * stride]; }
};

static double pairwise_host(const double* a, long long n, long long stride) {
  if (n <= 128) return pairwise_leaf(StridedGet{a, stride}, n);
  long long n2 = n / 2;
  n2 -= n2 % 8;
  return pairwise_host(a, n2, stride) + pairwise_host(a + n2 * stride, n - n2, stride);
}

__device__ __forceinline__ void note_log_path(int path, double arg, long long* status) {
  if (path != lcr::LOG_CR_FAST) atomicAdd(reinterpret_cast<unsigned long long*>(status), 1ull);
  if (path == lcr::LOG_CR_FAILED)
    atomicMin(reinterpret_cast<unsigned long long*>(status + 1), lcr::bits_of(arg));
}

__global__ void __launch_bounds__(256) log_cr_kernel(const double* __restrict__ x, long long n, double* __restrict__ y,
                                                     int force_accurate, long long* __restrict__ status) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int path;
    y[i] = lcr::log_cr(x[i], force_accurate != 0, &path);
    note_log_path(path, x[i], status);
  }
}

__global__ void __launch_bounds__(NZ_COLS* NZ_ROWS)
    sign_flags_kernel(const double* __restrict__ x, long long rows, long long F, long long n_cols,
                      const uint8_t* __restrict__ negate, int* __restrict__ flags) {
  const long long c = (long long)blockIdx.x * NZ_COLS + threadIdx.x;
  if (c >= n_cols) return;
  const bool neg = negate[c] != 0;
  int bad = 0;
  for (long long r = (long long)blockIdx.y * NZ_ROWS + threadIdx.y; r < rows; r += (long long)gridDim.y * NZ_ROWS) {
    const double v = x[r * F + c];
    bad |= !((neg ? -v : v) >= 0.0);
  }
  if (bad) atomicOr(flags + c, 1);
}

__global__ void __launch_bounds__(NZ_COLS* NZ_ROWS)
    transform_a_kernel(double* __restrict__ x, long long rows, long long F, long long n_cols,
                       const uint8_t* __restrict__ negate, const uint8_t* __restrict__ logm,
                       long long* __restrict__ status) {
  const long long c = (long long)blockIdx.x * NZ_COLS + threadIdx.x;
  if (c >= n_cols) return;
  const bool neg = negate[c] != 0, lg = logm[c] != 0;
  if (!neg && !lg) return;
  for (long long r = (long long)blockIdx.y * NZ_ROWS + threadIdx.y; r < rows; r += (long long)gridDim.y * NZ_ROWS) {
    double v = x[r * F + c];
    if (neg) v = -v;
    if (lg) {
      const double arg = lcr::add(v, 0.01);
      int path;
      v = lcr::log_cr(arg, false, &path);
      if (path != lcr::LOG_CR_FAST) note_log_path(path, arg, status);
    }
    x[r * F + c] = v;
  }
}

struct SquareGet {
  const double* a;
  long long stride;
  double mean;
  __device__ double operator()(long long i) const {
    const double d = lcr::sub(a[i * stride], mean);
    return lcr::mul(d, d);
  }
};

// node_vals[leaf * F + c] for leaves [start[leaf], start[leaf + 1])
template <bool SQUARES>
__global__ void __launch_bounds__(NZ_COLS* NZ_ROWS)
    leaf_kernel(const double* __restrict__ x, long long F, const long long* __restrict__ leaf_start,
                long long n_leaves, const double* __restrict__ mean, double* __restrict__ node_vals) {
  const long long c = (long long)blockIdx.x * NZ_COLS + threadIdx.x;
  if (c >= F) return;
  for (long long leaf = (long long)blockIdx.y * NZ_ROWS + threadIdx.y; leaf < n_leaves;
       leaf += (long long)gridDim.y * NZ_ROWS) {
    const long long r0 = leaf_start[leaf], n = leaf_start[leaf + 1] - r0;
    const double* col = x + r0 * F + c;
    double v;
    if (SQUARES) v = pairwise_leaf(SquareGet{col, F, mean[c]}, n);
    else v = pairwise_leaf(StridedGet{col, F}, n);
    node_vals[leaf * F + c] = v;
  }
}

__global__ void __launch_bounds__(256) combine_kernel(const long long* __restrict__ children, long long first,
                                                      long long count, long long F, double* __restrict__ node_vals) {
  const long long total = count * F;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long j = i / F, c = i - j * F;
    node_vals[(first + j) * F + c] =
        lcr::add(node_vals[children[2 * j] * F + c], node_vals[children[2 * j + 1] * F + c]);
  }
}

__global__ void finish_kernel(const double* __restrict__ root, long long F, long long n, bool take_sqrt,
                              double* __restrict__ out) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= F) return;
  const double v = __ddiv_rn(lcr::add(0.0, root[c]), (double)n);
  out[c] = take_sqrt ? __dsqrt_rn(v) : v;
}

__global__ void __launch_bounds__(NZ_COLS* NZ_ROWS)
    transform_b_kernel(double* __restrict__ x, long long rows, long long F, long long n_cols,
                       const double* __restrict__ mean, const double* __restrict__ std) {
  const long long c = (long long)blockIdx.x * NZ_COLS + threadIdx.x;
  if (c >= F) return;
  const bool keep = c < n_cols;
  const double m = keep ? mean[c] : 0.0, den = keep ? lcr::add(std[c], 1e-6) : 1.0;
  for (long long r = (long long)blockIdx.y * NZ_ROWS + threadIdx.y; r < rows; r += (long long)gridDim.y * NZ_ROWS)
    x[r * F + c] = keep ? __ddiv_rn(lcr::sub(x[r * F + c], m), den) : 0.0;
}

}  // namespace arb

using namespace arb;

static dim3 column_grid(long long cols, long long rows) {
  const long long gx = (cols + NZ_COLS - 1) / NZ_COLS;
  long long gy = (rows + NZ_ROWS - 1) / NZ_ROWS;
  const long long cap = ((long long)sm_count() * 16 + gx - 1) / gx;
  gy = gy < cap ? gy : cap;
  return dim3(unsigned(gx), unsigned(gy > 0 ? (gy < 65535 ? gy : 65535) : 1));
}

extern "C" int32_t arb_log_cr(const double* x, int64_t n, double* y, int32_t force_accurate, int64_t* status,
                              void* stream) {
  if (!x || !y || !status || n <= 0) {
    arb_set_error("arb_log_cr: null pointer or n <= 0");
    return ARB_E_INVALID_ARG;
  }
  const long long want = (n + 255) / 256, cap = (long long)sm_count() * 16;
  return launch(log_cr_kernel, dim3(unsigned(want < cap ? want : cap)), dim3(256), 0,
                static_cast<cudaStream_t>(stream), false, x, (long long)n, y, (int)force_accurate,
                reinterpret_cast<long long*>(status));
}

extern "C" int32_t arb_log_cr_host(const double* x, int64_t n, double* y, int32_t force_accurate, int64_t* status) {
  if (!x || !y || !status || n < 0) {
    arb_set_error("arb_log_cr_host: null pointer or n < 0");
    return ARB_E_INVALID_ARG;
  }
  for (int64_t i = 0; i < n; ++i) {
    int path;
    y[i] = lcr::log_cr(x[i], force_accurate != 0, &path);
    status[0] += path != lcr::LOG_CR_FAST;
    if (path == lcr::LOG_CR_FAILED && lcr::bits_of(x[i]) < static_cast<uint64_t>(status[1]))
      status[1] = static_cast<int64_t>(lcr::bits_of(x[i]));
  }
  return ARB_OK;
}

extern "C" int32_t arb_pairwise_sum_host(const double* x, int64_t n, int64_t stride, double* out) {
  if ((!x && n > 0) || !out || n < 0) {
    arb_set_error("arb_pairwise_sum_host: null pointer or n < 0");
    return ARB_E_INVALID_ARG;
  }
  *out = 0.0 + pairwise_host(x, n, stride);
  return ARB_OK;
}

extern "C" int32_t arb_norm_sign_flags(const double* x, int64_t rows, int64_t n_features, int64_t n_cols,
                                       const uint8_t* negate, int32_t* flags, void* stream) {
  if (!x || !negate || !flags || rows <= 0 || n_cols <= 0 || n_cols > n_features) {
    arb_set_error("arb_norm_sign_flags: null pointer, rows <= 0 or n_cols outside [1, n_features]");
    return ARB_E_INVALID_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (cudaMemsetAsync(flags, 0, sizeof(int32_t) * n_cols, st) != cudaSuccess) {
    cudaGetLastError();
    arb_set_error("arb_norm_sign_flags: cudaMemsetAsync failed");
    return ARB_E_CUDA;
  }
  return launch(sign_flags_kernel, column_grid(n_cols, rows), dim3(NZ_COLS, NZ_ROWS), 0, st, false, x,
                (long long)rows, (long long)n_features, (long long)n_cols, negate, reinterpret_cast<int*>(flags));
}

extern "C" int32_t arb_norm_transform_a(double* x, int64_t rows, int64_t n_features, int64_t n_cols,
                                        const uint8_t* negate, const uint8_t* log_mask, int64_t* status,
                                        void* stream) {
  if (!x || !negate || !log_mask || !status || rows <= 0 || n_cols <= 0 || n_cols > n_features) {
    arb_set_error("arb_norm_transform_a: null pointer, rows <= 0 or n_cols outside [1, n_features]");
    return ARB_E_INVALID_ARG;
  }
  return launch(transform_a_kernel, column_grid(n_cols, rows), dim3(NZ_COLS, NZ_ROWS), 0,
                static_cast<cudaStream_t>(stream), false, x, (long long)rows, (long long)n_features,
                (long long)n_cols, negate, log_mask, reinterpret_cast<long long*>(status));
}

extern "C" int32_t arb_norm_column_stats(const double* x, int64_t rows, int64_t n_features, const int64_t* leaf_start,
                                         int64_t n_leaves, const int64_t* children, const int64_t* level_counts,
                                         int64_t n_levels, double* node_vals, double* mean, double* std,
                                         void* stream) {
  if (!x || !leaf_start || !node_vals || !mean || !std || !level_counts || rows <= 0 || n_features <= 0 ||
      n_leaves <= 0 || n_levels < 0 || (n_levels > 0 && !children)) {
    arb_set_error("arb_norm_column_stats: null pointer or empty input");
    return ARB_E_INVALID_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long F = n_features;
  const long long* ls = reinterpret_cast<const long long*>(leaf_start);
  const long long* ch = reinterpret_cast<const long long*>(children);
  long long n_nodes = n_leaves;
  for (int64_t l = 0; l < n_levels; ++l) n_nodes += level_counts[l];
  const double* root = node_vals + (n_nodes - 1) * F;
  for (int pass = 0; pass < 2; ++pass) {
    const dim3 grid = column_grid(F, n_leaves);
    const int rc = pass ? launch(leaf_kernel<true>, grid, dim3(NZ_COLS, NZ_ROWS), 0, st, false, x, F, ls,
                                 (long long)n_leaves, static_cast<const double*>(mean), node_vals)
                        : launch(leaf_kernel<false>, grid, dim3(NZ_COLS, NZ_ROWS), 0, st, false, x, F, ls,
                                 (long long)n_leaves, static_cast<const double*>(nullptr), node_vals);
    if (rc) return rc;
    long long first = n_leaves, done = 0;
    for (int64_t l = 0; l < n_levels; ++l) {
      const long long count = level_counts[l];
      const long long want = (count * F + 255) / 256, cap = (long long)sm_count() * 16;
      if (int rc2 = launch(combine_kernel, dim3(unsigned(want < cap ? want : cap)), dim3(256), 0, st, false,
                           ch + 2 * done, first, count, F, node_vals))
        return rc2;
      first += count;
      done += count;
    }
    if (int rc3 = launch(finish_kernel, dim3(unsigned((F + 255) / 256)), dim3(256), 0, st, false, root, F,
                         (long long)rows, pass == 1, pass ? std : mean))
      return rc3;
  }
  return ARB_OK;
}

extern "C" int32_t arb_norm_transform_b(double* x, int64_t rows, int64_t n_features, int64_t n_cols,
                                        const double* mean, const double* std, void* stream) {
  if (!x || !mean || !std || rows <= 0 || n_cols <= 0 || n_cols > n_features) {
    arb_set_error("arb_norm_transform_b: null pointer, rows <= 0 or n_cols outside [1, n_features]");
    return ARB_E_INVALID_ARG;
  }
  return launch(transform_b_kernel, column_grid(n_features, rows), dim3(NZ_COLS, NZ_ROWS), 0,
                static_cast<cudaStream_t>(stream), false, x, (long long)rows, (long long)n_features,
                (long long)n_cols, mean, std);
}
