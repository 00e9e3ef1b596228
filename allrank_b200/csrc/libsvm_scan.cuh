// The one-block exclusive scan of the LibSVM reader's line index (libsvm.cu) and of the writer's row offsets
// (libsvm_write.cu).  `static`: each translation unit launches its own copy.
#pragma once
#include <cuda_runtime.h>

namespace arb {

constexpr int SCAN_THREADS = 1024;

// In-place exclusive scan of a[0, n) by one block; *total = the sum.
static __global__ void __launch_bounds__(SCAN_THREADS) exclusive_scan_kernel(long long* __restrict__ a, long long n,
                                                                             long long* __restrict__ total) {
  __shared__ long long warp_tot[SCAN_THREADS / 32];
  const long long seg = (n + SCAN_THREADS - 1) / SCAN_THREADS;
  const long long lo = threadIdx.x * seg, hi = lo + seg < n ? lo + seg : n;
  long long s = 0;
  for (long long i = lo; i < hi; ++i) s += a[i];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long incl = s;
  for (int o = 1; o < 32; o <<= 1) {
    const long long v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  long long run = incl - s;
  for (int w = 0; w < wid; ++w) run += warp_tot[w];
  for (long long i = lo; i < hi; ++i) {
    const long long v = a[i];
    a[i] = run;
    run += v;
  }
  if (threadIdx.x == SCAN_THREADS - 1) *total = run;
}

}  // namespace arb
