// Slate movers either side of the scorer (SURVEY.md 8(f) ranks 3 and 4) -- pure HBM-bound row traffic:
//
//   assemble_slates_kernel  the reference's per-slate FixLength transform + ToTensor + DataLoader collation
//                           (allrank/data/dataset_loading.py:32-93, :230-247) for a whole batch in one launch:
//                           the corpus lives in HBM as query-grouped rows (docs_x [N,F], docs_y [N], CSR offsets
//                           [Q+1]); each CTA builds one slate of length S -- zero/-1 padding when the query is
//                           shorter than S, otherwise a uniform sample without replacement that keeps the
//                           reference's "do not lose the only relevant item" rules.
//   gather_slates_kernel    inference_utils.__rank_slates (allrank/inference/inference_utils.py:37-60): X and y
//                           rows re-ordered by the descending score ranking (the ranking itself is the metrics
//                           kernel's out_order).
//
// Sampling uses a counter-based hash (seed, slate, attempt, item) instead of numpy's Mersenne stream, so sampled
// slates agree with the reference in distribution; padded slates are bit-identical.  oracle/slates_ref.py restates
// the hash on the host (HashSource) and drives the reference's _sample rules with it: every slate equals that model.
#include <cstdint>
#include <cuda_runtime.h>

#include "block_utils.cuh"
#include "common.h"
#include "dropout.cuh"

namespace arb {

constexpr int ASM_THREADS = 256;
constexpr int ASM_MAX_ATTEMPTS = 1024;   // the reference recurses without bound (dataset_loading.py:69-70); the
                                         // 1024th draw is kept even if it holds no relevant item

__device__ __forceinline__ uint32_t sample_hash(uint64_t seed, uint32_t slate, uint32_t attempt, uint32_t item) {
  uint32_t h = mix32(uint32_t(seed) ^ (slate * 0x9e3779b1u));
  h = mix32(h ^ uint32_t(seed >> 32) ^ (attempt * 0x85ebca6bu + 0x7f4a7c15u));
  return mix32(h ^ (item * 0xc2b2ae35u + 0x165667b1u));
}

// copy one row of F floats (float4 when both rows are 16-byte aligned)
__device__ __forceinline__ void copy_row(float* __restrict__ dst, const float* __restrict__ src, int F, int t, int nt,
                                         bool vec) {
  if (vec) {
    const float4* s4 = reinterpret_cast<const float4*>(src);
    float4* d4 = reinterpret_cast<float4*>(dst);
    for (int c = t; c < F / 4; c += nt) d4[c] = s4 ? s4[c] : make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    for (int c = t; c < F; c += nt) dst[c] = src ? src[c] : 0.f;
  }
}

// Dynamic shared memory: uint64 keys[np2(max query length)] (sampling only) followed by int sel[S].
__global__ void __launch_bounds__(ASM_THREADS) assemble_slates_kernel(
    const float* __restrict__ docs_x, const float* __restrict__ docs_y, const long long* __restrict__ offsets,
    const long long* __restrict__ queries, long long n_queries, int S, int F, int key_slots, unsigned long long seed,
    int vec,
    float* __restrict__ x_out, float* __restrict__ y_out, long long* __restrict__ idx_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  int* sel = reinterpret_cast<int*>(keys + key_slots);
  __shared__ float red[32];
  __shared__ int s_first_max;
  const int b = blockIdx.x;
  const long long q = queries[b];
  const bool known = q >= 0 && q < n_queries;          // an unknown query number yields an all-padding slate
  const long long base = known ? offsets[q] : 0;
  const int n = known ? int(offsets[q + 1] - base) : 0;
  const float* y = docs_y + base;

  if (n < S) {   // _pad (dataset_loading.py:76-93): rows in file order, then zeros / -1 / -1
    for (int r = threadIdx.x; r < S; r += blockDim.x) sel[r] = r < n ? r : -1;
  } else {       // _sample (:55-74)
    float tot = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) tot += y[i];
    tot = block_sum(tot, red);
    const int np2 = next_pow2(n);
    for (int attempt = 0;; ++attempt) {
      for (int i = threadIdx.x; i < np2; i += blockDim.x)
        keys[i] = i < n ? (uint64_t(sample_hash(seed, uint32_t(b), uint32_t(attempt), uint32_t(i))) << 32) | uint32_t(i)
                        : ~0ull;
      __syncthreads();
      bitonic_sort(keys, np2);            // the S smallest keys, in key order = np.random.choice(n, S, replace=False)
      float got = 0.f;
      for (int r = threadIdx.x; r < S; r += blockDim.x) got += y[uint32_t(keys[r])];
      got = block_sum(got, red);
      // draw again only while the sample sums to 0 and the query to more than 0 but not 1 (:69-70); a query sum
      // of 0, below 0 or NaN keeps the sample, a sum of 1 is patched below (:66-68)
      if (!(got == 0.f && tot > 0.f && tot != 1.0f) || attempt + 1 >= ASM_MAX_ATTEMPTS) break;
      __syncthreads();
    }
    float got = 0.f;
    for (int r = threadIdx.x; r < S; r += blockDim.x) { sel[r] = int(uint32_t(keys[r])); got += y[sel[r]]; }
    got = block_sum(got, red);
    if (got == 0.f && tot == 1.0f) {      // keep S-1 of the sample, append np.argmax(y): the first maximum
      float m = -CUDART_INF_F;
      for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, y[i]);
      m = block_max(m, red);
      if (threadIdx.x == 0) s_first_max = n;
      __syncthreads();
      for (int i = threadIdx.x; i < n; i += blockDim.x)
        if (y[i] == m) atomicMin(&s_first_max, i);
      __syncthreads();
      if (threadIdx.x == 0) sel[S - 1] = s_first_max;
    }
  }
  __syncthreads();
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int r = wid; r < S; r += nw) {     // one warp per output row: coalesced along the features
    const int i = sel[r];
    float* dst = x_out + (size_t(b) * S + r) * F;
    copy_row(dst, i >= 0 ? docs_x + size_t(base + i) * F : nullptr, F, lane, 32, vec != 0);
    if (lane == 0) {
      y_out[size_t(b) * S + r] = i >= 0 ? y[i] : -1.0f;        // PADDED_Y_VALUE (:15)
      idx_out[size_t(b) * S + r] = i;                          // PADDED_INDEX_VALUE = -1 (:16)
    }
  }
}

// out_x[b, r, :] = x[b, order[b, r], :],  out_y[b, r] = y[b, order[b, r]]
__global__ void __launch_bounds__(256) gather_slates_kernel(const float* __restrict__ x, const float* __restrict__ y,
                                                            const int* __restrict__ order, long long rows, int S,
                                                            int F, int vec, float* __restrict__ x_out,
                                                            float* __restrict__ y_out) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const long long b = row / S;
  const int src = order[row];
  copy_row(x_out + size_t(row) * F, x + (size_t(b) * S + src) * F, F, lane, 32, vec != 0);
  if (lane == 0) y_out[row] = y[b * S + src];
}

}  // namespace arb

using namespace arb;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

extern "C" size_t arb_assemble_slates_smem_bytes(int32_t max_query_len, int32_t S) {
  const int slots = max_query_len >= S ? next_pow2(max_query_len) : 0;
  return size_t(slots) * 8 + size_t(S) * 4;
}

extern "C" int32_t arb_assemble_slates(const float* docs_x, const float* docs_y, const int64_t* offsets,
                                       int64_t n_queries, const int64_t* queries, int32_t B, int32_t S,
                                       int32_t F, int32_t max_query_len, uint64_t seed, float* x_out, float* y_out,
                                       int64_t* idx_out, void* stream) {
  if (!docs_x || !docs_y || !offsets || !queries || !x_out || !y_out || !idx_out || B <= 0 || S <= 0 || F <= 0 ||
      max_query_len <= 0 || n_queries <= 0) {
    arb_set_error("arb_assemble_slates: null pointer or bad shape");
    return ARB_E_INVALID_ARG;
  }
  const size_t smem = arb_assemble_slates_smem_bytes(max_query_len, S);
  if (smem > 200 * 1024) {
    arb_set_error("arb_assemble_slates: queries above 16384 items (or slate_length above ~50k) are not supported");
    return ARB_E_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int vec = (F % 4 == 0) && aligned16(docs_x) && aligned16(x_out);
  const int key_slots = max_query_len >= S ? next_pow2(max_query_len) : 0;
  ProfScope ps(ARB_PROF_SLATES, double(B) * S * (8.0 * F + 16.0), st);
  return launch(assemble_slates_kernel, dim3(B), dim3(ASM_THREADS), smem, st, /*pdl=*/false, docs_x, docs_y,
                reinterpret_cast<const long long*>(offsets), reinterpret_cast<const long long*>(queries), n_queries, S,
                F, key_slots, seed, vec, x_out, y_out, reinterpret_cast<long long*>(idx_out));
}

extern "C" int32_t arb_gather_slates(const float* x, const float* y, const int32_t* order, int32_t B, int32_t S,
                                     int32_t F, float* x_out, float* y_out, void* stream) {
  if (!x || !y || !order || !x_out || !y_out || B <= 0 || S <= 0 || F <= 0) {
    arb_set_error("arb_gather_slates: null pointer or bad shape");
    return ARB_E_INVALID_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long rows = (long long)B * S;
  const int vec = (F % 4 == 0) && aligned16(x) && aligned16(x_out);
  ProfScope ps(ARB_PROF_SLATES, double(rows) * (8.0 * F + 12.0), st);
  return launch(gather_slates_kernel, dim3(unsigned((rows + 7) / 8)), dim3(256), 0, st, /*pdl=*/false, x, y, order, rows,
                S, F, vec, x_out, y_out);
}
