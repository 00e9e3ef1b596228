// Click models (allrank/click_models/*) on the device: arb_click_slates evaluates a flattened click-model tree over
// a batch of ranked slates, one CTA per slate (include/allrank_b200.h documents the node kinds).
//
//   compaction   the real items (y != pad) of the slate, in slate order, by a block prefix count: every model sees
//                only those, like MaskedRemainMasked (click_utils.py:30-53)
//   tree         nodes are evaluated children first into per-node byte masks in shared memory; under a MULTIPLE only
//                the chosen child's subtree runs, so only its errors are reported.  Errors set a per-slate status.
//   distances    fp64 from the fp32 features, (a_k - b_k)^2 / |a_k - b_k| summed over k in order with round-to-nearest
//                adds and multiplies (no FMA) and a correctly rounded sqrt: the loop scipy's cdist runs.  Each thread
//                owns whole pairs i < j.  The slate's real rows are staged once in shared memory as fp32 with an odd
//                row stride (the lanes of a warp read 32 different rows j without bank conflicts) when S x F fits;
//                larger slates read the rows from global memory through L1.  DUPLICATES takes a per-column minimum with
//                64-bit atomicMin (non-negative doubles order like their bit patterns); DIVERSE stores the upper
//                triangle in the caller's workspace.
//   quantile     numpy's linear method: the order statistics lo and lo+1 of the stored distances by an 8-pass radix
//                select over their bit patterns with a shared-memory histogram, then numpy's _lerp.
//   greedy scan  one warp walks the inner model's clicks top to bottom and takes each candidate's minimum distance over
//                the kept set from the stored triangle.
//
// Uniforms are 53-bit values of a counter hash of (seed, node, global slate index, position), so results do not
// depend on chunking or scheduling (numpy's stream is not reproduced).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <cuda_runtime.h>

#include "block_utils.cuh"
#include "common.h"
#include "dropout.cuh"

namespace arb {

constexpr int CLK_THREADS = 256;
constexpr int CLK_MAX_LIST = 1024;   // FIXED positions + MULTIPLE cumulative probabilities of one tree

struct ClickTree {
  arb_click_node node[ARB_CLICK_MAX_NODES];
  double list[CLK_MAX_LIST];
  int32_t post[ARB_CLICK_MAX_NODES];   // evaluation order: post-order depth-first (the reference's recursion order)
  int32_t n_nodes, n_list;
};

__host__ __device__ __forceinline__ uint64_t click_bits(uint64_t seed, uint32_t node, uint64_t slate, uint32_t item) {
  uint32_t a = mix32(uint32_t(seed) ^ (node * 0x9e3779b1u + 0x7f4a7c15u));
  a = mix32(a ^ uint32_t(seed >> 32) ^ (uint32_t(slate) * 0x85ebca6bu));
  a = mix32(a ^ (uint32_t(slate >> 32) * 0xc2b2ae35u) ^ (item * 0x27d4eb2fu + 0x165667b1u));
  const uint32_t hi = mix32(a ^ 0x68e31da4u), lo = mix32(a + 0xb5297a4du);
  return (uint64_t(hi) << 21) | (lo >> 11);   // 53 bits
}
__device__ __forceinline__ double click_uniform(uint64_t seed, uint32_t node, uint64_t slate, uint32_t item) {
  return double(click_bits(seed, node, slate, item)) * 0x1p-53;
}

// first pair index of row i of the row-major upper triangle (i < j) of an n x n matrix
__host__ __device__ __forceinline__ long long tri_row(long long i, long long n) { return i * (2 * n - i - 1) / 2; }

template <int METRIC>
__device__ __forceinline__ double pair_dist(const float* a, const float* b, int F) {
  double acc = 0.0;
  for (int k = 0; k < F; ++k) {
    const double d = __dsub_rn(double(a[k]), double(b[k]));
    if (METRIC == ARB_CLICK_METRIC_EUCLIDEAN || METRIC == ARB_CLICK_METRIC_SQEUCLIDEAN) acc = __dadd_rn(acc, __dmul_rn(d, d));
    else if (METRIC == ARB_CLICK_METRIC_CITYBLOCK) acc = __dadd_rn(acc, fabs(d));
    else acc = fmax(acc, fabs(d));
  }
  return METRIC == ARB_CLICK_METRIC_EUCLIDEAN ? __dsqrt_rn(acc) : acc;
}

// Where the features of real item i are: rows + (map ? map[i] : i) * ld (the staged rows, or x through ridx).
struct Rows {
  const float* base;
  const int* map;
  int ld;
  __device__ __forceinline__ const float* row(long long i) const { return base + size_t(map ? map[i] : int(i)) * ld; }
};

// All pairs i < j of the n real items: tri[p] = dist (when tri), colmin[j] = min(colmin[j], dist) (when colmin).
template <int METRIC>
__device__ void pair_pass_m(Rows rows, int n, int F, double* __restrict__ tri, unsigned long long* colmin) {
  const long long m = (long long)n * (n - 1) / 2;
  const double two_n1 = 2.0 * n - 1.0;
  for (long long p = threadIdx.x; p < m; p += blockDim.x) {
    long long i = (long long)((two_n1 - sqrt(two_n1 * two_n1 - 8.0 * double(p))) * 0.5);
    i = i < 0 ? 0 : (i > n - 2 ? n - 2 : i);
    while (i > 0 && tri_row(i, n) > p) --i;
    while (i < n - 2 && tri_row(i + 1, n) <= p) ++i;
    const long long j = p - tri_row(i, n) + i + 1;
    const double d = pair_dist<METRIC>(rows.row(i), rows.row(j), F);
    if (tri) tri[p] = d;
    if (colmin) atomicMin(colmin + j, (unsigned long long)__double_as_longlong(d));
  }
}

__device__ __forceinline__ void pair_pass(int metric, Rows rows, int n, int F, double* tri, unsigned long long* colmin) {
  switch (metric) {
    case ARB_CLICK_METRIC_EUCLIDEAN: pair_pass_m<ARB_CLICK_METRIC_EUCLIDEAN>(rows, n, F, tri, colmin); break;
    case ARB_CLICK_METRIC_SQEUCLIDEAN: pair_pass_m<ARB_CLICK_METRIC_SQEUCLIDEAN>(rows, n, F, tri, colmin); break;
    case ARB_CLICK_METRIC_CITYBLOCK: pair_pass_m<ARB_CLICK_METRIC_CITYBLOCK>(rows, n, F, tri, colmin); break;
    default: pair_pass_m<ARB_CLICK_METRIC_CHEBYSHEV>(rows, n, F, tri, colmin); break;
  }
}

// The k-th smallest (0-based) of the m non-negative doubles v, as its bit pattern.  Every thread gets the result.
__device__ uint64_t radix_select(const double* __restrict__ v, long long m, long long k, int* hist,
                                 unsigned long long* sel) {
  if (threadIdx.x == 0) { sel[0] = 0; sel[1] = 0; sel[2] = (unsigned long long)k; }
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int d = threadIdx.x; d < 256; d += blockDim.x) hist[d] = 0;
    __syncthreads();
    const uint64_t prefix = sel[0], mask = sel[1];
    for (long long p = threadIdx.x; p < m; p += blockDim.x) {
      const uint64_t b = (uint64_t)__double_as_longlong(v[p]);
      if ((b & mask) == prefix) atomicAdd(hist + ((b >> shift) & 255), 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      long long kk = (long long)sel[2], cum = 0;
      int d = 0;
      for (; d < 255; ++d) {
        if (cum + hist[d] > kk) break;
        cum += hist[d];
      }
      sel[0] = prefix | (uint64_t(d) << shift);
      sel[1] = mask | (uint64_t(255) << shift);
      sel[2] = (unsigned long long)(kk - cum);
    }
    __syncthreads();
  }
  const uint64_t r = sel[0];
  __syncthreads();
  return r;
}

// np.quantile(v, q) (method "linear"): h = (m-1) q, a = v_(floor h), b = v_(floor h + 1), _lerp(a, b, h - floor h).
__device__ double linear_quantile(const double* __restrict__ v, long long m, double q, int* hist,
                                  unsigned long long* sel, int* cnt) {
  const double h = __dmul_rn(double(m - 1), q);
  if (h >= double(m - 1)) return __longlong_as_double((long long)radix_select(v, m, m - 1, hist, sel));
  const double lo = floor(h);
  const double g = __dsub_rn(h, lo);
  const long long k = (long long)lo;
  const uint64_t abits = radix_select(v, m, k, hist, sel);
  // b: a again when more than k+1 values are <= a, else the smallest value above a
  if (threadIdx.x == 0) { *cnt = 0; sel[3] = ~0ull; }
  __syncthreads();
  int c = 0;
  unsigned long long above = ~0ull;
  for (long long p = threadIdx.x; p < m; p += blockDim.x) {
    const uint64_t b = (uint64_t)__double_as_longlong(v[p]);
    if (b <= abits) ++c;
    else above = b < above ? b : above;
  }
  atomicAdd(cnt, c);
  atomicMin(sel + 3, above);
  __syncthreads();
  const uint64_t bbits = (long long)*cnt > k + 1 ? abits : sel[3];
  __syncthreads();
  const double a = __longlong_as_double((long long)abits), b = __longlong_as_double((long long)bbits);
  const double diff = __dsub_rn(b, a);
  return g >= 0.5 ? __dsub_rn(b, __dmul_rn(diff, __dsub_rn(1.0, g))) : __dadd_rn(a, __dmul_rn(diff, g));
}

// The real rows into shared memory (coalesced along the features), once per slate, before its first distance pass.
// Ends with a barrier.
__device__ __forceinline__ void stage_rows(float* staged, int ld, const float* __restrict__ x, const int* ridx, int n,
                                        int F, int* ready) {
  if (staged && !*ready) {
    for (long long e = threadIdx.x; e < (long long)n * F; e += blockDim.x) {
      const int j = int(e / F), k = int(e - (long long)j * F);
      staged[size_t(j) * ld + k] = x[size_t(ridx[j]) * F + k];
    }
    __syncthreads();
    if (threadIdx.x == 0) *ready = 1;
  }
  __syncthreads();
}

__device__ __forceinline__ void set_status(int* s, int code) { atomicCAS(s, ARB_CLICK_OK, code); }

// Dynamic shared memory: uint64 buf[S] | int ridx[S] | uint8 masks[n_nodes][S] (16-byte multiple) |
// float rows[S][stage_ld] when stage_ld > 0 (the real rows, compacted, staged at the first distance pass)
__global__ void __launch_bounds__(CLK_THREADS, 1) click_kernel(
    ClickTree tree, const double* __restrict__ tables, const float* __restrict__ x_all, const float* __restrict__ y_all,
    int S, int F, int stage_ld, float pad, long long slate0, unsigned long long seed, float* __restrict__ clicks_all,
    int* __restrict__ status, double* __restrict__ tri_all, long long tri_stride) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(smem_raw);
  int* ridx = reinterpret_cast<int*>(buf + S);
  unsigned char* masks = reinterpret_cast<unsigned char*>(ridx + S);
  __shared__ ClickTree t;
  __shared__ int s_warp[32], s_hist[256], s_status, s_cnt, s_tri_ready, s_rows_ready;
  __shared__ unsigned long long s_sel[4];
  __shared__ unsigned char s_active[ARB_CLICK_MAX_NODES];

  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
  const int b = blockIdx.x;
  const uint64_t slate = uint64_t(slate0 + b);
  const float* y = y_all + size_t(b) * S;
  const float* x = x_all ? x_all + size_t(b) * S * F : nullptr;
  float* clicks = clicks_all + size_t(b) * S;
  double* tri = tri_all ? tri_all + size_t(b) * tri_stride : nullptr;

  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&tree);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&t);
    for (int w = tid; w < int(sizeof(ClickTree) / 4); w += nt) dst[w] = src[w];
  }

  // real items, in slate order
  int n = 0;
  for (int t0 = 0; t0 < S; t0 += nt) {
    const int p = t0 + tid;
    const bool real = p < S && y[p] != pad;
    const unsigned bal = __ballot_sync(FULL, real);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    int before = n, total = n;
    for (int w = 0; w < nw; ++w) {
      total += s_warp[w];
      if (w < wid) before += s_warp[w];
    }
    if (real) ridx[before + __popc(bal & ((1u << lane) - 1u))] = p;
    n = total;
    __syncthreads();
  }

  // which nodes run: all of them, except the children a MULTIPLE did not choose (and their subtrees)
  if (tid == 0) {
    s_status = ARB_CLICK_OK;
    s_tri_ready = 0;
    s_rows_ready = 0;
    for (int i = 0; i < t.n_nodes; ++i) s_active[i] = i == 0;
    for (int i = 0; i < t.n_nodes; ++i) {
      if (!s_active[i]) continue;
      const arb_click_node& nd = t.node[i];
      if (nd.kind == ARB_CLICK_MULTIPLE) {
        const double u = click_uniform(seed, uint32_t(i), slate, 0u);
        int c = 0;
        for (int k = 0; k < nd.n_children; ++k)
          if (u < t.list[nd.list_offset + k]) { c = k; break; }
        s_active[nd.first_child + c] = 1;
      } else {
        for (int k = 0; k < nd.n_children; ++k) s_active[nd.first_child + k] = 1;
      }
    }
  }
  __syncthreads();
  float* staged = stage_ld > 0 ? reinterpret_cast<float*>(masks + (size_t(t.n_nodes) * S + 15) / 16 * 16) : nullptr;
  Rows rows;
  rows.base = staged ? staged : x;
  rows.map = staged ? nullptr : ridx;
  rows.ld = staged ? stage_ld : F;

  for (int e = 0; e < t.n_nodes; ++e) {
    const int i = t.post[e];
    if (!s_active[i]) continue;
    const arb_click_node nd = t.node[i];
    unsigned char* m = masks + size_t(i) * S;
    const unsigned char* c0 = nd.n_children > 0 ? masks + size_t(nd.first_child) * S : nullptr;
    switch (nd.kind) {
      case ARB_CLICK_FIXED: {
        for (int j = tid; j < n; j += nt) m[j] = 0;
        __syncthreads();
        for (int k = tid; k < nd.n_list; k += nt) {
          const long long p = (long long)t.list[nd.list_offset + k];
          if (p < -n || p >= n) set_status(&s_status, ARB_CLICK_INDEX_ERROR);
          else m[p < 0 ? p + n : p] = 1;
        }
        break;
      }
      case ARB_CLICK_RANDOM: {
        const int want = nd.iparam;
        if (want > n) set_status(&s_status, ARB_CLICK_VALUE_ERROR);
        for (int j = tid; j < n; j += nt) buf[j] = click_bits(seed, uint32_t(i), slate, uint32_t(j));
        __syncthreads();
        for (int j = tid; j < n; j += nt) {   // rank of j's key, ties to the lower position
          const unsigned long long kj = buf[j];
          int r = 0;
          for (int q = 0; q < n && r < want; ++q) {
            const unsigned long long kq = buf[q];
            r += (kq < kj) || (kq == kj && q < j);
          }
          m[j] = r < want;
        }
        break;
      }
      case ARB_CLICK_RELEVANT: {
        const float thr = float(nd.fparam0);
        for (int j = tid; j < n; j += nt) m[j] = y[ridx[j]] >= thr;
        break;
      }
      case ARB_CLICK_CASCADE: {
        const double* tab = tables + size_t(nd.iparam) * S;
        const float thr = float(nd.fparam1);
        for (int j = tid; j < n; j += nt) {
          const bool observed = tab[j] >= click_uniform(seed, uint32_t(i), slate, uint32_t(j));
          m[j] = y[ridx[j]] * (observed ? 1.0f : 0.0f) >= thr;
        }
        break;
      }
      case ARB_CLICK_MULTIPLE: {
        int c = 0;
        for (int k = 0; k < nd.n_children; ++k)
          if (s_active[nd.first_child + k]) c = k;
        const unsigned char* cm = masks + size_t(nd.first_child + c) * S;
        for (int j = tid; j < n; j += nt) m[j] = cm[j];
        break;
      }
      case ARB_CLICK_CONDITIONED: {
        const bool any = nd.iparam != 0;
        for (int j = tid; j < n; j += nt) {
          bool r = !any;
          for (int k = 0; k < nd.n_children; ++k) {
            const bool v = masks[size_t(nd.first_child + k) * S + j] != 0;
            r = any ? (r || v) : (r && v);
          }
          m[j] = r;
        }
        break;
      }
      case ARB_CLICK_MAXCLICKS: {
        if (wid == 0) {
          int run = 0;
          for (int j0 = 0; j0 < n; j0 += 32) {
            const int j = j0 + lane;
            const bool c = j < n && c0[j];
            const unsigned bal = __ballot_sync(FULL, c);
            const int count = run + __popc(bal & (0xffffffffu >> (31 - lane)));
            if (j < n) m[j] = c && double(count) <= nd.fparam0;
            run += __popc(bal);
          }
        }
        break;
      }
      case ARB_CLICK_DUPLICATES: {
        if (n == 0) set_status(&s_status, ARB_CLICK_VALUE_ERROR);
        for (int j = tid; j < n; j += nt) buf[j] = 0x7ff0000000000000ull;   // +inf
        stage_rows(staged, stage_ld, x, ridx, n, F, &s_rows_ready);
        pair_pass(nd.iparam, rows, n, F, nullptr, buf);
        __syncthreads();
        for (int j = tid; j < n; j += nt) m[j] = __longlong_as_double((long long)buf[j]) > nd.fparam0;
        break;
      }
      case ARB_CLICK_DIVERSE: {
        int local = 0;
        for (int j = tid; j < n; j += nt) local += c0[j] != 0;
        if (__syncthreads_or(local) == 0) {           // nothing to keep
          for (int j = tid; j < n; j += nt) m[j] = 0;
          break;
        }
        const long long npairs = (long long)n * (n - 1) / 2;
        if (!s_tri_ready) {
          stage_rows(staged, stage_ld, x, ridx, n, F, &s_rows_ready);
          pair_pass(ARB_CLICK_METRIC_EUCLIDEAN, rows, n, F, tri, nullptr);
          __syncthreads();
          if (tid == 0) s_tri_ready = 1;
        }
        const double margin = npairs == 0 ? 0.0 : linear_quantile(tri, npairs, nd.fparam0, s_hist, s_sel, &s_cnt);
        if (wid == 0) {
          int* kept = reinterpret_cast<int*>(buf);
          int nk = 0;
          for (int j = 0; j < n; ++j) {
            if (!c0[j]) {
              if (lane == 0) m[j] = 0;
              continue;
            }
            double mn = __longlong_as_double(0x7ff0000000000000ll);
            for (int k = lane; k < nk; k += 32) mn = fmin(mn, tri[tri_row(kept[k], n) + (j - kept[k] - 1)]);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(FULL, mn, o));
            const bool keep = mn > margin;
            if (lane == 0) {
              m[j] = keep;
              if (keep) kept[nk] = j;
            }
            nk += keep;
            __syncwarp();
          }
        }
        break;
      }
      default: break;
    }
    __syncthreads();
  }

  const unsigned char* root = masks;
  for (int j = tid; j < n; j += nt) clicks[ridx[j]] = root[j] ? 1.0f : 0.0f;
  for (int p = tid; p < S; p += nt)
    if (y[p] == pad) clicks[p] = pad;
  if (tid == 0) status[b] = s_status;
}

}  // namespace arb

using namespace arb;

static bool click_needs_tri(const arb_click_node* nodes, int n_nodes) {
  for (int i = 0; i < n_nodes; ++i)
    if (nodes[i].kind == ARB_CLICK_DIVERSE) return true;
  return false;
}

static size_t click_tri_bytes(int S) {
  const size_t b = size_t(S) * size_t(S - 1) / 2 * sizeof(double);
  return (b + 255) / 256 * 256;
}

static size_t click_smem_bytes(int n_nodes, int S) {
  return size_t(S) * 8 + size_t(S) * 4 + (size_t(n_nodes) * S + 15) / 16 * 16;
}

// Staged rows take S x (F | 1) floats of shared memory when the kernel's total stays within this budget
constexpr size_t CLK_STAGE_SMEM_LIMIT = 200 * 1024;

static int click_fail(const char* msg) {
  arb_set_error(msg);
  return ARB_E_INVALID_ARG;
}

// Validates the tree and fills t (nodes, list, post-order); returns ARB_OK or ARB_E_INVALID_ARG with the message set.
static int click_tree(const arb_click_node* nodes, int n_nodes, const double* list, int n_list, ClickTree& t) {
  if (!nodes || n_nodes < 1 || n_nodes > ARB_CLICK_MAX_NODES)
    return click_fail("arb_click_slates: the tree needs 1 to 32 nodes");
  if (n_list < 0 || n_list > CLK_MAX_LIST || (n_list > 0 && !list))
    return click_fail("arb_click_slates: the position/probability list holds at most 1024 values");
  std::memset(&t, 0, sizeof(t));
  int parents[ARB_CLICK_MAX_NODES] = {0};
  for (int i = 0; i < n_nodes; ++i) {
    const arb_click_node& nd = nodes[i];
    if (nd.n_children < 0 || (nd.n_children > 0 && (nd.first_child <= i || nd.first_child + nd.n_children > n_nodes)))
      return click_fail("arb_click_slates: children must be later nodes inside the tree");
    for (int k = 0; k < nd.n_children; ++k) parents[nd.first_child + k]++;
    const bool leaf = nd.kind == ARB_CLICK_FIXED || nd.kind == ARB_CLICK_RANDOM || nd.kind == ARB_CLICK_RELEVANT ||
                      nd.kind == ARB_CLICK_CASCADE || nd.kind == ARB_CLICK_DUPLICATES;
    if (nd.kind < ARB_CLICK_FIXED || nd.kind > ARB_CLICK_DIVERSE) return click_fail("arb_click_slates: unknown node kind");
    if (leaf && nd.n_children != 0) return click_fail("arb_click_slates: a leaf model has children");
    if ((nd.kind == ARB_CLICK_MAXCLICKS || nd.kind == ARB_CLICK_DIVERSE) && nd.n_children != 1)
      return click_fail("arb_click_slates: MAXCLICKS and DIVERSE take exactly one child");
    if ((nd.kind == ARB_CLICK_MULTIPLE || nd.kind == ARB_CLICK_CONDITIONED) && nd.n_children < 1)
      return click_fail("arb_click_slates: MULTIPLE and CONDITIONED need at least one child");
    if ((nd.kind == ARB_CLICK_FIXED || nd.kind == ARB_CLICK_MULTIPLE) &&
        (nd.n_list < 0 || nd.list_offset < 0 || nd.list_offset + nd.n_list > n_list))
      return click_fail("arb_click_slates: a node's list lies outside list_host");
    if (nd.kind == ARB_CLICK_MULTIPLE && nd.n_list != nd.n_children)
      return click_fail("arb_click_slates: MULTIPLE needs one cumulative probability per child");
    if (nd.kind == ARB_CLICK_RANDOM && nd.iparam < 0) return click_fail("arb_click_slates: RANDOM needs n_clicks >= 0");
    if (nd.kind == ARB_CLICK_CASCADE && nd.iparam < 0) return click_fail("arb_click_slates: bad CASCADE table index");
    if (nd.kind == ARB_CLICK_CONDITIONED && (nd.iparam < 0 || nd.iparam > 1))
      return click_fail("arb_click_slates: CONDITIONED combines with all (0) or any (1)");
    if (nd.kind == ARB_CLICK_DUPLICATES && (nd.iparam < ARB_CLICK_METRIC_EUCLIDEAN || nd.iparam > ARB_CLICK_METRIC_CHEBYSHEV))
      return click_fail("arb_click_slates: unknown DUPLICATES metric");
    if (nd.kind == ARB_CLICK_DIVERSE && !(nd.fparam0 >= 0.0 && nd.fparam0 <= 1.0))
      return click_fail("arb_click_slates: DIVERSE quantile must lie in [0, 1]");
  }
  if (parents[0] != 0) return click_fail("arb_click_slates: node 0 must be the root");
  for (int i = 1; i < n_nodes; ++i)
    if (parents[i] != 1) return click_fail("arb_click_slates: every node but the root needs exactly one parent");
  // post-order depth first: children in order, then the node
  int stack[ARB_CLICK_MAX_NODES], next[ARB_CLICK_MAX_NODES], sp = 0, k = 0;
  stack[sp] = 0; next[sp] = 0; ++sp;
  while (sp > 0) {
    const int v = stack[sp - 1];
    if (next[sp - 1] < nodes[v].n_children) {
      const int c = nodes[v].first_child + next[sp - 1]++;
      stack[sp] = c; next[sp] = 0; ++sp;
    } else {
      t.post[k++] = v;
      --sp;
    }
  }
  std::memcpy(t.node, nodes, sizeof(arb_click_node) * n_nodes);
  if (n_list > 0) std::memcpy(t.list, list, sizeof(double) * n_list);
  t.n_nodes = n_nodes;
  t.n_list = n_list;
  return ARB_OK;
}

extern "C" size_t arb_click_workspace_bytes(const arb_click_node* nodes_host, int32_t n_nodes, int32_t B, int32_t S,
                                            int32_t F) {
  (void)F;
  if (!nodes_host || n_nodes < 1 || n_nodes > ARB_CLICK_MAX_NODES || B <= 0 || S <= 1) return 0;
  return click_needs_tri(nodes_host, n_nodes) ? size_t(B) * click_tri_bytes(S) : 0;
}

extern "C" int32_t arb_click_slates(const arb_click_node* nodes_host, int32_t n_nodes, const double* list_host,
                                    int32_t n_list, const double* observe_tables, const float* x, const float* y,
                                    int32_t B, int32_t S, int32_t F, float pad, int64_t slate_offset, uint64_t seed,
                                    float* clicks, int32_t* status, void* workspace, size_t ws_bytes, void* stream) {
  std::unique_ptr<ClickTree> tp(new ClickTree);   // (~9.5 KB: kept off the stack; the launch copies it)
  ClickTree& t = *tp;
  if (int rc = click_tree(nodes_host, n_nodes, list_host, n_list, t)) return rc;
  if (!y || !clicks || !status || B < 0 || S < 1) return click_fail("arb_click_slates: null pointer or bad shape");
  if (S > ARB_CLICK_MAX_SLATE) {
    arb_set_error("arb_click_slates: slates above 4096 items are not supported");
    return ARB_E_UNSUPPORTED;
  }
  bool need_x = false;
  for (int i = 0; i < n_nodes; ++i) {
    need_x |= nodes_host[i].kind == ARB_CLICK_DUPLICATES || nodes_host[i].kind == ARB_CLICK_DIVERSE;
    if (nodes_host[i].kind == ARB_CLICK_CASCADE && !observe_tables)
      return click_fail("arb_click_slates: CASCADE needs observe_tables");
  }
  if (need_x && (!x || F < 1)) return click_fail("arb_click_slates: the tree measures distances and needs x [B,S,F]");
  if (B == 0) return ARB_OK;
  const bool need_tri = click_needs_tri(nodes_host, n_nodes) && S > 1;
  const size_t per = need_tri ? click_tri_bytes(S) : 0;
  long long chunk = B;
  if (need_tri) {
    chunk = workspace ? (long long)(ws_bytes / per) : 0;
    if (chunk < 1) {
      arb_set_error("arb_click_slates: the workspace does not hold one slate's distances (arb_click_workspace_bytes)");
      return ARB_E_WORKSPACE;
    }
  }
  size_t smem = click_smem_bytes(n_nodes, S);
  int stage_ld = 0;
  if (need_x && smem + size_t(S) * size_t(F | 1) * sizeof(float) <= CLK_STAGE_SMEM_LIMIT) {
    stage_ld = F | 1;
    smem += size_t(S) * size_t(stage_ld) * sizeof(float);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (long long c0 = 0; c0 < B; c0 += chunk) {
    const long long nb = std::min<long long>(chunk, B - c0);
    if (int rc = launch(click_kernel, dim3(unsigned(nb)), dim3(CLK_THREADS), smem, st, /*pdl=*/false, t,
                        observe_tables, need_x ? x + size_t(c0) * S * F : nullptr, y + size_t(c0) * S, S, F, stage_ld, pad,
                        (long long)(slate_offset + c0), (unsigned long long)seed, clicks + size_t(c0) * S,
                        status + c0, need_tri ? static_cast<double*>(workspace) : nullptr,
                        (long long)(per / sizeof(double))))
      return rc;
  }
  return ARB_OK;
}
