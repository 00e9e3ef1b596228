// Slate kernels: ranking metrics and the O(S) / O(S^2) listwise losses, forward + backward fused.
//
// One CTA owns one slate.  A slate is S scores + S labels (2.9 KB at S=240), so everything after the
// two coalesced loads lives in shared memory / registers: the in-SMEM bitonic sort, the pair loops,
// the reductions.  Algorithmic HBM traffic per slate: 8*S bytes in, 4*S bytes of gradient out
// (12*S+4 with the loss partial) -- versus the 3.5-9 MB per slate the reference materialises.
//
// Reference semantics are cited per kernel; DESIGN.md section 4 has the derivations of the backward passes.
#include <cstdint>
#include <cuda_runtime.h>

#include "block_utils.cuh"
#include "common.h"

namespace arb {

// ------------------------------------------------------------------------------------------------
// Loading + sorting a slate (shared by metrics / approxNDCG / lambdaLoss)
// ------------------------------------------------------------------------------------------------
struct SlateSmem {
  uint64_t* keys;   // [np2]  (score desc, position asc) sort keys
  uint32_t* ikeys;  // [np2]  label-descending keys for the ideal ordering
  float* s;         // [S] scores in score order (-inf for padded items)
  float* t;         // [S] labels in score order (0 for padded items)
  float* a;         // [S] per-item scratch
  float* b;         // [S] per-item scratch
  float* c;         // [S] per-item scratch
  float* red;       // [32] reduction scratch
  double* dred;     // [32]
};

__host__ __device__ inline size_t slate_smem_bytes(int S) {
  const int np2 = next_pow2(S);
  return size_t(np2) * 8 + size_t(np2) * 4 + size_t(S) * 4 * 5 + 32 * 4 + 32 * 8 + 64;
}

__device__ inline SlateSmem carve(unsigned char* base, int S) {
  const int np2 = next_pow2(S);
  SlateSmem m;
  m.keys = reinterpret_cast<uint64_t*>(base);
  base += size_t(np2) * 8;
  m.dred = reinterpret_cast<double*>(base);
  base += 32 * 8;
  m.ikeys = reinterpret_cast<uint32_t*>(base);
  base += size_t(np2) * 4;
  m.s = reinterpret_cast<float*>(base);
  base += size_t(S) * 4;
  m.t = reinterpret_cast<float*>(base);
  base += size_t(S) * 4;
  m.a = reinterpret_cast<float*>(base);
  base += size_t(S) * 4;
  m.b = reinterpret_cast<float*>(base);
  base += size_t(S) * 4;
  m.c = reinterpret_cast<float*>(base);
  base += size_t(S) * 4;
  m.red = reinterpret_cast<float*>(base);
  return m;
}

// Builds both orderings.  After the call: keys[i] low 32 bits = original position of the item ranked i by
// score; s[i]/t[i] = its masked score / label; ikeys sorted so that ideal label j = ordered_to_float(~ikeys[j]).
__device__ __forceinline__ float ideal_label(uint32_t ikey) {
  uint32_t o = ~ikey;
  uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
  return __uint_as_float(u);
}

__device__ inline void load_and_sort(const float* __restrict__ yp, const float* __restrict__ yt, int S, float pad,
                                     const SlateSmem& m, bool want_ideal) {
  const int np2 = next_pow2(S);
  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    if (i < S) {
      const float lab = yt[i];
      const bool is_pad = (lab == pad);
      const float sc = is_pad ? -CUDART_INF_F : yp[i];
      m.keys[i] = desc_key(sc, uint32_t(i));
      m.ikeys[i] = ~float_to_ordered(is_pad ? -CUDART_INF_F : lab);
      m.a[i] = sc;                    // staging, original order
      m.b[i] = is_pad ? -CUDART_INF_F : lab;
    } else {
      m.keys[i] = ~0ull;
      m.ikeys[i] = ~0u;
    }
  }
  __syncthreads();
  bitonic_sort(m.keys, np2);
  if (want_ideal) bitonic_sort(m.ikeys, np2);
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const uint32_t pos = uint32_t(m.keys[i]);
    m.s[i] = m.a[pos];
    m.t[i] = m.b[pos];   // -inf marks a padded item
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// Metrics: dcg / ndcg / mrr          reference: allrank/models/metrics.py:7-113
// ------------------------------------------------------------------------------------------------
struct AtList {
  int n;
  int dcg[ARB_MAX_ATS];   // clipped to S (metrics.py:60)
  int mrr[ARB_MAX_ATS];   // unclipped (metrics.py:101)
};

__device__ __forceinline__ float gain_of(float label, int mode) {
  return mode == ARB_GAIN_POW2 ? pow2_minus_1(label) : label;
}

__global__ void __launch_bounds__(256) metrics_kernel(const float* __restrict__ y_pred,
                                                      const float* __restrict__ y_true, int B, int S,
                                                      const float* __restrict__ discounts, AtList ats,
                                                      int gain_mode, float pad, float filler,
                                                      float* __restrict__ out_dcg, float* __restrict__ out_idcg,
                                                      float* __restrict__ out_ndcg, float* __restrict__ mrr_pos,
                                                      float* __restrict__ mrr_best,
                                                      int32_t* __restrict__ out_order) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  SlateSmem m = carve(smem_raw, S);
  const bool want_dcg = out_dcg || out_idcg || out_ndcg;
  load_and_sort(y_pred + size_t(b) * S, y_true + size_t(b) * S, S, pad, m, want_dcg);

  int max_at = 0;
  for (int q = 0; q < ats.n; ++q) max_at = max(max_at, ats.dcg[q]);

  // weighted gains in ranked order: a = by score, b = ideal (labels sorted by themselves); pads carry label 0
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const float lab = (m.t[i] == -CUDART_INF_F) ? 0.0f : m.t[i];
    m.c[i] = lab;
    if (want_dcg) {
      const float d = discounts[i];
      m.a[i] = gain_of(lab, gain_mode) * d;
      float il = ideal_label(m.ikeys[i]);
      il = (il == -CUDART_INF_F) ? 0.0f : il;
      m.b[i] = gain_of(il, gain_mode) * d;
    }
    if (out_order) out_order[size_t(b) * S + i] = int32_t(uint32_t(m.keys[i]));
  }
  __syncthreads();

  if (want_dcg) {
    // torch.cumsum on CPU accumulates fp32 inputs sequentially in double (verified against the golden
    // vectors); two lanes of different warps walk the two sequences so the values can match bit for bit.
    const int role = (threadIdx.x == 0) ? 0 : (threadIdx.x == 32 ? 1 : -1);
    if (role >= 0) {
      const float* w = role == 0 ? m.a : m.b;
      float* cum = role == 0 ? m.s : m.t;   // s/t are free now: reuse as cumulative tables
      double acc = 0.0;
      for (int i = 0; i < max_at; ++i) {
        acc += double(w[i]);
        cum[i] = float(acc);
      }
    }
    __syncthreads();
    for (int q = threadIdx.x; q < ats.n; q += blockDim.x) {
      const int at = ats.dcg[q];
      const float d = at > 0 ? m.s[at - 1] : 0.0f;
      const float id = at > 0 ? m.t[at - 1] : 0.0f;
      const size_t o = size_t(b) * ats.n + q;
      if (out_dcg) out_dcg[o] = d;
      if (out_idcg) out_idcg[o] = id;
      if (out_ndcg) out_ndcg[o] = (id == 0.0f) ? filler : d / id;
    }
  }

  if (mrr_pos) {
    // first position (in score order) holding the slate's maximum label: torch.max(dim=1) semantics
    float best = -CUDART_INF_F;
    int where = 0x7fffffff;
    for (int i = threadIdx.x; i < S; i += blockDim.x) {
      const float v = m.c[i];
      if (v > best) { best = v; where = i; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(FULL, best, o);
      const int ow = __shfl_xor_sync(FULL, where, o);
      if (ob > best || (ob == best && ow < where)) { best = ob; where = ow; }
    }
    __syncthreads();
    int* iw = reinterpret_cast<int*>(m.dred);
    if ((threadIdx.x & 31) == 0) { m.red[threadIdx.x >> 5] = best; iw[threadIdx.x >> 5] = where; }
    __syncthreads();
    if (threadIdx.x == 0) {
      const int nw = (blockDim.x + 31) >> 5;
      for (int w = 1; w < nw; ++w) {
        if (m.red[w] > best || (m.red[w] == best && iw[w] < where)) { best = m.red[w]; where = iw[w]; }
      }
      mrr_pos[b] = float(where);
      mrr_best[b] = best;
    }
  }
}

// mrr epilogue: the "no relevant item" rule is one scalar for the whole batch (metrics.py:108-109).
__global__ void mrr_finalize_kernel(const float* __restrict__ mrr_pos, const float* __restrict__ mrr_best, int B,
                                    AtList ats, float* __restrict__ out_mrr) {
  __shared__ double red[32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) acc += double(mrr_best[i]);
  acc = block_sum(acc, red);
  const bool none_relevant = (float(acc) == 0.0f);
  for (int i = threadIdx.x; i < B * ats.n; i += blockDim.x) {
    const int b = i / ats.n, q = i % ats.n;
    const float pos = mrr_pos[b];
    float r = 1.0f / (pos + 1.0f);
    if (none_relevant) r = 0.0f;
    out_mrr[i] = r * ((pos < float(ats.mrr[q])) ? 1.0f : 0.0f);
  }
}

// ------------------------------------------------------------------------------------------------
// Batch finalisation shared by the losses.
//   mode 0: loss = sum(val)                     (scaling already folded into val / grad)
//   mode 1: loss = sum(val) / sum(cnt), grad *= 1/sum(cnt)              (lambdaLoss reduction="mean")
//   mode 2: like 1, but sum(cnt) == 0 gives loss 0 and zero grad        (neuralNDCG, neuralNDCG.py:66-69)
// Deterministic: fixed-order double accumulation.
// ------------------------------------------------------------------------------------------------
__global__ void finalize_kernel(const float* __restrict__ val, const float* __restrict__ cnt, int B, int mode,
                                float* __restrict__ loss, float* __restrict__ grad, size_t n_grad) {
  __shared__ double red[32];
  double v = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    v += double(val[i]);
    if (mode != 0) c += double(cnt[i]);
  }
  v = block_sum(v, red);
  if (mode != 0) c = block_sum(c, red);
  float scale = 1.0f;
  if (mode == 0) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *loss = float(v);
    return;
  }
  if (c == 0.0) {
    scale = (mode == 2) ? 0.0f : CUDART_NAN_F;
    if (blockIdx.x == 0 && threadIdx.x == 0) *loss = (mode == 2) ? 0.0f : CUDART_NAN_F;
  } else {
    scale = float(1.0 / c);
    if (blockIdx.x == 0 && threadIdx.x == 0) *loss = float(v / c);
  }
  if (grad) {
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n_grad; i += size_t(gridDim.x) * blockDim.x)
      grad[i] = (scale == 0.0f) ? 0.0f : grad[i] * scale;
  }
}

// ------------------------------------------------------------------------------------------------
// listNet                                     reference: allrank/models/losses/listNet.py:8-30
//   loss_b = -sum_i q_i log(p_i + eps),  p = softmax(scores), q = softmax(labels), pads at -inf
//   d loss_b / d s_k = -(r_k - p_k R),   r_i = q_i p_i / (p_i + eps),  R = sum_i r_i
// One warp per slate (O(S) work, 8 items per lane at S=240), coalesced strided loads.
// ------------------------------------------------------------------------------------------------
constexpr int LISTNET_MAX_PER_LANE = 40;  // S <= 1280 in registers; larger slates use the block kernel below

__global__ void __launch_bounds__(128) listnet_warp_kernel(const float* __restrict__ y_pred,
                                                           const float* __restrict__ y_true, int B, int S,
                                                           float eps, float pad, float inv_B,
                                                           float* __restrict__ val, float* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* yp = y_pred + size_t(b) * S;
  const float* yt = y_true + size_t(b) * S;
  float s[LISTNET_MAX_PER_LANE], t[LISTNET_MAX_PER_LANE];
  float ms = -CUDART_INF_F, mt = -CUDART_INF_F;
#pragma unroll
  for (int r = 0; r < LISTNET_MAX_PER_LANE; ++r) {
    const int i = lane + 32 * r;
    s[r] = t[r] = -CUDART_INF_F;
    if (i < S) {
      const float lab = yt[i];
      if (lab != pad) { s[r] = yp[i]; t[r] = lab; }
    }
    ms = fmaxf(ms, s[r]);
    mt = fmaxf(mt, t[r]);
  }
  ms = warp_max(ms);
  mt = warp_max(mt);
  float zs = 0.f, zt = 0.f;
#pragma unroll
  for (int r = 0; r < LISTNET_MAX_PER_LANE; ++r) {
    s[r] = expf(s[r] - ms);   // all-padded slate: -inf - -inf = NaN, like the reference (SURVEY quirk Q2)
    t[r] = expf(t[r] - mt);
    if (lane + 32 * r < S) { zs += s[r]; zt += t[r]; }
  }
  zs = warp_sum(zs);
  zt = warp_sum(zt);
  float lossb = 0.f, R = 0.f;
#pragma unroll
  for (int r = 0; r < LISTNET_MAX_PER_LANE; ++r) {
    if (lane + 32 * r < S) {
      const float p = s[r] / zs, q = t[r] / zt;
      lossb -= q * logf(p + eps);
      const float rr = q * p / (p + eps);
      R += rr;
      s[r] = p;
      t[r] = rr;
    }
  }
  lossb = warp_sum(lossb);
  R = warp_sum(R);
  if (lane == 0) val[b] = lossb * inv_B;
  if (grad) {
#pragma unroll
    for (int r = 0; r < LISTNET_MAX_PER_LANE; ++r) {
      const int i = lane + 32 * r;
      if (i < S) grad[size_t(b) * S + i] = -(t[r] - s[r] * R) * inv_B;
    }
  }
}

// Same maths, one CTA per slate, items kept in shared memory: any S.
__global__ void __launch_bounds__(256) listnet_block_kernel(const float* __restrict__ y_pred,
                                                            const float* __restrict__ y_true, int B, int S,
                                                            float eps, float pad, float inv_B,
                                                            float* __restrict__ val, float* __restrict__ grad) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s = reinterpret_cast<float*>(smem_raw);
  float* t = s + S;
  float* red = t + S;
  const int b = blockIdx.x;
  float ms = -CUDART_INF_F, mt = -CUDART_INF_F;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const float lab = y_true[size_t(b) * S + i];
    const bool is_pad = lab == pad;
    s[i] = is_pad ? -CUDART_INF_F : y_pred[size_t(b) * S + i];
    t[i] = is_pad ? -CUDART_INF_F : lab;
    ms = fmaxf(ms, s[i]);
    mt = fmaxf(mt, t[i]);
  }
  ms = block_max(ms, red);
  mt = block_max(mt, red);
  float zs = 0.f, zt = 0.f;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    s[i] = expf(s[i] - ms);
    t[i] = expf(t[i] - mt);
    zs += s[i];
    zt += t[i];
  }
  zs = block_sum(zs, red);
  zt = block_sum(zt, red);
  float lossb = 0.f, R = 0.f;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const float p = s[i] / zs, q = t[i] / zt;
    lossb -= q * logf(p + eps);
    const float rr = q * p / (p + eps);
    R += rr;
    s[i] = p;
    t[i] = rr;
  }
  lossb = block_sum(lossb, red);
  R = block_sum(R, red);
  if (threadIdx.x == 0) val[b] = lossb * inv_B;
  if (grad)
    for (int i = threadIdx.x; i < S; i += blockDim.x) grad[size_t(b) * S + i] = -(t[i] - s[i] * R) * inv_B;
}

// ------------------------------------------------------------------------------------------------
// listMLE                                     reference: allrank/models/losses/listMLE.py:7-38
//   shuffle columns by `perm`, sort labels descending, z = scores in that order (pads -> -inf) minus max,
//   tail_i = sum_{j>=i} exp(z_j),  loss_b = sum_{valid i} log(tail_i + eps) - z_i
//   d/dz_k = e_k * C_k - 1,  C_k = sum_{valid i<=k} 1/(tail_i + eps);   the max-shift contributes
//   sum_i eps/(tail_i+eps) to the arg-max item (autograd of listMLE.py:28-30 does the same).
// ------------------------------------------------------------------------------------------------
__device__ inline void block_inclusive_scan(float* x, int n, float* red, bool reverse) {
  // Blocked scan: each thread owns a contiguous chunk; chunk totals are scanned by thread 0.
  const int T = blockDim.x;
  const int chunk = (n + T - 1) / T;
  const int lo = threadIdx.x * chunk, hi = min(n, lo + chunk);
  float acc = 0.f;
  for (int i = lo; i < hi; ++i) {
    const int j = reverse ? n - 1 - i : i;
    acc += x[j];
    x[j] = acc;
  }
  __syncthreads();
  float* tot = red;  // needs >= blockDim.x floats
  tot[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float run = 0.f;
    for (int w = 0; w < T; ++w) { const float v = tot[w]; tot[w] = run; run += v; }
  }
  __syncthreads();
  const float off = tot[threadIdx.x];
  for (int i = lo; i < hi; ++i) {
    const int j = reverse ? n - 1 - i : i;
    x[j] += off;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256) listmle_kernel(const float* __restrict__ y_pred,
                                                      const float* __restrict__ y_true, int B, int S, float eps,
                                                      float pad, const int64_t* __restrict__ perm,
                                                      const int32_t* __restrict__ order, float inv_B,
                                                      float* __restrict__ val, float* __restrict__ grad) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  const int np2 = next_pow2(S);
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);
  float* z = reinterpret_cast<float*>(keys + np2);   // [S]
  float* e = z + S;                                  // [S] exp / tail
  float* cc = e + S;                                 // [S] 1/(tail+eps) / prefix
  int* src = reinterpret_cast<int*>(cc + S);         // [S] original column of sorted item i
  float* red = reinterpret_cast<float*>(src + S);    // [blockDim.x]

  for (int i = threadIdx.x; i < np2; i += blockDim.x) {
    if (i < S) {
      const int col = int(perm[i]);
      const float lab = y_true[size_t(b) * S + col];
      keys[i] = desc_key(lab, uint32_t(i));   // labels descending; pads (-1) sort below every real label >= 0
      e[i] = lab;                             // shuffled labels
      src[i] = col;
    } else {
      keys[i] = ~0ull;
    }
  }
  __syncthreads();
  if (order == nullptr) bitonic_sort(keys, np2);
  // gather in sorted order
  float mx = -CUDART_INF_F;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const int j = order ? order[size_t(b) * S + i] : int(uint32_t(keys[i]));
    const float lab = e[j];
    const int col = src[j];
    const float sc = (lab == pad) ? -CUDART_INF_F : y_pred[size_t(b) * S + col];
    z[i] = sc;
    cc[i] = __int_as_float(col);
    mx = fmaxf(mx, sc);
  }
  mx = block_max(mx, red);
  __syncthreads();
  int amax = 0x7fffffff;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    src[i] = __float_as_int(cc[i]);
    if (z[i] == mx) amax = min(amax, i);
    // pads stay -inf: in an all-padded slate mx is -inf too and -inf - -inf would make them NaN, i.e. "valid"
    // below, where the reference masks them to 0 and the slate adds nothing
    if (z[i] != -CUDART_INF_F) z[i] = z[i] - mx;
    e[i] = expf(z[i]);
  }
  // first arg-max in sorted order (torch.max(dim) returns the first maximal index)
  amax = -int(block_max(float(-amax), red));
  __syncthreads();
  for (int i = threadIdx.x; i < S; i += blockDim.x) cc[i] = e[i];
  __syncthreads();
  block_inclusive_scan(cc, S, red, /*reverse=*/true);   // cc[i] = tail_i
  float lossb = 0.f, shift = 0.f;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const bool valid = z[i] != -CUDART_INF_F;
    const float tail = cc[i];
    if (valid) {
      lossb += logf(tail + eps) - z[i];
      shift += eps / (tail + eps);
    }
    cc[i] = valid ? 1.0f / (tail + eps) : 0.0f;
  }
  lossb = block_sum(lossb, red);
  shift = block_sum(shift, red);
  __syncthreads();
  block_inclusive_scan(cc, S, red, /*reverse=*/false);  // cc[k] = C_k
  if (threadIdx.x == 0) val[b] = lossb * inv_B;
  if (grad) {
    for (int i = threadIdx.x; i < S; i += blockDim.x) {
      const bool valid = z[i] != -CUDART_INF_F;
      float g = 0.f;
      if (valid) {
        g = e[i] * cc[i] - 1.0f;
        // the max-shift z = raw - max routes -sum_k dL/dz_k = sum_i eps/(tail_i+eps) to the arg-max item
        if (i == amax) g += shift;
      }
      grad[size_t(b) * S + src[i]] = g * inv_B;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// approxNDCGLoss                               reference: allrank/models/losses/approxNDCG.py:7-53
//   a_i = 1 + sum_{j != i} max(sigmoid(-alpha (s_i - s_j)), eps)        (valid i, j)
//   loss_b = -sum_i G_i / log2(1 + a_i),   G_i = (2^t_i - 1) / max(maxDCG, eps)
//   d loss_b/d s_k = alpha * sum_{i != k} w_ik ( [sig_ik >= eps] h_i - [sig_ki >= eps] h_k ),
//       w_ik = sig_ik sig_ki,  h_i = G_i / (log2(1+a_i)^2 (1+a_i) ln 2)
// Thread k owns row k; the other operand is a shared-memory broadcast.
// ------------------------------------------------------------------------------------------------
// sigmoid for the S x S pair loops: the kernel is bound by instruction issue (about 85 instructions per pair with
// expf and IEEE division), so the pair terms use the SFU forms -- ex2.approx and rcp.approx, 2 ulp each -- on the
// overflow-free branch exp(-|x|); a sum of up to S such terms keeps the loss within 1e-6 relative of the reference
// (the 1e-5 bound of SURVEY.md 8c; tests/test_gpu_losses.py).
__device__ __forceinline__ float pair_sigmoid(float x) {
  const float ex = __expf(-fabsf(x));
  const float big = __fdividef(1.0f, 1.0f + ex);
  return x >= 0.f ? big : ex * big;
}

__global__ void __launch_bounds__(256) approx_ndcg_kernel(const float* __restrict__ y_pred,
                                                          const float* __restrict__ y_true, int B, int S,
                                                          float eps, float pad, float alpha, float inv_B,
                                                          float* __restrict__ val, float* __restrict__ grad) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  SlateSmem m = carve(smem_raw, S);
  load_and_sort(y_pred + size_t(b) * S, y_true + size_t(b) * S, S, pad, m, true);

  // number of valid items: they occupy ranks [0, n) unless a real score is -inf (handled by the flag test)
  float part = 0.f;
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    float il = ideal_label(m.ikeys[j]);
    il = fmaxf(il, 0.0f);   // clamp_(min=0) turns the -inf pads into label 0, gain 0
    part += pow2_minus_1(il) / log2f(2.0f + float(j));
  }
  const float max_dcg = fmaxf(block_sum(part, m.red), eps);

  float* G = m.a;
  float* h = m.b;
  float lossb = 0.f;
  // the pair loops stop at the last real item of the score order (pads sort behind every finite score, so for the usual
  // slate this is the item count: half the S x S pairs of an MSLR-shaped batch); the per-item flag test stays
  float hi_part = 0.f;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const bool valid = m.t[i] != -CUDART_INF_F;
    G[i] = valid ? pow2_minus_1(fmaxf(m.t[i], 0.0f)) / max_dcg : 0.0f;
    if (valid) hi_part = float(i + 1);
  }
  const int n_hi = int(block_max(hi_part, m.red));
  __syncthreads();
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const bool valid = m.t[i] != -CUDART_INF_F;
    float a = 1.0f;
    if (valid) {
      const float si = m.s[i];
      float acc = 0.f;
      for (int j = 0; j < n_hi; ++j) {
        if (j != i && m.t[j] != -CUDART_INF_F) acc += fmaxf(pair_sigmoid(-alpha * (si - m.s[j])), eps);
      }
      a += acc;
    }
    const float L = log2f(1.0f + a);
    lossb -= G[i] / L;
    h[i] = G[i] / (L * L * (1.0f + a) * 0.6931471805599453f);
  }
  lossb = block_sum(lossb, m.red);
  if (threadIdx.x == 0) val[b] = lossb * inv_B;
  if (!grad) return;
  __syncthreads();
  for (int k = threadIdx.x; k < S; k += blockDim.x) {
    const bool valid = m.t[k] != -CUDART_INF_F;
    float g = 0.f;
    if (valid) {
      const float sk = m.s[k], hk = h[k];
      for (int i = 0; i < n_hi; ++i) {
        if (i == k || m.t[i] == -CUDART_INF_F) continue;
        const float x = alpha * (m.s[i] - sk);      // sig_ik = sigmoid(-x), sig_ki = sigmoid(x)
        const float ex = __expf(-fabsf(x));
        const float big = __fdividef(1.0f, 1.0f + ex), small = ex * big;
        const float sig_ik = x >= 0.f ? small : big;
        const float sig_ki = x >= 0.f ? big : small;
        const float w = sig_ik * sig_ki;
        g += w * ((sig_ik >= eps ? h[i] : 0.0f) - (sig_ki >= eps ? hk : 0.0f));
      }
      g *= alpha;
    }
    grad[size_t(b) * S + uint32_t(m.keys[k])] = g * inv_B;
  }
}

// ------------------------------------------------------------------------------------------------
// lambdaLoss (7 weighing schemes)              reference: allrank/models/losses/lambdaLoss.py:7-114
//   for every selected ordered pair (i,j) in score order (both valid, i,j < k, t_i > t_j unless ndcgLoss1):
//     x = clamp(s_i - s_j, +-1e8); p = max(sigmoid(sigma x), eps); q = max(p^w, eps); term = log_b(q)
//   loss = -sum terms (or / #pairs).   d(-term)/dx = -w sigma (1-p) / ln(b) when neither clamp is active.
// Thread r owns item r and visits every partner c once, taking the pair in whichever direction is selected.
// ------------------------------------------------------------------------------------------------
struct LambdaCfg {
  int scheme, k, log_base;
  float sigma, mu, eps;
};

__device__ __forceinline__ float lambda_weight(const LambdaCfg& cfg, int i, int j, const float* G,
                                               const float* invD, const float* toe, const float* t) {
  switch (cfg.scheme) {
    case ARB_SCHEME_NDCGLOSS1: return G[i] * invD[i];   // (G / D)[:, :, None]; the kernel divides by log2 directly
    case ARB_SCHEME_NDCGLOSS2: return toe[abs(i - j)] * fabsf(G[i] - G[j]);
    case ARB_SCHEME_LAMBDARANK: return fabsf(invD[i] - invD[j]) * fabsf(G[i] - G[j]);
    case ARB_SCHEME_NDCGLOSS2PP:
      return cfg.mu * (toe[abs(i - j)] * fabsf(G[i] - G[j])) + fabsf(invD[i] - invD[j]) * fabsf(G[i] - G[j]);
    case ARB_SCHEME_RANKNET_GTDIFF: return fabsf(t[i] - t[j]);
    case ARB_SCHEME_RANKNET_GTDIFF_POWED: return fabsf(t[i] * t[i] - t[j] * t[j]);
    default: return 1.0f;
  }
}

// value and d(-term)/dx of one selected pair
__device__ __forceinline__ void lambda_pair(const LambdaCfg& cfg, float si, float sj, float w, float log_eps,
                                            float inv_ln_base, float& term, float& dneg) {
  const float raw = si - sj;
  const float x = fminf(fmaxf(raw, -1e8f), 1e8f);
  const float p = sigmoidf_(cfg.sigma * x);
  const bool p_ok = p >= cfg.eps;
  const float pc = p_ok ? p : cfg.eps;
  // log_b(pc^w) = w log_b(pc); compare in the log domain against log_b(eps) for the outer clamp
  const float lq = w * (cfg.log_base == ARB_LOG_BINARY ? log2f(pc) : logf(pc));
  const bool q_ok = lq >= log_eps;
  term = q_ok ? lq : log_eps;
  const bool x_ok = (raw >= -1e8f) && (raw <= 1e8f);
  dneg = (p_ok && q_ok && x_ok) ? -w * cfg.sigma * (1.0f - p) * inv_ln_base : 0.0f;
}

__global__ void __launch_bounds__(256) lambda_loss_kernel(const float* __restrict__ y_pred,
                                                          const float* __restrict__ y_true, int B, int S,
                                                          float pad, LambdaCfg cfg, float* __restrict__ val,
                                                          float* __restrict__ cnt, float* __restrict__ grad) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  SlateSmem m = carve(smem_raw, S);
  float* toe = reinterpret_cast<float*>(smem_raw + slate_smem_bytes(S));  // [S] extra
  load_and_sort(y_pred + size_t(b) * S, y_true + size_t(b) * S, S, pad, m, true);
  const int kk = (cfg.k <= 0 || cfg.k > S) ? S : cfg.k;

  float part = 0.f;
  for (int j = threadIdx.x; j < kk; j += blockDim.x) {
    const float il = fmaxf(ideal_label(m.ikeys[j]), 0.0f);
    part += pow2_minus_1(il) / log2f(2.0f + float(j));
  }
  const float max_dcg = fmaxf(block_sum(part, m.red), cfg.eps);

  float* G = m.a;
  float* invD = m.b;
  float* tl = m.c;   // clamped labels
  float hi_part = 0.f;    // the pair loop stops at the last real item of the score order (see approx_ndcg_kernel)
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const bool valid = m.t[i] != -CUDART_INF_F;
    if (valid) hi_part = float(i + 1);
    tl[i] = valid ? fmaxf(m.t[i], 0.0f) : 0.0f;
    G[i] = pow2_minus_1(tl[i]) / max_dcg;
    const float D = log2f(2.0f + float(i));
    invD[i] = 1.0f / D;
    // Toeplitz table of ndcgLoss2: lag l >= 1 -> |1/D[l-1] - 1/D[l]| with D[m] = log2(m+2)   (lambdaLoss.py:88-92)
    toe[i] = (i == 0) ? 0.0f : fabsf(1.0f / log2f(1.0f + float(i)) - 1.0f / log2f(2.0f + float(i)));
  }
  const int c_hi = min(kk, int(block_max(hi_part, m.red)));
  __syncthreads();

  const float log_eps = cfg.log_base == ARB_LOG_BINARY ? log2f(cfg.eps) : logf(cfg.eps);
  const float inv_ln_base = cfg.log_base == ARB_LOG_BINARY ? 1.4426950408889634f : 1.0f;
  float lossb = 0.f, npairs = 0.f;
  for (int r = threadIdx.x; r < S; r += blockDim.x) {
    float g = 0.f;
    const bool active = (r < kk) && (m.t[r] != -CUDART_INF_F);
    if (active) {
      const float sr = m.s[r], tr = m.t[r];
      for (int c = 0; c < c_hi; ++c) {
        const float tc = m.t[c];
        if (tc == -CUDART_INF_F) continue;
        float term, d;
        if (cfg.scheme == ARB_SCHEME_NDCGLOSS1) {
          // every ordered pair of valid items is selected, the diagonal included (lambdaLoss.py:39-42)
          lambda_pair(cfg, sr, m.s[c], G[r] / log2f(2.0f + float(r)), log_eps, inv_ln_base, term, d);
          lossb -= term;
          npairs += 1.0f;
          g += d;
          if (c != r) {
            lambda_pair(cfg, m.s[c], sr, G[c] / log2f(2.0f + float(c)), log_eps, inv_ln_base, term, d);
            g -= d;
          } else {
            g -= d;   // x = s_r - s_r: both roles cancel
          }
        } else if (tr > tc) {
          lambda_pair(cfg, sr, m.s[c], lambda_weight(cfg, r, c, G, invD, toe, tl), log_eps, inv_ln_base, term, d);
          lossb -= term;
          npairs += 1.0f;
          g += d;
        } else if (tc > tr) {
          lambda_pair(cfg, m.s[c], sr, lambda_weight(cfg, c, r, G, invD, toe, tl), log_eps, inv_ln_base, term, d);
          g -= d;
        }
      }
    }
    if (grad) grad[size_t(b) * S + uint32_t(m.keys[r])] = g;
  }
  lossb = block_sum(lossb, m.red);
  npairs = block_sum(npairs, m.red);
  if (threadIdx.x == 0) { val[b] = lossb; cnt[b] = npairs; }
}


// ------------------------------------------------------------------------------------------------
// "Next-row" losses of allrank.models.losses that reuse the machinery above (SURVEY.md 8f rank 1).
// ------------------------------------------------------------------------------------------------
// rankNet / rankNet_weightByGTDiff / rankNet_weightByGTDiff_pow     reference: losses/rankNet.py:9-79
//   BCEWithLogits(target = 1, weight = w) over every ordered pair (i,j) of real items with t_i > t_j:
//   term = w * softplus(-(s_i - s_j)),  loss = mean over all selected pairs of the batch.
//   weight_mode 0: 1   1: |t_i - t_j|   2: |t_i^2 - t_j^2|
__device__ __forceinline__ float softplus_neg(float x) {   // log(1 + exp(-x)), stable
  return fmaxf(-x, 0.0f) + log1pf(expf(-fabsf(x)));
}
__global__ void __launch_bounds__(256) ranknet_kernel(const float* __restrict__ y_pred,
                                                      const float* __restrict__ y_true, int B, int S, float pad,
                                                      int weight_mode, float* __restrict__ val,
                                                      float* __restrict__ cnt, float* __restrict__ grad) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s = reinterpret_cast<float*>(smem_raw);
  float* t = s + S;
  float* red = t + S;
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < S; i += blockDim.x) {
    const float lab = y_true[size_t(b) * S + i];
    t[i] = (lab == pad) ? -CUDART_INF_F : lab;
    s[i] = y_pred[size_t(b) * S + i];
  }
  __syncthreads();
  float lossb = 0.f, npairs = 0.f;
  for (int r = threadIdx.x; r < S; r += blockDim.x) {
    float g = 0.f;
    const float tr = t[r], sr = s[r];
    if (tr != -CUDART_INF_F) {
      for (int c = 0; c < S; ++c) {
        const float tc = t[c];
        if (tc == -CUDART_INF_F || tc == tr) continue;
        const float w = weight_mode == 0 ? 1.0f : (weight_mode == 1 ? fabsf(tr - tc) : fabsf(tr * tr - tc * tc));
        if (tr > tc) {            // pair (r, c): x = s_r - s_c
          const float x = sr - s[c];
          lossb += w * softplus_neg(x);
          npairs += 1.0f;
          g -= w * (1.0f / (1.0f + expf(x)));      // d/ds_r = -w sigmoid(-x)
        } else {                  // pair (c, r): x = s_c - s_r, d/ds_r = +w sigmoid(-x)
          const float x = s[c] - sr;
          g += w * (1.0f / (1.0f + expf(x)));
        }
      }
    }
    if (grad) grad[size_t(b) * S + r] = g;
  }
  lossb = block_sum(lossb, red);
  npairs = block_sum(npairs, red);
  if (threadIdx.x == 0) { val[b] = lossb; cnt[b] = npairs; }
}

// binary_listNet (losses/binary_listNet.py:8-33), pointwise_rmse (pointwise.py:6-32), bce (bce.py:8-32):
// O(S) per slate, one warp per slate, mode selects the formula.  Each pass streams the slate, item i on lane i % 32,
// and recomputes what it needs from the inputs, so any slate length runs with a handful of registers.
//   mode 0 binary_listNet: -sum_i (y_i / max(sum y,1 if 0)) log(softmax(s)_i + eps)           mean over batch
//   mode 1 pointwise_rmse: sqrt( sum_valid (y_i - L s_i)^2 / n_valid )                          mean over batch
//   mode 2 bce           : sum_valid -(y log p + (1-y) log(1-p)) (logs clamped at -100),  / #slates with a valid item
__global__ void __launch_bounds__(128) pointwise_warp_kernel(const float* __restrict__ y_pred,
                                                             const float* __restrict__ y_true, int B, int S,
                                                             float pad, int mode, float param, float eps, float inv_B,
                                                             float* __restrict__ val, float* __restrict__ cnt,
                                                             float* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* yp = y_pred + size_t(b) * S;
  const float* yt = y_true + size_t(b) * S;
  float* gb = grad ? grad + size_t(b) * S : nullptr;
  float nvalid = 0.f, lossb = 0.f;
  if (mode == 2) {
    for (int i = lane; i < S; i += 32) {
      const float y = yt[i];
      float g = 0.f;
      if (y != pad) {
        const float p = yp[i];
        nvalid += 1.f;
        lossb -= y * fmaxf(logf(p), -100.0f) + (1.0f - y) * fmaxf(logf(1.0f - p), -100.0f);
        g = (p - y) / fmaxf(p * (1.0f - p), 1e-12f);       // BCELoss backward
      }
      if (gb) gb[i] = g;
    }
    nvalid = warp_sum(nvalid);
    lossb = warp_sum(lossb);
    if (lane == 0) { val[b] = lossb; cnt[b] = nvalid > 0.f ? 1.f : 0.f; }
    return;
  }
  float tsum = 0.f, ms = -CUDART_INF_F;
  for (int i = lane; i < S; i += 32) {
    const float lab = yt[i];
    if (lab != pad) { nvalid += 1.f; tsum += lab; ms = fmaxf(ms, yp[i]); }
  }
  nvalid = warp_sum(nvalid);
  tsum = warp_sum(tsum);
  if (mode == 0) {
    ms = warp_max(ms);
    const float norm = (tsum == 0.0f) ? 1.0f : tsum;
    float zs = 0.f;
    for (int i = lane; i < S; i += 32)
      if (yt[i] != pad) zs += expf(yp[i] - ms);
    zs = warp_sum(zs);
    // padded items: q = 0 and p = 0, so they add -0 to the loss and 0 to R (all-padded slate: p = 0/0, NaN)
    float R = 0.f;
    for (int i = lane; i < S; i += 32) {
      const float lab = yt[i];
      const bool ok = lab != pad;
      const float p = (ok ? expf(yp[i] - ms) : 0.f) / zs, q = (ok ? lab : 0.f) / norm;
      lossb -= q * logf(p + eps);
      R += q * p / (p + eps);
    }
    lossb = warp_sum(lossb);
    R = warp_sum(R);
    if (lane == 0) { val[b] = lossb * inv_B; cnt[b] = 1.f; }
    if (gb) {
      for (int i = lane; i < S; i += 32) {
        const float lab = yt[i];
        const bool ok = lab != pad;
        const float p = (ok ? expf(yp[i] - ms) : 0.f) / zs, q = (ok ? lab : 0.f) / norm;
        gb[i] = -(q * p / (p + eps) - p * R) * inv_B;
      }
    }
  } else {
    float sq = 0.f;
    for (int i = lane; i < S; i += 32) {
      const float lab = yt[i];
      if (lab != pad) {
        const float e = lab - param * yp[i];
        sq += e * e;
      }
    }
    sq = warp_sum(sq);
    const float rmse = sqrtf(sq / nvalid);
    if (lane == 0) { val[b] = rmse * inv_B; cnt[b] = 1.f; }
    if (gb) {
      for (int i = lane; i < S; i += 32) {
        const float lab = yt[i];
        gb[i] = lab != pad ? (-param * (lab - param * yp[i]) / (nvalid * rmse)) * inv_B : 0.f;
      }
    }
  }
}

// ordinal (losses/ordinal.py:8-50): y_pred [B,S,n] probabilities, target level j of an item with label t is
// 1[t >= j+1] (with_ordinals :8-22).  BCE per (item, level) with PyTorch's BCELoss conventions (logs clamped at
// -100, backward divides by max(p(1-p), 1e-12)); padded items contribute nothing.  One warp per slate; the n
// levels of an item are contiguous, so lanes stride over the flattened [S*n] row for coalesced loads.
//   val[b] = sum of the BCE terms, cnt[b] = number of valid items  -> finalize mode 1 (sum / total valid items)
__global__ void __launch_bounds__(128) ordinal_warp_kernel(const float* __restrict__ y_pred,
                                                           const float* __restrict__ y_true, int B, int S, int n,
                                                           float pad, float* __restrict__ val,
                                                           float* __restrict__ cnt, float* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* yp = y_pred + size_t(b) * S * n;
  const float* yt = y_true + size_t(b) * S;
  float lossb = 0.f, nvalid = 0.f;
  for (int e = lane; e < S * n; e += 32) {
    const int i = e / n, j = e - i * n;
    const float lab = yt[i];
    float g = 0.f;
    if (lab != pad) {
      const float p = yp[e];
      const float y = (lab >= float(j + 1)) ? 1.0f : 0.0f;
      lossb -= y * fmaxf(logf(p), -100.0f) + (1.0f - y) * fmaxf(logf(1.0f - p), -100.0f);
      g = (p - y) / fmaxf(p * (1.0f - p), 1e-12f);
      if (j == 0) nvalid += 1.0f;
    }
    if (grad) grad[size_t(b) * S * n + e] = g;
  }
  lossb = warp_sum(lossb);
  nvalid = warp_sum(nvalid);
  if (lane == 0) { val[b] = lossb; cnt[b] = nvalid; }
}

}  // namespace arb

// ================================================================================================
// C ABI
// ================================================================================================
using namespace arb;

// the largest dynamic shared memory a block may use on sm_90
constexpr size_t MAX_SMEM = 227 * 1024;

#define ARB_CHECK_ARGS(cond, msg)            \
  do {                                       \
    if (!(cond)) {                           \
      arb_set_error(msg);                    \
      return ARB_E_INVALID_ARG;              \
    }                                        \
  } while (0)

extern "C" int32_t arb_rank_metrics(const float* y_pred, const float* y_true, int32_t B, int32_t S,
                                    const float* discounts, const int32_t* ats_dcg_host,
                                    const int32_t* ats_mrr_host, int32_t n_ats, int32_t gain_mode,
                                    float pad_value, float filler, float* out_dcg, float* out_idcg,
                                    float* out_ndcg, float* out_mrr, int32_t* out_order, float* mrr_scratch,
                                    void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && B >= 0 && S > 0, "arb_rank_metrics: null input or bad shape");
  ARB_CHECK_ARGS(n_ats >= 0 && n_ats <= ARB_MAX_ATS, "arb_rank_metrics: too many ats (max 32)");
  const bool want_dcg = out_dcg || out_idcg || out_ndcg;
  ARB_CHECK_ARGS(!want_dcg || (discounts && ats_dcg_host), "arb_rank_metrics: dcg needs discounts and ats");
  ARB_CHECK_ARGS(!out_mrr || (ats_mrr_host && mrr_scratch), "arb_rank_metrics: mrr needs ats and scratch");
  if (B == 0) return ARB_OK;
  AtList ats;
  ats.n = n_ats;
  for (int i = 0; i < n_ats; ++i) {
    ats.dcg[i] = ats_dcg_host ? ats_dcg_host[i] : 0;
    ats.mrr[i] = ats_mrr_host ? ats_mrr_host[i] : 0;
    ARB_CHECK_ARGS(ats.dcg[i] >= 0 && ats.dcg[i] <= S, "arb_rank_metrics: dcg ats must be clipped to [0,S]");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = slate_smem_bytes(S);
  if (smem > MAX_SMEM) { arb_set_error("arb_rank_metrics: slate too long for shared memory"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_METRICS, double(B) * (8.0 * S + 4.0 * n_ats), st);
  if (int rc = launch(metrics_kernel, dim3(B), dim3(256), smem, st, /*pdl=*/false, y_pred, y_true, B, S, discounts, ats,
                      gain_mode, pad_value, filler, out_dcg, out_idcg, out_ndcg, out_mrr ? mrr_scratch : nullptr,
                      out_mrr ? mrr_scratch + B : nullptr, out_order))
    return rc;
  if (!out_mrr) return ARB_OK;
  return launch(mrr_finalize_kernel, dim3(1), dim3(256), 0, st, /*pdl=*/false, mrr_scratch, mrr_scratch + B, B, ats,
                out_mrr);
}

static int finalize(const float* val, const float* cnt, int B, int mode, float* loss, float* grad, size_t n_grad,
                    cudaStream_t st) {
  int blocks = 1;
  if (mode != 0 && grad) blocks = int(std::min<size_t>((n_grad + 1023) / 1024, 132 * 4));
  if (blocks < 1) blocks = 1;
  return launch(finalize_kernel, dim3(blocks), dim3(256), 0, st, /*pdl=*/false, val, cnt, B, mode, loss, grad, n_grad);
}

int arb_finalize_mean_over_count(const float* val, const float* cnt, int B, float* loss, float* grad, size_t n_grad,
                                 cudaStream_t st) {
  return finalize(val, cnt, B, 2, loss, grad, n_grad, st);
}

extern "C" int32_t arb_listnet(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps,
                               float pad_value, float* loss, float* grad, float* scratch, void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && loss && scratch && B > 0 && S > 0, "arb_listnet: null pointer or bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const float inv_B = 1.0f / float(B);
  int rc;
  if (S <= 32 * LISTNET_MAX_PER_LANE) {
    const int wpb = 4;
    ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
    rc = launch(listnet_warp_kernel, dim3((B + wpb - 1) / wpb), dim3(wpb * 32), 0, st, /*pdl=*/false, y_pred, y_true, B,
                S, eps, pad_value, inv_B, scratch, grad);
  } else {
    const size_t smem = size_t(S) * 8 + 128;
    if (smem > MAX_SMEM) { arb_set_error("arb_listnet: slate too long"); return ARB_E_UNSUPPORTED; }
    rc = launch(listnet_block_kernel, dim3(B), dim3(256), smem, st, /*pdl=*/false, y_pred, y_true, B, S, eps, pad_value,
                inv_B, scratch, grad);
  }
  if (rc) return rc;
  return finalize(scratch, nullptr, B, 0, loss, nullptr, 0, st);
}

extern "C" int32_t arb_listmle(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps,
                               float pad_value, const int64_t* perm, const int32_t* order, float* loss,
                               float* grad, float* scratch, void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && loss && scratch && perm && B > 0 && S > 0,
                 "arb_listmle: null pointer or bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = size_t(next_pow2(S)) * 8 + size_t(S) * 16 + 256 * 4 + 64;
  if (smem > MAX_SMEM) { arb_set_error("arb_listmle: slate too long"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
  if (int rc = launch(listmle_kernel, dim3(B), dim3(256), smem, st, /*pdl=*/false, y_pred, y_true, B, S, eps, pad_value,
                      perm, order, 1.0f / float(B), scratch, grad))
    return rc;
  return finalize(scratch, nullptr, B, 0, loss, nullptr, 0, st);
}

extern "C" int32_t arb_approx_ndcg(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps,
                                   float pad_value, float alpha, float* loss, float* grad, float* scratch,
                                   void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && loss && scratch && B > 0 && S > 0,
                 "arb_approx_ndcg: null pointer or bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = slate_smem_bytes(S);
  if (smem > MAX_SMEM) { arb_set_error("arb_approx_ndcg: slate too long"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
  if (int rc = launch(approx_ndcg_kernel, dim3(B), dim3(256), smem, st, /*pdl=*/false, y_pred, y_true, B, S, eps,
                      pad_value, alpha, 1.0f / float(B), scratch, grad))
    return rc;
  return finalize(scratch, nullptr, B, 0, loss, nullptr, 0, st);
}

extern "C" int32_t arb_lambda_loss(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps,
                                   float pad_value, int32_t scheme, int32_t k, float sigma, float mu,
                                   int32_t reduction, int32_t log_base, float* loss, float* grad, float* scratch,
                                   void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && loss && scratch && B > 0 && S > 0,
                 "arb_lambda_loss: null pointer or bad shape");
  ARB_CHECK_ARGS(scheme >= 0 && scheme <= 7, "arb_lambda_loss: unknown weighing scheme");
  ARB_CHECK_ARGS(reduction == ARB_REDUCTION_SUM || reduction == ARB_REDUCTION_MEAN,
                 "Reduction method can be either sum or mean");
  ARB_CHECK_ARGS(log_base == ARB_LOG_BINARY || log_base == ARB_LOG_NATURAL,
                 "Reduction logarithm base can be either natural or binary");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = slate_smem_bytes(S) + size_t(S) * 4;
  if (smem > MAX_SMEM) { arb_set_error("arb_lambda_loss: slate too long"); return ARB_E_UNSUPPORTED; }
  LambdaCfg cfg{scheme, k, log_base, sigma, mu, eps};
  ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
  if (int rc = launch(lambda_loss_kernel, dim3(B), dim3(256), smem, st, /*pdl=*/false, y_pred, y_true, B, S, pad_value,
                      cfg, scratch, scratch + B, grad))
    return rc;
  return finalize(scratch, scratch + B, B, reduction == ARB_REDUCTION_MEAN ? 1 : 0, loss, grad, size_t(B) * S, st);
}

extern "C" int32_t arb_ranknet(const float* y_pred, const float* y_true, int32_t B, int32_t S, float pad_value,
                               int32_t weight_mode, float* loss, float* grad, float* scratch, void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && loss && scratch && B > 0 && S > 0, "arb_ranknet: null pointer or bad shape");
  ARB_CHECK_ARGS(weight_mode >= 0 && weight_mode <= 2, "arb_ranknet: weight_mode must be 0, 1 or 2");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = size_t(S) * 8 + 256;
  if (smem > MAX_SMEM) { arb_set_error("arb_ranknet: slate too long"); return ARB_E_UNSUPPORTED; }
  {
    ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
    if (int rc = launch(ranknet_kernel, dim3(B), dim3(256), smem, st, /*pdl=*/false, y_pred, y_true, B, S, pad_value,
                        weight_mode, scratch, scratch + B, grad))
      return rc;
  }
  return finalize(scratch, scratch + B, B, 1, loss, grad, size_t(B) * S, st);   // mean over selected pairs
}

extern "C" int32_t arb_pointwise_loss(const float* y_pred, const float* y_true, int32_t B, int32_t S, float pad_value,
                                      int32_t mode, float param, float eps, float* loss, float* grad, float* scratch,
                                      void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && loss && scratch && B > 0 && S > 0, "arb_pointwise_loss: null pointer or bad shape");
  ARB_CHECK_ARGS(mode >= 0 && mode <= 2, "arb_pointwise_loss: mode must be 0 (binary_listNet), 1 (rmse) or 2 (bce)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int wpb = 4;
  {
    ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
    if (int rc = launch(pointwise_warp_kernel, dim3((B + wpb - 1) / wpb), dim3(wpb * 32), 0, st, /*pdl=*/false, y_pred,
                        y_true, B, S, pad_value, mode, param, eps, 1.0f / float(B), scratch, scratch + B, grad))
      return rc;
  }
  // binary_listNet / rmse: mean over the batch is already folded in; bce: divide by the number of non-empty slates
  return finalize(scratch, scratch + B, B, mode == 2 ? 1 : 0, loss, grad, size_t(B) * S, st);
}

extern "C" int32_t arb_ordinal(const float* y_pred, const float* y_true, int32_t B, int32_t S, int32_t n,
                               float pad_value, float* loss, float* grad, float* scratch, void* stream) {
  ARB_CHECK_ARGS(y_pred && y_true && loss && scratch && B > 0 && S > 0 && n > 0, "arb_ordinal: null pointer or bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int wpb = 4;
  {
    ProfScope ps(ARB_PROF_LOSS, double(B) * S * ((grad ? 8.0 : 4.0) * n + 4.0) + 4.0, st);
    if (int rc = launch(ordinal_warp_kernel, dim3((B + wpb - 1) / wpb), dim3(wpb * 32), 0, st, /*pdl=*/false, y_pred,
                        y_true, B, S, n, pad_value, scratch, scratch + B, grad))
      return rc;
  }
  return finalize(scratch, scratch + B, B, 1, loss, grad, size_t(B) * S * n, st);   // / total number of valid items
}
