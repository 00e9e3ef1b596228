// neuralNDCG: NeuralSort relaxation + Sinkhorn scaling + soft DCG, forward and backward in one launch.
//
// Reference: allrank/models/losses/neuralNDCG.py:10-70, loss_utils.py:8-31 (sinkhorn_scaling),
//            loss_utils.py:34-67 (deterministic_neural_sort).
//
// The reference materialises [B,S,S] tensors for NeuralSort and for each of the 50 Sinkhorn iterations
// under autograd (146 MB per slate at S=240).  Here one CTA owns one slate and keeps ONE matrix:
//
//   M0[j,i] = softmax_i( (coef_j * s_i - rowtot_i) / tau ),   rowtot_i = sum_k |s_i - s_k|     (valid j,i)
//
// because Sinkhorn scaling only ever multiplies rows and columns: after any number of iterations the
// matrix is diag(u) M0 diag(v).  An iteration is two mat-vecs (column sums, row sums); the clamp(min=1e-10)
// of loss_utils.py:22-23 is a clamp on those sums and is reproduced exactly on the scale vectors.  The
// padded block (mask x mask, filled with ones) is decoupled from the valid block and multiplied by zero at
// the end (neuralNDCG.py:45), so only the n_valid x n_valid block is computed.
//
// Backward is the exact reverse sweep through the (non-converged) iterations: u_t, v_t are saved
// (2*n*T floats), adjoints of M0 accumulate as rank-1 updates in a second matrix, then flow through the
// row softmax and the |s_i - s_k| sums to d loss / d s.   DESIGN.md section 4.5 has the derivation.
//
// Both matrices + history live in shared memory when they fit (n_valid <= ~140 with 50 iterations);
// larger slates use a caller-provided global workspace that stays L2-resident.
#include <cstdint>
#include <cuda_runtime.h>

#include "block_utils.cuh"
#include "common.h"

namespace arb {

struct NeuralCfg {
  float pad, tau, tol;
  int powered, k, max_iter;      // powered: 0 = identity gains, 1 = 2^x-1 gains and ideal DCG,
                                 //          2 = identity gains but 2^x-1 ideal DCG (neuralNDCG_transposed, :126-128)
};

constexpr int NN_THREADS = 256;
constexpr float NN_EPS = 1e-10f;   // DEFAULT_EPS, allrank/models/losses/__init__.py:1

__host__ __device__ inline size_t nn_small_floats(int S) {
  // per-item arrays: pos, s, g, coef, alpha, rowtot, u, v, x, y, xbar(ubar), vbar  + ideal keys + red
  return size_t(S) * 12 + size_t(next_pow2(S)) + 64 + 64;
}
__host__ __device__ inline size_t nn_big_floats(int n, int T, bool need_grad) {
  const size_t pitch = size_t(n) | 1;
  return need_grad ? 2 * size_t(n) * pitch + 2 * size_t(n) * size_t(T) : size_t(n) * pitch;
}

__global__ void __launch_bounds__(NN_THREADS) neural_ndcg_kernel(
    const float* __restrict__ y_pred, const float* __restrict__ y_true, int B, int S,
    const float* __restrict__ discounts, NeuralCfg cfg, float* __restrict__ val, float* __restrict__ cnt,
    float* __restrict__ grad, float* __restrict__ ws, size_t ws_stride, size_t smem_big_floats) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, NW = NN_THREADS / 32;
  const bool need_grad = grad != nullptr;
  const int T = cfg.max_iter;

  float* f = reinterpret_cast<float*>(smem_raw);
  int* pos = reinterpret_cast<int*>(f);  f += S;
  float* s = f;       f += S;
  float* g = f;       f += S;
  float* coef = f;    f += S;
  float* alpha = f;   f += S;
  float* rowtot = f;  f += S;
  float* u = f;       f += S;
  float* v = f;       f += S;
  float* xa = f;      f += S;
  float* xb = f;      f += S;
  float* ubar = f;    f += S;
  float* vbar = f;    f += S;
  uint32_t* ikeys = reinterpret_cast<uint32_t*>(f);  f += next_pow2(S);
  float* red = f;     f += 64;
  int* ishare = reinterpret_cast<int*>(f);  f += 64;
  float* big = f;

  const float* yp = y_pred + size_t(b) * S;
  const float* yt = y_true + size_t(b) * S;

  // ---- compact the valid items (any mask pattern; allRank pads at the tail) ----
  const int np2 = next_pow2(S);
  for (int i = tid; i < np2; i += NN_THREADS) {
    if (i < S) {
      const float lab = yt[i];
      ikeys[i] = ~float_to_ordered(lab == cfg.pad ? -CUDART_INF_F : lab);
    } else {
      ikeys[i] = ~0u;
    }
  }
  if (tid == 0) {
    int n = 0;
    for (int i = 0; i < S; ++i)
      if (yt[i] != cfg.pad) pos[n++] = i;
    ishare[0] = n;
  }
  __syncthreads();
  const int n = ishare[0];
  bitonic_sort(ikeys, np2);
  const int kk = (cfg.k <= 0 || cfg.k > S) ? S : cfg.k;

  // ideal DCG@k exactly like metrics.dcg(y_true, y_true, ats=[k]) (sequential double accumulation)
  if (tid == 0) {
    double acc = 0.0;
    for (int j = 0; j < kk; ++j) {
      uint32_t o = ~ikeys[j];
      float lab = __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
      if (lab == -CUDART_INF_F) lab = 0.0f;
      const float gain = cfg.powered != 0 ? pow2_minus_1(lab) : lab;
      acc += double(gain * discounts[j]);
    }
    red[32] = float(acc);
  }
  __syncthreads();
  const float idcg = red[32];
  if (idcg == 0.0f || n == 0) {   // neuralNDCG.py:62-63: slate contributes 0 and is left out of the mean
    if (tid == 0) { val[b] = 0.0f; cnt[b] = 0.0f; }
    if (need_grad) for (int i = tid; i < S; i += NN_THREADS) grad[size_t(b) * S + i] = 0.0f;
    return;
  }

  const size_t pitch = size_t(n) | 1;
  const bool fits = nn_big_floats(n, T, need_grad) <= smem_big_floats;
  float* base = fits ? big : (ws + size_t(b) * ws_stride);
  float* M0 = base;
  float* Mb = need_grad ? base + size_t(n) * pitch : nullptr;
  float* hist_u = need_grad ? base + 2 * size_t(n) * pitch : nullptr;
  float* hist_v = need_grad ? hist_u + size_t(n) * T : nullptr;

  const float inv_tau = 1.0f / cfg.tau;
  for (int a = tid; a < n; a += NN_THREADS) {
    const int p = pos[a];
    const float lab = yt[p];
    s[a] = yp[p];
    g[a] = cfg.powered == 1 ? pow2_minus_1(lab) : lab;
    coef[a] = (p < n) ? float(n + 1 - 2 * (p + 1)) : 0.0f;           // loss_utils.py:54-56
    alpha[a] = (p < kk) ? -discounts[p] / (idcg + NN_EPS) : 0.0f;    // neuralNDCG.py:53-61
    u[a] = 1.0f;
    v[a] = 1.0f;
  }
  __syncthreads();
  for (int a = tid; a < n; a += NN_THREADS) {
    const float sa = s[a];
    float acc = 0.f;
    for (int c = 0; c < n; ++c) acc += fabsf(sa - s[c]);
    rowtot[a] = acc;
  }
  __syncthreads();

  // ---- M0: row softmax of the NeuralSort logits; one warp per rank row ----
  for (int j = wid; j < n; j += NW) {
    const float cj = coef[j];
    float mx = -CUDART_INF_F;
    for (int i = lane; i < n; i += 32) {
      const float l = (cj * s[i] - rowtot[i]) / cfg.tau;
      M0[j * pitch + i] = l;
      mx = fmaxf(mx, l);
    }
    mx = warp_max(mx);
    float z = 0.f;
    for (int i = lane; i < n; i += 32) {
      const float e = expf(M0[j * pitch + i] - mx);
      M0[j * pitch + i] = e;
      z += e;
    }
    z = warp_sum(z);
    for (int i = lane; i < n; i += 32) M0[j * pitch + i] = M0[j * pitch + i] / z;
  }
  __syncthreads();

  // ---- Sinkhorn iterations on the scale vectors ----
  int iters = 0;
  for (int t = 0; t < T; ++t) {
    // column sums of diag(u) M0 diag(v)
    float dev = 0.f;
    for (int i = tid; i < n; i += NN_THREADS) {
      float acc = 0.f;
      for (int j = 0; j < n; ++j) acc += u[j] * M0[j * pitch + i];
      const float cs = v[i] * acc;
      xa[i] = cs;
      dev = fmaxf(dev, fabsf(cs - 1.0f));
    }
    dev = block_max(dev, red);
    if (t > 0 && dev < cfg.tol) break;   // loss_utils.py:25-26 (per slate here; the reference tests the whole batch)
    for (int i = tid; i < n; i += NN_THREADS) {
      const float cs = xa[i];
      const bool clamped = cs < NN_EPS;
      v[i] = v[i] / (clamped ? NN_EPS : cs);
      if (need_grad) hist_v[size_t(t) * n + i] = clamped ? -v[i] : v[i];
    }
    __syncthreads();
    // row sums, one warp per row
    for (int j = wid; j < n; j += NW) {
      float acc = 0.f;
      for (int i = lane; i < n; i += 32) acc += M0[j * pitch + i] * v[i];
      acc = warp_sum(acc);
      if (lane == 0) {
        const float rs = u[j] * acc;
        const bool clamped = rs < NN_EPS;
        const float un = u[j] / (clamped ? NN_EPS : rs);
        u[j] = un;
        if (need_grad) hist_u[size_t(t) * n + j] = clamped ? -un : un;
      }
    }
    __syncthreads();
    iters = t + 1;
  }
  __syncthreads();

  // ---- soft DCG: loss_b = sum_j alpha_j u_j sum_i M0[j,i] v_i g_i ----
  float lossb = 0.f;
  for (int j = wid; j < n; j += NW) {
    float acc = 0.f;
    for (int i = lane; i < n; i += 32) acc += M0[j * pitch + i] * v[i] * g[i];
    acc = warp_sum(acc);
    if (lane == 0) {
      lossb += alpha[j] * u[j] * acc;
      ubar[j] = alpha[j] * acc;                 // d loss_b / d u_j
    }
  }
  lossb = block_sum(lossb, red);
  if (tid == 0) { val[b] = lossb; cnt[b] = 1.0f; }
  if (!need_grad) return;

  // d loss_b / d v_i and the first rank-1 term of Mbar
  for (int i = tid; i < n; i += NN_THREADS) {
    float acc = 0.f;
    for (int j = 0; j < n; ++j) acc += alpha[j] * u[j] * M0[j * pitch + i];
    vbar[i] = g[i] * acc;
    xb[i] = v[i] * g[i];
  }
  for (int j = tid; j < n; j += NN_THREADS) xa[j] = alpha[j] * u[j];
  __syncthreads();
  for (int j = wid; j < n; j += NW)
    for (int i = lane; i < n; i += 32) Mb[j * pitch + i] = xa[j] * xb[i];
  __syncthreads();

  // ---- reverse sweep through the Sinkhorn iterations ----
  for (int t = iters - 1; t >= 0; --t) {
    // row step: u_t = u_{t-1} / max(rs, eps), rs = u_{t-1} * (M0 v_t)
    //   unclamped: u_t = 1/(M0 v_t)  ->  bbar = -ubar * u_t^2 ; clamped: u_t = u_{t-1}/eps
    const float* ut = hist_u + size_t(t) * n;
    const float* vt = hist_v + size_t(t) * n;
    for (int j = tid; j < n; j += NN_THREADS) {
      const float uj = ut[j];
      if (uj < 0.f) { xa[j] = 0.f; ubar[j] = ubar[j] / NN_EPS; }   // flows straight to u_{t-1}
      else          { xa[j] = -ubar[j] * uj * uj; ubar[j] = 0.f; }
    }
    __syncthreads();
    // vbar_t += M0^T bbar ; Mbar += bbar v_t^T
    for (int i = tid; i < n; i += NN_THREADS) {
      float acc = 0.f;
      for (int j = 0; j < n; ++j) acc += xa[j] * M0[j * pitch + i];
      vbar[i] += acc;
    }
    for (int j = wid; j < n; j += NW) {
      const float bj = xa[j];
      if (bj != 0.f)
        for (int i = lane; i < n; i += 32) Mb[j * pitch + i] += bj * fabsf(vt[i]);
    }
    __syncthreads();
    // column step: v_t = v_{t-1} / max(cs, eps), cs = v_{t-1} * (M0^T u_{t-1})
    const float* up = (t > 0) ? hist_u + size_t(t - 1) * n : nullptr;   // u_{t-1} (all ones before iteration 0)
    for (int i = tid; i < n; i += NN_THREADS) {
      const float vi = vt[i];
      if (vi < 0.f) { xb[i] = 0.f; vbar[i] = vbar[i] / NN_EPS; }   // to v_{t-1}
      else          { xb[i] = -vbar[i] * vi * vi; vbar[i] = 0.f; }
    }
    __syncthreads();
    // ubar_{t-1} += M0 abar ; Mbar += u_{t-1} abar^T
    for (int j = wid; j < n; j += NW) {
      const float uj = up ? fabsf(up[j]) : 1.0f;
      float acc = 0.f;
      for (int i = lane; i < n; i += 32) {
        const float ai = xb[i];
        acc += M0[j * pitch + i] * ai;
        Mb[j * pitch + i] += uj * ai;
      }
      acc = warp_sum(acc);
      if (lane == 0) ubar[j] += acc;
    }
    __syncthreads();
  }

  // ---- row softmax backward: lbar[j,i] = M0[j,i] (Mbar[j,i] - <M0[j,:], Mbar[j,:]>) ----
  for (int j = wid; j < n; j += NW) {
    float dot = 0.f;
    for (int i = lane; i < n; i += 32) dot += M0[j * pitch + i] * Mb[j * pitch + i];
    dot = warp_sum(dot);
    for (int i = lane; i < n; i += 32) Mb[j * pitch + i] = M0[j * pitch + i] * (Mb[j * pitch + i] - dot);
  }
  __syncthreads();
  // logits l[j,i] = (coef_j s_i - rowtot_i)/tau:   direct_i = sum_j lbar coef_j / tau ;  rbar_i = -sum_j lbar / tau
  for (int i = tid; i < n; i += NN_THREADS) {
    float d = 0.f, r = 0.f;
    for (int j = 0; j < n; ++j) {
      const float lb = Mb[j * pitch + i];
      d += lb * coef[j];
      r += lb;
    }
    xa[i] = d * inv_tau;
    xb[i] = -r * inv_tau;
  }
  __syncthreads();
  // rowtot_i = sum_k |s_i - s_k|  ->  sbar_m = direct_m + sum_i (rbar_m + rbar_i) sign(s_m - s_i)
  for (int i = tid; i < S; i += NN_THREADS) grad[size_t(b) * S + i] = 0.0f;
  __syncthreads();
  for (int m = tid; m < n; m += NN_THREADS) {
    const float sm = s[m], rm = xb[m];
    float acc = xa[m];
    for (int i = 0; i < n; ++i) {
      const float d = sm - s[i];
      const float sg = (d > 0.f) ? 1.0f : (d < 0.f ? -1.0f : 0.0f);
      acc += (rm + xb[i]) * sg;
    }
    grad[size_t(b) * S + pos[m]] = acc;
  }
}


// ------------------------------------------------------------------------------------------------ register-tiled variant
// Slates with at most 128 items (BASELINE config 4: S = 120): the whole n x n matrix M0 and its adjoint live in the
// REGISTERS of a 1024-thread CTA -- warp w owns rows {w, w+32, w+64, w+96}, lane l owns columns {l, l+32, l+64,
// l+96}, 4 x 4 elements per thread.  A Sinkhorn iteration is then 16 FMAs per thread plus one warp-shuffle row
// reduction and one shared-memory column reduction; nothing of size n^2 is read from shared memory inside the
// 2 x 50 iteration loops (the generic kernel above re-reads the matrix from shared memory ~300 times per slate).
constexpr int RG_THREADS = 1024;
constexpr int RG_N = 128;

__host__ __device__ inline size_t rg_smem_bytes(int T) {
  return (size_t(12) * RG_N + RG_N /*ikeys*/ + 64 + 8 + 2 * 32 * RG_N /*part,part2*/ + 2 * size_t(T) * RG_N) * 4 + 64;
}

__global__ void __launch_bounds__(RG_THREADS, 1) neural_ndcg_reg_kernel(
    const float* __restrict__ y_pred, const float* __restrict__ y_true, int B, int S,
    const float* __restrict__ discounts, NeuralCfg cfg, float* __restrict__ val, float* __restrict__ cnt,
    float* __restrict__ grad, float* __restrict__ dump_p0, float* __restrict__ dump_p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  const int tid = threadIdx.x, l = tid & 31, w = tid >> 5;
  const bool need_grad = grad != nullptr;
  const int T = cfg.max_iter;

  float* f = reinterpret_cast<float*>(smem_raw);
  int* pos = reinterpret_cast<int*>(f);  f += RG_N;
  float* s = f;       f += RG_N;
  float* g = f;       f += RG_N;
  float* coef = f;    f += RG_N;
  float* alpha = f;   f += RG_N;
  float* rowtot = f;  f += RG_N;
  float* u = f;       f += RG_N;
  float* v = f;       f += RG_N;
  float* xa = f;      f += RG_N;
  float* xb = f;      f += RG_N;
  float* ubar = f;    f += RG_N;
  float* vbar = f;    f += RG_N;
  uint32_t* ikeys = reinterpret_cast<uint32_t*>(f);  f += RG_N;
  float* red = f;     f += 64;
  int* ishare = reinterpret_cast<int*>(f);  f += 8;
  float* part = f;    f += 32 * RG_N;
  float* part2 = f;   f += 32 * RG_N;
  float* hist_u = f;  f += size_t(T) * RG_N;
  float* hist_v = f;

  const float* yp = y_pred + size_t(b) * S;
  const float* yt = y_true + size_t(b) * S;

  const int np2 = next_pow2(S);
  for (int i = tid; i < np2; i += RG_THREADS) {
    if (i < S) {
      const float lab = yt[i];
      ikeys[i] = ~float_to_ordered(lab == cfg.pad ? -CUDART_INF_F : lab);
    } else {
      ikeys[i] = ~0u;
    }
  }
  if (tid == 0) {
    int n = 0;
    for (int i = 0; i < S; ++i)
      if (yt[i] != cfg.pad) pos[n++] = i;
    ishare[0] = n;
  }
  __syncthreads();
  const int n = ishare[0];
  bitonic_sort(ikeys, np2);
  const int kk = (cfg.k <= 0 || cfg.k > S) ? S : cfg.k;
  if (tid == 0) {
    double acc = 0.0;
    for (int j = 0; j < kk; ++j) {
      uint32_t o = ~ikeys[j];
      float lab = __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
      if (lab == -CUDART_INF_F) lab = 0.0f;
      const float gain = cfg.powered != 0 ? pow2_minus_1(lab) : lab;
      acc += double(gain * discounts[j]);
    }
    red[32] = float(acc);
  }
  __syncthreads();
  const float idcg = red[32];
  if (idcg == 0.0f || n == 0) {
    if (tid == 0) { val[b] = 0.0f; cnt[b] = 0.0f; }
    if (need_grad) for (int i = tid; i < S; i += RG_THREADS) grad[size_t(b) * S + i] = 0.0f;
    return;
  }
  for (int a = tid; a < RG_N; a += RG_THREADS) {
    if (a < n) {
      const int p = pos[a];
      const float lab = yt[p];
      s[a] = yp[p];
      g[a] = cfg.powered == 1 ? pow2_minus_1(lab) : lab;
      coef[a] = (p < n) ? float(n + 1 - 2 * (p + 1)) : 0.0f;
      alpha[a] = (p < kk) ? -discounts[p] / (idcg + NN_EPS) : 0.0f;
    } else {
      s[a] = 0.f; g[a] = 0.f; coef[a] = 0.f; alpha[a] = 0.f;
    }
    u[a] = 1.0f; v[a] = 1.0f; ubar[a] = 0.f; vbar[a] = 0.f; xa[a] = 0.f; xb[a] = 0.f;
  }
  __syncthreads();
  for (int a = tid; a < RG_N; a += RG_THREADS) {
    float acc = 0.f;
    if (a < n) {
      const float sa = s[a];
      for (int c = 0; c < n; ++c) acc += fabsf(sa - s[c]);
    }
    rowtot[a] = acc;
  }
  __syncthreads();

  // ---- M0 in registers: m0[k][c] = element (row w+32k, column l+32c)
  float m0[4][4], mb[4][4];
  bool rok[4], cok[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { rok[k] = (w + 32 * k) < n; cok[k] = (l + 32 * k) < n; }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float cj = coef[w + 32 * k];
    float mx = -CUDART_INF_F;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int i = l + 32 * c;
      const float lg = (cj * s[i] - rowtot[i]) / cfg.tau;
      m0[k][c] = (rok[k] && cok[c]) ? lg : -CUDART_INF_F;
      mx = fmaxf(mx, m0[k][c]);
    }
    mx = warp_max(mx);
    float z = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float e = (rok[k] && cok[c]) ? expf(m0[k][c] - mx) : 0.0f;
      m0[k][c] = e;
      z += e;
    }
    z = warp_sum(z);
#pragma unroll
    for (int c = 0; c < 4; ++c) m0[k][c] = rok[k] ? m0[k][c] / z : 0.0f;
  }

  // debug dump (arb_neural_sort_debug): the NeuralSort matrix P_hat[rank j, item i] of the real items, in the slate's
  // own [S, S] layout (loss_utils.py:34-67); rows / columns of padded items stay as the caller initialised them
  if (dump_p0) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (rok[k] && cok[c]) dump_p0[(size_t(b) * S + (w + 32 * k)) * S + pos[l + 32 * c]] = m0[k][c];
  }

  // column reduction helper: per-thread partials over its 4 rows -> sums over all rows, result in dst[0..127]
  auto col_reduce = [&](const float (&cp)[4], float* scratch, float* dst) {
#pragma unroll
    for (int c = 0; c < 4; ++c) scratch[w * RG_N + l + 32 * c] = cp[c];
    __syncthreads();
    if (tid < RG_N) {
      float t = 0.f;
#pragma unroll 8
      for (int ww = 0; ww < 32; ++ww) t += scratch[ww * RG_N + tid];
      dst[tid] = t;
    }
    __syncthreads();
  };

  // ---- Sinkhorn iterations on the scale vectors
  int iters = 0;
  for (int t = 0; t < T; ++t) {
    float cp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float uk = u[w + 32 * k];
#pragma unroll
      for (int c = 0; c < 4; ++c) cp[c] += uk * m0[k][c];
    }
    col_reduce(cp, part, xa);                      // xa[i] = sum_j u_j M0[j,i]
    float dev = 0.f;
    if (tid < RG_N) {
      const float cs = (tid < n) ? v[tid] * xa[tid] : 1.0f;
      xa[tid] = cs;
      dev = fabsf(cs - 1.0f);
      dev = warp_max(dev);
      if (l == 0) red[w] = dev;
    }
    __syncthreads();
    dev = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    if (t > 0 && dev < cfg.tol) break;
    if (tid < n) {
      const float cs = xa[tid];
      const bool clamped = cs < NN_EPS;
      const float vn = v[tid] / (clamped ? NN_EPS : cs);
      v[tid] = vn;
      if (need_grad) hist_v[size_t(t) * RG_N + tid] = clamped ? -vn : vn;
    }
    __syncthreads();
    float vc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) vc[c] = v[l + 32 * c];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float rp = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) rp += m0[k][c] * vc[c];
      rp = warp_sum(rp);
      const int j = w + 32 * k;
      if (l == 0 && j < n) {
        const float rs = u[j] * rp;
        const bool clamped = rs < NN_EPS;
        const float un = u[j] / (clamped ? NN_EPS : rs);
        u[j] = un;
        if (need_grad) hist_u[size_t(t) * RG_N + j] = clamped ? -un : un;
      }
    }
    __syncthreads();
    iters = t + 1;
  }
  __syncthreads();

  if (dump_p) {   // the Sinkhorn-scaled matrix diag(u) M0 diag(v) (loss_utils.py:8-31)
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (rok[k] && cok[c])
          dump_p[(size_t(b) * S + (w + 32 * k)) * S + pos[l + 32 * c]] = u[w + 32 * k] * m0[k][c] * v[l + 32 * c];
  }

  // ---- soft DCG and the adjoints of u, v, M0 at the end of the iterations
  float lossb = 0.f;
  {
    float vg[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) vg[c] = v[l + 32 * c] * g[l + 32 * c];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float acc = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) acc += m0[k][c] * vg[c];
      acc = warp_sum(acc);
      const int j = w + 32 * k;
      if (l == 0 && j < n) {
        lossb += alpha[j] * u[j] * acc;
        ubar[j] = alpha[j] * acc;
      }
    }
  }
  lossb = block_sum(lossb, red);
  if (tid == 0) { val[b] = lossb; cnt[b] = 1.0f; }
  if (!need_grad) return;
  {
    float cp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = w + 32 * k;
      const float au = alpha[j] * u[j];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        cp[c] += au * m0[k][c];
        mb[k][c] = au * (v[l + 32 * c] * g[l + 32 * c]);
      }
    }
    col_reduce(cp, part, xb);
    if (tid < RG_N) vbar[tid] = g[tid] * xb[tid];
    __syncthreads();
  }

  // ---- reverse sweep
  for (int t = iters - 1; t >= 0; --t) {
    const float* ut = hist_u + size_t(t) * RG_N;
    const float* vt = hist_v + size_t(t) * RG_N;
    if (tid < RG_N) {
      float x = 0.f;
      if (tid < n) {
        const float uj = ut[tid];
        if (uj < 0.f) { x = 0.f; ubar[tid] = ubar[tid] / NN_EPS; }
        else          { x = -ubar[tid] * uj * uj; ubar[tid] = 0.f; }
      }
      xa[tid] = x;
    }
    __syncthreads();
    {
      float cp[4] = {0.f, 0.f, 0.f, 0.f};
      float vtc[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) vtc[c] = cok[c] ? fabsf(vt[l + 32 * c]) : 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float bj = xa[w + 32 * k];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          cp[c] += bj * m0[k][c];
          mb[k][c] += bj * vtc[c];
        }
      }
      col_reduce(cp, part, xb);                    // xb[i] = (M0^T bbar)_i
    }
    if (tid < RG_N) {
      float x = 0.f;
      if (tid < n) {
        const float vb = vbar[tid] + xb[tid];
        const float vi = vt[tid];
        if (vi < 0.f) { x = 0.f; vbar[tid] = vb / NN_EPS; }
        else          { x = -vb * vi * vi; vbar[tid] = 0.f; }
      }
      xb[tid] = x;                                  // abar
    }
    __syncthreads();
    {
      const float* up = (t > 0) ? hist_u + size_t(t - 1) * RG_N : nullptr;
      float ab[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) ab[c] = xb[l + 32 * c];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int j = w + 32 * k;
        const float uj = (j < n) ? (up ? fabsf(up[j]) : 1.0f) : 0.0f;
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          acc += m0[k][c] * ab[c];
          mb[k][c] += uj * ab[c];
        }
        acc = warp_sum(acc);
        if (l == 0 && j < n) ubar[j] += acc;
      }
    }
    __syncthreads();
  }

  // ---- row softmax backward, then logits -> scores
  {
    float cpd[4] = {0.f, 0.f, 0.f, 0.f}, cpr[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float dot = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) dot += m0[k][c] * mb[k][c];
      dot = warp_sum(dot);
      const float cj = coef[w + 32 * k];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float lb = m0[k][c] * (mb[k][c] - dot);
        cpd[c] += lb * cj;
        cpr[c] += lb;
      }
    }
    col_reduce(cpd, part, xa);
    col_reduce(cpr, part2, xb);
  }
  const float inv_tau = 1.0f / cfg.tau;
  if (tid < RG_N) {
    xa[tid] = xa[tid] * inv_tau;       // direct_i
    xb[tid] = -xb[tid] * inv_tau;      // rbar_i
  }
  for (int i = tid; i < S; i += RG_THREADS) grad[size_t(b) * S + i] = 0.0f;
  __syncthreads();
  if (tid < n) {
    const float sm = s[tid], rm = xb[tid];
    float acc = xa[tid];
    for (int i = 0; i < n; ++i) {
      const float d = sm - s[i];
      const float sg = (d > 0.f) ? 1.0f : (d < 0.f ? -1.0f : 0.0f);
      acc += (rm + xb[i]) * sg;
    }
    grad[size_t(b) * S + pos[tid]] = acc;
  }
}

}  // namespace arb

using namespace arb;

static size_t nn_smem_budget() { return 220 * 1024; }

extern "C" size_t arb_neural_ndcg_workspace_bytes(int32_t B, int32_t S, int32_t max_iter) {
  if (B <= 0 || S <= 0) return 0;
  const size_t small = nn_small_floats(S) * 4;
  const size_t big = nn_big_floats(S, max_iter, true) * 4;
  if (S <= RG_N && rg_smem_bytes(max_iter) <= nn_smem_budget()) return 0;
  if (small + big <= nn_smem_budget()) return 0;
  return size_t(B) * big;
}

extern "C" int32_t arb_neural_ndcg(const float* y_pred, const float* y_true, int32_t B, int32_t S,
                                      const float* discounts, float pad_value, float temperature,
                                      int32_t powered_relevancies, int32_t k, int32_t max_iter, float tol,
                                      float* loss, float* grad, float* scratch, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  if (!(y_pred && y_true && discounts && loss && scratch && B > 0 && S > 0 && max_iter >= 0 && temperature > 0.f)) {
    arb_set_error("arb_neural_ndcg: null pointer or bad argument");
    return ARB_E_INVALID_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (S <= RG_N && rg_smem_bytes(max_iter) <= nn_smem_budget()) {
    // register-tiled kernel: the whole matrix and its adjoint stay in the registers of a 1024-thread CTA
    const size_t smem_rg = rg_smem_bytes(max_iter);
    NeuralCfg cfg_rg{pad_value, temperature, tol, powered_relevancies, k, max_iter};
    {
      ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
      if (int rc = launch(neural_ndcg_reg_kernel, dim3(B), dim3(RG_THREADS), smem_rg, st, /*pdl=*/false, y_pred, y_true,
                          B, S, discounts, cfg_rg, scratch, scratch + B, grad, nullptr, nullptr))
        return rc;
    }
    return arb_finalize_mean_over_count(scratch, scratch + B, B, loss, grad, size_t(B) * S, st);
  }
  const size_t small = nn_small_floats(S) * 4;
  if (small > nn_smem_budget()) { arb_set_error("arb_neural_ndcg: slate too long"); return ARB_E_UNSUPPORTED; }
  const size_t big_all = nn_big_floats(S, max_iter, grad != nullptr) * 4;
  size_t smem = std::min(small + big_all, nn_smem_budget());
  const size_t smem_big_floats = (smem - small) / 4;
  const size_t need_ws = arb_neural_ndcg_workspace_bytes(B, S, max_iter);
  if (small + big_all > nn_smem_budget()) {
    if (!workspace || workspace_bytes < need_ws) {
      arb_set_error("arb_neural_ndcg: workspace too small (see arb_neural_ndcg_workspace_bytes)");
      return ARB_E_WORKSPACE;
    }
  }
  NeuralCfg cfg{pad_value, temperature, tol, powered_relevancies, k, max_iter};
  const size_t ws_stride = nn_big_floats(S, max_iter, true);
  ProfScope ps(ARB_PROF_LOSS, double(B) * ((grad ? 12.0 : 8.0) * S + 4.0), st);
  if (int rc = launch(neural_ndcg_kernel, dim3(B), dim3(NN_THREADS), smem, st, /*pdl=*/false, y_pred, y_true, B, S,
                      discounts, cfg, scratch, scratch + B, grad, static_cast<float*>(workspace), ws_stride,
                      smem_big_floats))
    return rc;
  // mean over the slates with idcg != 0 (neuralNDCG.py:69); all-dead batch -> 0 (:66-67)
  return arb_finalize_mean_over_count(scratch, scratch + B, B, loss, grad, size_t(B) * S, st);
}

// Debug / parity hook for SURVEY.md 8(a) rows a17, a18: the matrices the fused neuralNDCG kernel works with, for slates of
// at most 128 items -- p0_out = deterministic_neural_sort(y_pred, tau, mask) and p_out = sinkhorn_scaling(p0, mask, tol,
// max_iter) restricted to the real items (entries of padded rows / columns are left untouched: pass zero-filled
// [B,S,S] buffers).  Slates without a relevant item are skipped by the kernel (left untouched too).
extern "C" int32_t arb_neural_sort_debug(const float* y_pred, const float* y_true, int32_t B, int32_t S,
                                         const float* discounts, float pad_value, float temperature, int32_t max_iter,
                                         float tol, float* p0_out, float* p_out, float* scratch, void* stream) {
  if (!(y_pred && y_true && discounts && p0_out && p_out && scratch && B > 0 && S > 0 && max_iter >= 0 && temperature > 0.f)) {
    arb_set_error("arb_neural_sort_debug: null pointer or bad argument");
    return ARB_E_INVALID_ARG;
  }
  if (S > RG_N || rg_smem_bytes(max_iter) > nn_smem_budget()) {
    arb_set_error("arb_neural_sort_debug: serves slates of at most 128 items");
    return ARB_E_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  NeuralCfg cfg{pad_value, temperature, tol, 1, 0, max_iter};
  return launch(neural_ndcg_reg_kernel, dim3(B), dim3(RG_THREADS), rg_smem_bytes(max_iter), st, /*pdl=*/false, y_pred,
                y_true, B, S, discounts, cfg, scratch, scratch + B, nullptr, p0_out, p_out);
}
