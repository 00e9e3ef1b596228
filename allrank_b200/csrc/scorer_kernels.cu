// SIMT kernels of the scorer (everything that is not a tensor-core contraction):
//   row LayerNorm forward / backward (the reference's custom LayerNorm: unbiased std, eps added to the std,
//   allrank/models/transformer.py:59-81), key-masked row softmax forward / backward (transformer.py:148-153),
//   bias-gradient column sums, final LayerNorm + linear head forward / backward (model.py:111-117).
// The LayerNorm and head kernels give each row 8, 16 or 32 lanes by width (the row layout below), the others a warp per
// row; coalesced 128-bit accesses where the width allows, warp-shuffle reductions; they are HBM-bound (DESIGN.md
// section 3 lists bytes per row).
#include <cstdint>
#include <string>
#include <type_traits>
#include <cuda_runtime.h>

#include "block_utils.cuh"
#include "common.h"
#include "dropout.cuh"
#include "scorer_kernels.h"

namespace arb {

constexpr int ROWS_PER_BLOCK = 8;   // 8 warps

// ------------------------------------------------------------------------------------------------ row layout
// The row kernels give each row LPR lanes: a lane owns NJ float4 of ONE row, float4 j at column
// ((lane % LPR) + LPR * j) * 4, so that the LPR lanes of a row read LPR * 16 contiguous bytes per instruction and a
// warp holds 32 / LPR rows at once.  A row reduction is log2(LPR) shuffle steps that serve all rows of the warp at once
// (one row per warp needs five steps per row and reduction: ncu put the LayerNorm forward at 75 % issue-active with
// shuffles and their adds a third of it).  A lane's columns reach the capacity 4 * LPR * NJ; those at or beyond the
// width are masked: loads give 0, stores skip them.
// LayerNorm and the head take (LPR, NJ) = (8, 4) up to W = 128, (16, 4) up to 256, (32, 4) up to 512 and (32, 8) up
// to 1024 (with_row_layout); the column sums and the multi-output head keep one row per warp (LPR = 32,
// NJ = ceil(W / 128)).
template <int LPR>
__device__ __forceinline__ int r_col(int lane, int j) { return ((lane % LPR) + LPR * j) * 4; }
template <int LPR>
__device__ __forceinline__ float r_sum(float v) {
#pragma unroll
  for (int off = 1; off < LPR; off <<= 1) v += __shfl_xor_sync(FULL, v, off);
  return v;
}
template <int LPR, int NJ>
__device__ __forceinline__ void r_load(const float* __restrict__ row, int width, int lane, float4 (&v)[NJ]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = r_col<LPR>(lane, j);
    v[j] = c < width ? *reinterpret_cast<const float4*>(row + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
template <int LPR, int NJ>
__device__ __forceinline__ void r_store(float* __restrict__ row, int width, int lane, const float4 (&v)[NJ]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = r_col<LPR>(lane, j);
    if (c < width) *reinterpret_cast<float4*>(row + c) = v[j];
  }
}

// bf16 rows (the scorer's bf16 mode keeps GEMM operands -- LayerNorm outputs, hidden activations, the gradients that
// feed weight / input-gradient products -- as bfloat16): a lane's 4 elements are 8 bytes.
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
template <int LPR, int NJ>
__device__ __forceinline__ void r_load_bf16(const uint16_t* __restrict__ row, int width, int lane, float4 (&v)[NJ]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = r_col<LPR>(lane, j);
    if (c < width) {
      const uint2 u = *reinterpret_cast<const uint2*>(row + c);
      v[j] = make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                         __uint_as_float(u.y & 0xffff0000u));
    } else {
      v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}
template <int LPR, int NJ>
__device__ __forceinline__ void r_store_bf16(uint16_t* __restrict__ row, int width, int lane, const float4 (&v)[NJ]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = r_col<LPR>(lane, j);
    if (c < width)
      *reinterpret_cast<uint2*>(row + c) = make_uint2(pack_bf16x2(v[j].x, v[j].y), pack_bf16x2(v[j].z, v[j].w));
  }
}
template <int NJ>
__device__ __forceinline__ void r_zero(float4 (&v)[NJ]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
}
// dropout counter row * width + column: the same as the GEMM epilogues'
template <int LPR, int NJ>
__device__ __forceinline__ void r_drop(float4 (&v)[NJ], long long row, int width, int lane, const DropSite& site) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    float* e = &v[j].x;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const unsigned long long idx = (unsigned long long)row * (unsigned long long)width + (r_col<LPR>(lane, j) + t);
      e[t] = drop_keep(idx, site.seed, site.thresh) ? e[t] * site.scale : 0.0f;
    }
  }
}
// sum the per-column accumulators of the warp's row groups, then over the block's warps, then into the block's slot of
// `dst` (DetParts)
template <int LPR, int NJ>
__device__ __forceinline__ void r_reduce_columns(float4 (&acc)[NJ], float (*sh)[4 * LPR * NJ + 4], int width, int lane,
                                                 int wid, float* __restrict__ dst) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    float* e = &acc[j].x;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
#pragma unroll
      for (int off = LPR; off < 32; off <<= 1) e[t] += __shfl_xor_sync(FULL, e[t], off);
    }
  }
  if (lane < LPR) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) *reinterpret_cast<float4*>(&sh[wid][r_col<LPR>(lane, j)]) = acc[j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < ROWS_PER_BLOCK; ++w) t += sh[w][c];
    dst[size_t(blockIdx.x) * width + c] = t;        // this block's slot (DetParts)
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ LayerNorm fwd
// y = a * (x - mean) / (std_unbiased + eps) + b ; saves mean and std per row.
// A warp walks `steps` steps of 32 / LPR rows, the loads of the next step issued before the arithmetic of the current
// one: one row per warp leaves only 512 B in flight per warp at d_model = 128, far too little to cover the HBM latency
// (Little's law), and a warp that retires after a single step spends a third of its life waiting for its first loads
// and for a new block to be scheduled.
// MAP: packed rows with a row-mapped output (rowmap_out); a template flag so that the plain kernels compile unchanged
// PAD: a row of n real columns stored at the pitch width = round_up(n, 4) with zero pads (DESIGN.md 4.16): the
// statistics run over the n real columns (the zero pads add nothing to the sum; the squares are masked per element)
// and the zero pads of the gain and bias write +0 into the pads of y; also a template flag
template <int LPR, int NJ, bool FILLED, bool MAP, bool PAD = false>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) ln_fwd_kernel(const float* __restrict__ x,
                                                                    const float* __restrict__ a,
                                                                    const float* __restrict__ b, float eps,
                                                                    long long rows, int width, float* __restrict__ y,
                                                                    float* __restrict__ mean_o,
                                                                    float* __restrict__ std_o, int torch_mode,
                                                                    uint16_t* __restrict__ y16,
                                                                    const int* __restrict__ rows_dev, int steps,
                                                                    const int* __restrict__ rowmap_out, int n) {
  if (FILLED) width = 4 * LPR * NJ;   // (see with_row_layout)
  if (!PAD) n = width;
  arb_pdl_wait();
  constexpr int RW = 32 / LPR;
  const int lane = threadIdx.x & 31, rg = lane / LPR;
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5)) * (RW * steps);
  if (base >= rows) return;
  if (rows_dev) { rows = min(rows, (long long)__ldg(rows_dev)); if (base >= rows) return; }
  float4 ga[NJ], gb[NJ], cur[NJ], nxt[NJ];
  r_load<LPR>(a, width, lane, ga);
  r_load<LPR>(b, width, lane, gb);
  if (base + rg < rows) r_load<LPR>(x + (base + rg) * width, width, lane, cur); else r_zero(cur);
#pragma unroll 1
  for (int s = 0; s < steps; ++s) {
    if (base + (long long)s * RW >= rows) break;
    const long long row = base + (long long)s * RW + rg;
    if (s + 1 < steps) { if (row + RW < rows) r_load<LPR>(x + (row + RW) * width, width, lane, nxt); else r_zero(nxt); }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) sum += cur[j].x + cur[j].y + cur[j].z + cur[j].w;
    const float m = r_sum<LPR>(sum) / float(n);
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = r_col<LPR>(lane, j);
      if (c < width) {
        float d0 = cur[j].x - m, d1 = cur[j].y - m, d2 = cur[j].z - m, d3 = cur[j].w - m;
        if (PAD) { if (c >= n) d0 = 0.f; if (c + 1 >= n) d1 = 0.f; if (c + 2 >= n) d2 = 0.f; if (c + 3 >= n) d3 = 0.f; }
        ss += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
      }
    }
    ss = r_sum<LPR>(ss);
    // torch_mode: nn.LayerNorm (biased variance, eps inside the root; FCModel's input_norm, model.py:27) -- the saved
    // "std" is then sqrt(var + eps) and the backward is called with eps = 0
    const float sdq = torch_mode ? sqrtf(ss / float(n) + eps) : sqrtf(ss / float(n - 1));
    // one reciprocal per row instead of a division per element: the kernel is bound by instruction issue as much as
    // by HBM (an IEEE division is ~10 instructions), and a * (x - mean) * (1 / (std + eps)) differs from the
    // reference's a * (x - mean) / (std + eps) by one rounding (6e-8 relative)
    const float rinv = 1.0f / (torch_mode ? sdq : sdq + eps);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      cur[j].x = ga[j].x * (cur[j].x - m) * rinv + gb[j].x;
      cur[j].y = ga[j].y * (cur[j].y - m) * rinv + gb[j].y;
      cur[j].z = ga[j].z * (cur[j].z - m) * rinv + gb[j].z;
      cur[j].w = ga[j].w * (cur[j].w - m) * rinv + gb[j].w;
    }
    if (row < rows) {
      if (y16) r_store_bf16<LPR>(y16 + row * width, width, lane, cur);   // bf16 mode: the GEMM operand copy only
      else {   // packed rows with rowmap_out: row r goes to y[rowmap_out[r]] (alignment rows: nowhere)
        const long long yr = MAP ? (long long)rowmap_out[row] : row;
        if (!MAP || yr >= 0) r_store<LPR>(y + yr * width, width, lane, cur);
      }
      if (lane % LPR == 0) { mean_o[row] = m; std_o[row] = sdq; }
    }
#pragma unroll
    for (int j = 0; j < NJ; ++j) cur[j] = nxt[j];
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm bwd
// dx = [dres +] r (dxh - mean(dxh)) - r^2 (sum_k dxh_k c_k) / ((d-1) std) * c,   dxh = dy * a, c = x - mean,
// r = 1/(std+eps).   grad_a += sum_rows dy * xhat,  grad_b += sum_rows dy  (block partials -> DetParts slots).
// MAP: packed rows reading a row-mapped gradient (rowmap_in); a template flag as in ln_fwd_kernel
// PAD: n real columns at the pitch width as in ln_fwd_kernel: c = x - mean and the outputs are +0 in the pads, and the
// dropout counter of dx_masked is row * n + column
template <int LPR, int NJ, bool FILLED, bool MAP, bool PAD = false>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32, NJ <= 4 ? 2 : 1) ln_bwd_kernel(
    const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ a,
    const float* __restrict__ mean_i, const float* __restrict__ std_i, float eps, const float* __restrict__ dres,
    long long rows, int width, int steps, float* __restrict__ dx, float* __restrict__ grad_a,
    float* __restrict__ grad_b, float* __restrict__ dx_masked, DropSite site, float* __restrict__ colsum_out,
    int torch_mode, const uint16_t* __restrict__ dy16_in, uint16_t* __restrict__ dy16_out,
    const int* __restrict__ rows_dev, const int* __restrict__ rowmap_in, int n) {
  if (FILLED) width = 4 * LPR * NJ;   // (see with_row_layout)
  if (!PAD) n = width;
  arb_pdl_wait();
  site.seed = drop_seed(site);
  constexpr int RW = 32 / LPR;
  if (rows_dev) rows = min(rows, (long long)__ldg(rows_dev));
  if ((long long)blockIdx.x * ROWS_PER_BLOCK * RW * steps >= rows) return;      // whole block beyond the live rows
  __shared__ float sh[ROWS_PER_BLOCK][4 * LPR * NJ + 4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, rg = lane / LPR;
  float4 ga[NJ], acc_a[NJ], acc_b[NJ], acc_c[NJ];
  r_load<LPR>(a, width, lane, ga);
  r_zero(acc_a); r_zero(acc_b); r_zero(acc_c);
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + wid) * (RW * steps);
#pragma unroll 1
  for (int s = 0; s < steps; ++s) {
    if (base + (long long)s * RW >= rows) break;
    const long long row = base + (long long)s * RW + rg;
    const bool ok = row < rows;
    float4 g[NJ], xr[NJ], res[NJ];
    float mean = 0.f, sd = 1.f;
    r_zero(g); r_zero(xr); r_zero(res);
    if (ok) {
      if (dy16_in) r_load_bf16<LPR>(dy16_in + row * width, width, lane, g);
      else if (MAP) {   // packed rows: dy of row r is dy[rowmap_in[r]]; alignment rows have a zero gradient
        const long long src = rowmap_in[row];
        if (src >= 0) r_load<LPR>(dy + src * width, width, lane, g);
      } else r_load<LPR>(dy + row * width, width, lane, g);
      r_load<LPR>(x + row * width, width, lane, xr);
      if (dres) r_load<LPR>(dres + row * width, width, lane, res);
      mean = mean_i[row]; sd = std_i[row];
    }
    const float r = 1.0f / (sd + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const bool in = ok && r_col<LPR>(lane, j) < width;
      float* gv = &g[j].x;
      float* xv = &xr[j].x;
      const float* av = &ga[j].x;
      float* aa = &acc_a[j].x;
      float* ab = &acc_b[j].x;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float cc = in && (!PAD || r_col<LPR>(lane, j) + t < n) ? xv[t] - mean : 0.f;
        const float dyv = gv[t];
        aa[t] += dyv * cc * r;     // dy * xhat
        ab[t] += dyv;
        const float dxh = dyv * av[t];
        gv[t] = dxh;
        xv[t] = cc;
        s1 += dxh;
        s2 += dxh * cc;
      }
    }
    s1 = r_sum<LPR>(s1);
    s2 = r_sum<LPR>(s2);
    const float m1 = s1 / float(n);
    const float coef = torch_mode ? r * r * r * s2 / float(n)
                                  : ((sd > 0.f) ? r * r * s2 / (float(n - 1) * sd) : 0.f);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      float* gv = &g[j].x;
      const float* xv = &xr[j].x;
      const float* rv = &res[j].x;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        float o = r * (gv[t] - m1) - coef * xv[t];
        if (dres) o += rv[t];
        if (PAD && r_col<LPR>(lane, j) + t >= n) o = 0.f;   // (r (0 - m1) is not 0)
        gv[t] = o;
      }
    }
    if (ok) {
      r_store<LPR>(dx + row * width, width, lane, g);
      if (dx_masked) {   // the same gradient through the dropout of the sublayer below (mask regenerated)
        r_drop<LPR>(g, row, n, lane, site);
        r_store<LPR>(dx_masked + row * width, width, lane, g);
      }
      // bf16 mode: the copy the weight / input-gradient GEMMs of the sublayer below read (after its dropout mask)
      if (dy16_out) r_store_bf16<LPR>(dy16_out + row * width, width, lane, g);
      if (colsum_out) {  // bias gradient of the linear below = column sums of what that linear receives
#pragma unroll
        for (int j = 0; j < NJ; ++j) { acc_c[j].x += g[j].x; acc_c[j].y += g[j].y; acc_c[j].z += g[j].z; acc_c[j].w += g[j].w; }
      }
    }
  }
  if (grad_a) r_reduce_columns<LPR>(acc_a, sh, width, lane, wid, grad_a);
  if (grad_b) r_reduce_columns<LPR>(acc_b, sh, width, lane, wid, grad_b);
  if (colsum_out) r_reduce_columns<LPR>(acc_c, sh, width, lane, wid, colsum_out);
}

// ------------------------------------------------------------------------------------------------ softmax fwd
// In place on the attention logits [B, h, S, pitch]: key-masked row softmax (padded keys -> probability 0).
// A slate whose keys are all padded yields NaN rows, as the reference does (quirk Q2).
// DROP: inverted dropout applied AFTER the normalisation (transformer.py:153-155); element index
// ((b*h+head)*S + q)*S + key -- the same counter the fused attention kernels use, so a fused forward and this
// unfused path regenerate identical masks.
template <bool DROP>
__global__ void __launch_bounds__(256) softmax_fwd_kernel(float* __restrict__ sc, const uint8_t* __restrict__ mask,
                                                          int B, int h, int S, int pitch, DropSite site) {
  if (DROP) site.seed = drop_seed(site);
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const long long total = (long long)B * h * S;
  if (row >= total) return;
  const int b = int(row / ((long long)h * S));
  float* p = sc + row * pitch;
  const uint8_t* mk = mask + (long long)b * S;
  constexpr int MAXE = 48;   // S <= 1536 in registers
  float v[MAXE];
  float mx = -CUDART_INF_F;
#pragma unroll
  for (int k = 0; k < MAXE; ++k) {
    const int j = lane + 32 * k;
    v[k] = -CUDART_INF_F;
    if (j < S) {
      v[k] = mk[j] ? -CUDART_INF_F : p[j];
      mx = fmaxf(mx, v[k]);
    }
  }
  mx = warp_max(mx);
  float z = 0.f;
#pragma unroll
  for (int k = 0; k < MAXE; ++k) {
    const int j = lane + 32 * k;
    if (j < S) { v[k] = expf(v[k] - mx); z += v[k]; }
  }
  z = warp_sum(z);
#pragma unroll
  for (int k = 0; k < MAXE; ++k) {
    const int j = lane + 32 * k;
    if (j < S) {
      float e = v[k] / z;
      if (DROP) {
        const unsigned long long idx = (unsigned long long)row * (unsigned long long)S + j;
        e = drop_keep(idx, site.seed, site.thresh) ? e * site.scale : 0.0f;
      }
      p[j] = e;
    }
  }
}

// In place on dP: dS = P * (dP - sum_j P_j dP_j).
// DROP: `dp` holds the gradient w.r.t. the DROPPED probabilities P~ = m P / (1-p); the mask m is regenerated,
// dP = m dP~ / (1-p), and `prob` (the undropped P, recomputed by the caller) is overwritten with P~ for the
// dV = P~^T dO product that follows.
template <bool DROP>
__global__ void __launch_bounds__(256) softmax_bwd_kernel(float* __restrict__ dp, float* __restrict__ prob,
                                                          long long rows, int S, int pitch, DropSite site) {
  if (DROP) site.seed = drop_seed(site);
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  float* g = dp + row * pitch;
  float* p = prob + row * pitch;
  constexpr int MAXE = 48;
  float pv[MAXE], gv[MAXE];
  float t = 0.f;
#pragma unroll
  for (int k = 0; k < MAXE; ++k) {
    const int j = lane + 32 * k;
    pv[k] = gv[k] = 0.f;
    if (j < S) {
      pv[k] = p[j]; gv[k] = g[j];
      if (DROP) {
        const unsigned long long idx = (unsigned long long)row * (unsigned long long)S + j;
        const bool keep = drop_keep(idx, site.seed, site.thresh);
        gv[k] = keep ? gv[k] * site.scale : 0.0f;
        p[j] = keep ? pv[k] * site.scale : 0.0f;
      }
      t += pv[k] * gv[k];
    }
  }
  t = warp_sum(t);
#pragma unroll
  for (int k = 0; k < MAXE; ++k) {
    const int j = lane + 32 * k;
    if (j < S) g[j] = pv[k] * (gv[k] - t);
  }
}

// ------------------------------------------------------------------------------------------------ fp32 -> bf16
__global__ void __launch_bounds__(256) to_bf16_kernel(const float4* __restrict__ src, uint2* __restrict__ dst, long long n) {
  arb_pdl_wait();
  const long long n4 = n / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = src[i];
    dst[i] = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {          // the (up to three) trailing elements
    const float* s1 = reinterpret_cast<const float*>(src);
    uint16_t* d1 = reinterpret_cast<uint16_t*>(dst);
    for (long long i = 4 * n4; i < n; ++i) d1[i] = uint16_t(pack_bf16x2(s1[i], 0.f) & 0xffffu);
  }
}

__global__ void __launch_bounds__(256) tf32_weight_copy_kernel(const float* __restrict__ P, long long n, WeightMats m,
                                                              int rnd, float* __restrict__ pr, float* __restrict__ pt) {
  arb_pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = P[i];
    if (rnd) {
      uint32_t r;
      asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
      v = __uint_as_float(r);
    }
    pr[i] = v;
    long long o = -1;     // the matrix holding element i: offset, rows (out), columns (in)
    int rows = 0, cols = 0;
    for (int j = 0; j < m.n_fc; ++j)
      if (i >= m.fc_w[j] && i < m.fc_w[j] + (long long)m.fc_out[j] * m.fc_in[j]) { o = m.fc_w[j]; rows = m.fc_out[j]; cols = m.fc_in[j]; }
    if (o < 0 && m.n_layers > 0 && i >= m.enc0 && i < m.enc0 + m.n_layers * m.enc_stride) {
      const long long base = m.enc0 + (i - m.enc0) / m.enc_stride * m.enc_stride, j = i - base;
      const long long d = m.d, dw = m.dw, fw = m.fw;
      if (j < 3 * d * d) { o = base; rows = int(3 * d); cols = int(d); }
      else if (j >= m.o_wo && j < m.o_wo + d * d) { o = base + m.o_wo; rows = int(d); cols = int(d); }
      else if (j >= m.o_w1 && j < m.o_w1 + fw * dw) { o = base + m.o_w1; rows = int(fw); cols = int(dw); }
      else if (j >= m.o_w2 && j < m.o_w2 + dw * fw) { o = base + m.o_w2; rows = int(dw); cols = int(fw); }
    }
    if (o >= 0) {
      const long long e = i - o, r = e / cols, c = e % cols;
      pt[o + c * rows + r] = v;
    }
  }
}

// Padded heads: the padded copies of W_qkv, its transpose, b_qkv, W_o and its transpose (HeadPad), every element
// written, the pads as +0.  Padded row (column) g * hs + t holds the real row (column) g * w + t when t < w; rows
// (columns) of the residual stream from d to dw are pads too.
__global__ void __launch_bounds__(256) head_pad_copy_kernel(const float* __restrict__ pr, const float* __restrict__ P,
                                                            HeadPad m, float* __restrict__ out) {
  arb_pdl_wait();
  const long long d = m.d, dw = m.dw, dp = m.dp(), size = m.size(), n = size * m.n_layers;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long l = i / size, j = i - l * size, base = m.enc0 + l * m.enc_stride;
    long long src;      // offset of the real element in the flat parameters, or -1 for a pad
    const float* from = pr;
    auto real = [&](long long padded) { const long long g = padded / m.hs, t = padded - g * m.hs; return t < m.w ? g * m.w + t : -1; };
    if (j < m.wqkvt()) {                     // wqkv [3 dp, dw]
      const long long r = real(j / dw), c = j % dw;
      src = r < 0 || c >= d ? -1 : base + r * d + c;
    } else if (j < m.bqkv()) {               // wqkvt [dw, 3 dp]
      const long long e = j - m.wqkvt(), r = real(e % (3 * dp)), c = e / (3 * dp);
      src = r < 0 || c >= d ? -1 : base + r * d + c;
    } else if (j < m.wo()) {                 // bqkv [3 dp]: the fp32 bias, as the unpadded QKV linear reads it
      const long long r = real(j - m.bqkv());
      src = r < 0 ? -1 : base + m.o_bqkv + r;
      from = P;
    } else if (j < m.wot()) {                // wo [dw, dp]
      const long long e = j - m.wo(), c = real(e % dp), r = e / dp;
      src = c < 0 || r >= d ? -1 : base + m.o_wo + r * d + c;
    } else {                                 // wot [dp, dw]
      const long long e = j - m.wot(), c = real(e / dw), r = e % dw;
      src = c < 0 || r >= d ? -1 : base + m.o_wo + r * d + c;
    }
    out[i] = src < 0 ? 0.0f : from[src];
  }
}

// Padded heads: G += the real rows / columns of one layer's padded weight and bias gradients (HeadPad::g*), one
// thread per real element.
__global__ void __launch_bounds__(256) head_pad_grads_kernel(const float* __restrict__ gp, HeadPad m, long long base,
                                                             float* __restrict__ G) {
  arb_pdl_wait();
  const long long d = m.d, dp = m.dp(), n_w = 3 * d * d, n_b = 3 * d, n = n_w + n_b + d * d;
  auto padded = [&](long long real) { const long long g = real / m.w; return g * m.hs + (real - g * m.w); };
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (i < n_w) {                           // W_qkv [3d, d] (padded: [3 dp, dw])
      G[base + i] += gp[m.gwqkv() + padded(i / d) * m.dw + i % d];
    } else if (i < n_w + n_b) {              // b_qkv [3d]
      const long long e = i - n_w;
      G[base + m.o_bqkv + e] += gp[m.gbqkv() + padded(e)];
    } else {                                 // W_o [d, d]
      const long long e = i - n_w - n_b;
      G[base + m.o_wo + e] += gp[m.gwo() + e / d * dp + padded(e % d)];
    }
  }
}

// ------------------------------------------------------------------------------------------------ slate extents
__global__ void __launch_bounds__(256) slate_extent_kernel(const uint8_t* __restrict__ mask,
                                                           const float* __restrict__ dscores, int n_out, int B, int S,
                                                           int* __restrict__ extent) {
  arb_pdl_wait();
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  int last = -1;
  for (int r = lane; r < S; r += 32) {
    bool live = mask[(long long)b * S + r] == 0;
    if (!live && dscores) {
      for (int j = 0; j < n_out; ++j) live |= dscores[((long long)b * S + r) * n_out + j] != 0.0f;
    }
    if (live) last = r;
  }
  last = warp_max_int(last);
  if (lane == 0) extent[b] = last + 1;
}

// ------------------------------------------------------------------------------------------------ column sums
// out[c] += sum_rows in[row, c]   (bias gradients).  A warp reads whole rows with 128-bit loads (4 rows in
// flight per lane), 8 warps per block stride over the block's rows, then one shared-memory reduction and one
// store per column per block into the block's DetParts slot.
template <int NV>
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ in, long long rows, int width,
                                                     long long ld, int rows_per_block, float* __restrict__ out) {
  __shared__ float sh[ROWS_PER_BLOCK][128 * NV + 4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  float4 acc[NV];
  r_zero(acc);
  long long r = r0 + wid;
  for (; r + 24 < r1; r += 32) {
    float4 a0[NV], a1[NV], a2[NV], a3[NV];
    r_load<32>(in + r * ld, width, lane, a0);
    r_load<32>(in + (r + 8) * ld, width, lane, a1);
    r_load<32>(in + (r + 16) * ld, width, lane, a2);
    r_load<32>(in + (r + 24) * ld, width, lane, a3);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      acc[k].x += (a0[k].x + a1[k].x) + (a2[k].x + a3[k].x);
      acc[k].y += (a0[k].y + a1[k].y) + (a2[k].y + a3[k].y);
      acc[k].z += (a0[k].z + a1[k].z) + (a2[k].z + a3[k].z);
      acc[k].w += (a0[k].w + a1[k].w) + (a2[k].w + a3[k].w);
    }
  }
  for (; r < r1; r += 8) {
    float4 a0[NV];
    r_load<32>(in + r * ld, width, lane, a0);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      acc[k].x += a0[k].x; acc[k].y += a0[k].y; acc[k].z += a0[k].z; acc[k].w += a0[k].w;
    }
  }
  r_reduce_columns<32>(acc, sh, width, lane, wid, out);
}

// ------------------------------------------------------------------------------------------------ head fwd
// score = act( w . LN(x) + bias )  (final encoder LayerNorm fused; has_norm = 0 for FC-only models)
// The activations (ARB_ACT_*) in torch's fp32 formulas at its default arguments (aten/src/ATen/native/cuda: the ELU
// family with expm1, Softplus with log1p(exp(z)) up to its threshold, LogSigmoid as min(z, 0) - log1p(exp(-|z|)),
// Hardsigmoid as clamp(z + 3, 0, 6) * (1 / 6)).
constexpr float SELU_SCALE = 1.0507009873554805f;
constexpr float SELU_NEG = 1.6732632423543772f * SELU_SCALE;   // alpha * lambda, multiplied in fp32 as torch does
__device__ __forceinline__ float act_fwd(float z, int act) {
  switch (act) {
    case ARB_ACT_TANH: return tanhf(z);
    case ARB_ACT_SIGMOID: return 1.0f / (1.0f + expf(-z));
    case ARB_ACT_RELU: return fmaxf(z, 0.f);
    case ARB_ACT_LEAKY_RELU: return z > 0.f ? z : z * 0.01f;
    case ARB_ACT_ELU: case ARB_ACT_CELU: return z > 0.f ? z : expm1f(z);
    case ARB_ACT_SELU: return z > 0.f ? z * SELU_SCALE : expm1f(z) * SELU_NEG;
    case ARB_ACT_SOFTPLUS: return z > 20.f ? z : log1pf(expf(z));
    case ARB_ACT_SOFTSIGN: return z / (fabsf(z) + 1.0f);
    case ARB_ACT_HARDTANH: return fminf(fmaxf(z, -1.f), 1.f);
    case ARB_ACT_RELU6: return fminf(fmaxf(z, 0.f), 6.f);
    case ARB_ACT_HARDSIGMOID: return fminf(fmaxf(z + 3.f, 0.f), 6.f) * (1.0f / 6.0f);
    case ARB_ACT_LOGSIGMOID: return fminf(z, 0.f) - log1pf(expf(-fabsf(z)));
    case ARB_ACT_HARDSHRINK: return z >= -0.5f && z <= 0.5f ? 0.f : z;
    case ARB_ACT_SOFTSHRINK: return z > 0.5f ? z - 0.5f : (z < -0.5f ? z + 0.5f : 0.f);
    default: return z;
  }
}
// act'(z) from the output y = act(z) (include/allrank_b200.h, ARB_ACT_*)
__device__ __forceinline__ float act_bwd(float y, int act) {
  switch (act) {
    case ARB_ACT_TANH: return 1.0f - y * y;
    case ARB_ACT_SIGMOID: return y * (1.0f - y);
    case ARB_ACT_RELU: return y > 0.f ? 1.0f : 0.0f;   // y > 0 <=> z > 0
    case ARB_ACT_LEAKY_RELU: return y > 0.f ? 1.0f : 0.01f;
    case ARB_ACT_ELU: case ARB_ACT_CELU: return y > 0.f ? 1.0f : y + 1.0f;
    case ARB_ACT_SELU: return y > 0.f ? SELU_SCALE : y + SELU_NEG;
    case ARB_ACT_SOFTPLUS: return y > 20.f ? 1.0f : -expm1f(-y);   // sigmoid(z) = 1 - exp(-softplus(z))
    case ARB_ACT_SOFTSIGN: { const float t = 1.0f - fabsf(y); return t * t; }
    case ARB_ACT_HARDTANH: return y > -1.f && y < 1.f ? 1.0f : 0.0f;
    case ARB_ACT_RELU6: return y > 0.f && y < 6.f ? 1.0f : 0.0f;
    case ARB_ACT_HARDSIGMOID: return y > 0.f && y < 1.f ? 1.0f / 6.0f : 0.0f;
    case ARB_ACT_LOGSIGMOID: return -expm1f(y);                    // sigmoid(-z) = 1 - exp(logsigmoid(z))
    case ARB_ACT_HARDSHRINK: case ARB_ACT_SOFTSHRINK: return y != 0.f ? 1.0f : 0.0f;
    default: return 1.0f;
  }
}

template <int LPR, int NJ, bool FILLED>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) head_fwd_kernel(
    const float* __restrict__ x, const float* __restrict__ a, const float* __restrict__ b, float eps,
    const float* __restrict__ w, const float* __restrict__ wb, int has_norm, int act, long long rows, int width,
    float* __restrict__ score, float* __restrict__ mean_o, float* __restrict__ std_o,
    const int* __restrict__ rows_dev, const int* __restrict__ rowmap, int steps) {
  if (FILLED) width = 4 * LPR * NJ;   // (see with_row_layout)
  arb_pdl_wait();
  constexpr int RW = 32 / LPR;
  const int lane = threadIdx.x & 31, rg = lane / LPR;
  // `steps` steps of 32 / LPR rows per warp, the next step's loads (rows and their row-map entries) issued before the
  // arithmetic of the current one (see ln_fwd_kernel)
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5)) * (RW * steps);
  if (base >= rows) return;
  if (rows_dev) { rows = min(rows, (long long)__ldg(rows_dev)); if (base >= rows) return; }
  float4 ga[NJ], gb[NJ], gw[NJ], cur[NJ], nxt[NJ];
  r_load<LPR>(w, width, lane, gw);
  if (has_norm) { r_load<LPR>(a, width, lane, ga); r_load<LPR>(b, width, lane, gb); } else { r_zero(ga); r_zero(gb); }
  const float bias = wb[0];
  long long at = -1, at_n = -1;
  if (base + rg < rows) {
    r_load<LPR>(x + (base + rg) * width, width, lane, cur);
    at = rowmap ? (long long)rowmap[base + rg] : base + rg;
  } else {
    r_zero(cur);
  }
#pragma unroll 1
  for (int s = 0; s < steps; ++s) {
    if (base + (long long)s * RW >= rows) break;
    const long long row = base + (long long)s * RW + rg;
    if (s + 1 < steps) {
      at_n = -1;
      if (row + RW < rows) {
        r_load<LPR>(x + (row + RW) * width, width, lane, nxt);
        at_n = rowmap ? (long long)rowmap[row + RW] : row + RW;
      } else {
        r_zero(nxt);
      }
    }
    float m = 0.f, sdv = 0.f;
    if (has_norm) {
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) sum += cur[j].x + cur[j].y + cur[j].z + cur[j].w;
      m = r_sum<LPR>(sum) / float(width);
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        if (r_col<LPR>(lane, j) < width) {
          const float d0 = cur[j].x - m, d1 = cur[j].y - m, d2 = cur[j].z - m, d3 = cur[j].w - m;
          ss += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
        }
      }
      sdv = sqrtf(r_sum<LPR>(ss) / float(width - 1));
      const float rinv = 1.0f / (sdv + eps);      // (one reciprocal per row: see ln_fwd_kernel)
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        cur[j].x = ga[j].x * (cur[j].x - m) * rinv + gb[j].x;
        cur[j].y = ga[j].y * (cur[j].y - m) * rinv + gb[j].y;
        cur[j].z = ga[j].z * (cur[j].z - m) * rinv + gb[j].z;
        cur[j].w = ga[j].w * (cur[j].w - m) * rinv + gb[j].w;
      }
    }
    // (masked columns hold 0: their gain and bias are loaded as 0)
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) dot += cur[j].x * gw[j].x + cur[j].y * gw[j].y + cur[j].z * gw[j].z + cur[j].w * gw[j].w;
    dot = r_sum<LPR>(dot);
    if (row < rows && lane % LPR == 0) {
      // packed rows: the score goes to the item's place in the [B, S] tensor (alignment rows have none)
      if (at >= 0) score[at] = act_fwd(dot + bias, act);
      if (has_norm && mean_o) { mean_o[row] = m; std_o[row] = sdv; }
    }
    at = at_n;
#pragma unroll
    for (int j = 0; j < NJ; ++j) cur[j] = nxt[j];
  }
}

// head backward: dz = dscore * act'(z);  d xf = dz * w;  grad_w += dz * xf;  grad_wb += dz;  then LayerNorm bwd.
template <int LPR, int NJ, bool FILLED>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32, NJ <= 4 ? 2 : 1) head_bwd_kernel(
    const float* __restrict__ dscore, const float* __restrict__ score, const float* __restrict__ x,
    const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ mean_i,
    const float* __restrict__ std_i, float eps, const float* __restrict__ w, int has_norm, int act, long long rows,
    int width, int steps, float* __restrict__ dx, float* __restrict__ grad_a, float* __restrict__ grad_b,
    float* __restrict__ grad_w, float* __restrict__ grad_wb, float* __restrict__ dx_masked, DropSite site,
    float* __restrict__ colsum_out, uint16_t* __restrict__ dy16_out, const int* __restrict__ rows_dev,
    const int* __restrict__ rowmap) {
  if (FILLED) width = 4 * LPR * NJ;   // (see with_row_layout)
  arb_pdl_wait();
  site.seed = drop_seed(site);
  constexpr int RW = 32 / LPR;
  if (rows_dev) rows = min(rows, (long long)__ldg(rows_dev));
  if ((long long)blockIdx.x * ROWS_PER_BLOCK * RW * steps >= rows) return;
  __shared__ float sh[ROWS_PER_BLOCK][4 * LPR * NJ + 4];
  __shared__ float shb[ROWS_PER_BLOCK];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, rg = lane / LPR;
  float4 ga[NJ], gb[NJ], gw[NJ], acc_a[NJ], acc_b[NJ], acc_w[NJ], acc_c[NJ];
  r_load<LPR>(w, width, lane, gw);
  if (has_norm) { r_load<LPR>(a, width, lane, ga); r_load<LPR>(b, width, lane, gb); } else { r_zero(ga); r_zero(gb); }
  r_zero(acc_a); r_zero(acc_b); r_zero(acc_w); r_zero(acc_c);
  float acc_wb = 0.f;
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + wid) * (RW * steps);
#pragma unroll 1
  for (int s = 0; s < steps; ++s) {
    if (base + (long long)s * RW >= rows) break;
    const long long row = base + (long long)s * RW + rg;
    const bool ok = row < rows;
    float4 xr[NJ], g[NJ];
    r_zero(xr);
    long long at = -1;
    float mean = 0.f, sd = 1.f;
    if (ok) {
      r_load<LPR>(x + row * width, width, lane, xr);
      // packed rows: score and its gradient sit at the item's place in the [B, S] tensors; alignment rows have neither
      at = rowmap ? (long long)rowmap[row] : row;
      if (has_norm) { mean = mean_i[row]; sd = std_i[row]; }
    }
    const float out = at >= 0 ? score[at] : 0.f;
    const float dz = at >= 0 ? dscore[at] * act_bwd(out, act) : 0.f;
    if (lane % LPR == 0) acc_wb += dz;
    if (!has_norm) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const float* xv = &xr[j].x;
        const float* wv = &gw[j].x;
        float* gv = &g[j].x;
        float* aw = &acc_w[j].x;
#pragma unroll
        for (int t = 0; t < 4; ++t) { gv[t] = dz * wv[t]; aw[t] += dz * xv[t]; }
      }
    } else {
      const float r = 1.0f / (sd + eps);
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const bool in = ok && r_col<LPR>(lane, j) < width;
        float* xv = &xr[j].x;
        const float* wv = &gw[j].x;
        const float* av = &ga[j].x;
        const float* bv = &gb[j].x;
        float* gv = &g[j].x;
        float* aa = &acc_a[j].x;
        float* ab = &acc_b[j].x;
        float* aw = &acc_w[j].x;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float cc = in ? xv[t] - mean : 0.f;
          const float xh = cc * r;
          const float xf = av[t] * xh + bv[t];     // the final norm's output, recomputed (xh = (x - mean) / (std + eps))
          const float dyv = dz * wv[t];            // d loss / d xf
          aw[t] += dz * xf;
          aa[t] += dyv * xh;
          ab[t] += dyv;
          const float dxh = dyv * av[t];
          gv[t] = dxh;
          xv[t] = cc;
          s1 += dxh;
          s2 += dxh * cc;
        }
      }
      s1 = r_sum<LPR>(s1);
      s2 = r_sum<LPR>(s2);
      const float m1 = s1 / float(width);
      const float coef = (sd > 0.f) ? r * r * s2 / (float(width - 1) * sd) : 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        float* gv = &g[j].x;
        const float* xv = &xr[j].x;
#pragma unroll
        for (int t = 0; t < 4; ++t) gv[t] = r * (gv[t] - m1) - coef * xv[t];
      }
    }
    if (ok) {
      r_store<LPR>(dx + row * width, width, lane, g);
      if (dx_masked) { r_drop<LPR>(g, row, width, lane, site); r_store<LPR>(dx_masked + row * width, width, lane, g); }
      if (dy16_out) r_store_bf16<LPR>(dy16_out + row * width, width, lane, g);
      if (colsum_out) {
#pragma unroll
        for (int j = 0; j < NJ; ++j) { acc_c[j].x += g[j].x; acc_c[j].y += g[j].y; acc_c[j].z += g[j].z; acc_c[j].w += g[j].w; }
      }
    }
  }
  if (has_norm && grad_a) r_reduce_columns<LPR>(acc_a, sh, width, lane, wid, grad_a);
  if (has_norm && grad_b) r_reduce_columns<LPR>(acc_b, sh, width, lane, wid, grad_b);
  if (grad_w) r_reduce_columns<LPR>(acc_w, sh, width, lane, wid, grad_w);
  if (colsum_out) r_reduce_columns<LPR>(acc_c, sh, width, lane, wid, colsum_out);
  acc_wb = warp_sum(acc_wb);
  if (lane == 0) shb[wid] = acc_wb;
  __syncthreads();
  if (threadIdx.x == 0 && grad_wb) {
    float t = 0.f;
    for (int ww = 0; ww < ROWS_PER_BLOCK; ++ww) t += shb[ww];
    grad_wb[blockIdx.x] = t;                        // this block's slot (DetParts)
  }
}

// ------------------------------------------------------------------------------------------------ multi-output head
// post_model.d_output = n > 1 (model.py:104-117; the ordinal loss reads n probabilities per item):
//   score[row, j] = act( w_j . xf[row] + b_j ),   xf = the final LayerNorm's output (or the FC output), kept in HBM.
// n is small (the number of relevance levels), so the kernels loop over it; the weight rows stay in L1.
template <int NV>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) head_multi_fwd_kernel(const float* __restrict__ xf,
                                                                            const float* __restrict__ w,
                                                                            const float* __restrict__ wb, int act,
                                                                            long long rows, int width, int n,
                                                                            float* __restrict__ score) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5);
  if (row >= rows) return;
  float4 r[NV], gw[NV];
  r_load<32>(xf + row * width, width, lane, r);
  for (int j = 0; j < n; ++j) {
    r_load<32>(w + (long long)j * width, width, lane, gw);
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) dot += r[k].x * gw[k].x + r[k].y * gw[k].y + r[k].z * gw[k].z + r[k].w * gw[k].w;
    dot = warp_sum(dot);
    if (lane == 0) score[row * n + j] = act_fwd(dot + wb[j], act);
  }
}

// d xf[row] = sum_j dz_j w_j;  grad_w[j] += sum_rows dz_j xf[row];  grad_wb[j] += sum_rows dz_j;  dz = dscore * act'.
// dx_masked / colsum_out: the FC-only model has no final norm, so this kernel also emits the gradient seen through
// the FC dropout and the FC bias gradient (what head_bwd_kernel does for n = 1).
template <int NV>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) head_multi_bwd_kernel(
    const float* __restrict__ dscore, const float* __restrict__ score, const float* __restrict__ xf,
    const float* __restrict__ w, int act, long long rows, int width, int n, int rows_per_warp,
    float* __restrict__ dxf, float* __restrict__ grad_w, float* __restrict__ grad_wb, float* __restrict__ dx_masked,
    DropSite site, float* __restrict__ colsum_out) {
  __shared__ float sh[ROWS_PER_BLOCK][128 * NV + 4];
  __shared__ float shb[ROWS_PER_BLOCK];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long first = ((long long)blockIdx.x * ROWS_PER_BLOCK + wid) * rows_per_warp;
  float4 acc[NV], gw[NV];
  r_zero(acc);
  if (dx_masked) site.seed = drop_seed(site);   // (here rather than at entry: NV = 2 then spills)
  for (int it = 0; it < rows_per_warp; ++it) {
    const long long row = first + it;
    if (row >= rows) break;
    float4 g[NV];
    r_zero(g);
    for (int j = 0; j < n; ++j) {
      const float out = score[row * n + j];
      const float dz = dscore[row * n + j] * act_bwd(out, act);
      r_load<32>(w + (long long)j * width, width, lane, gw);
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        g[k].x += dz * gw[k].x; g[k].y += dz * gw[k].y; g[k].z += dz * gw[k].z; g[k].w += dz * gw[k].w;
      }
    }
    r_store<32>(dxf + row * width, width, lane, g);
    if (dx_masked) { r_drop<32>(g, row, width, lane, site); r_store<32>(dx_masked + row * width, width, lane, g); }
    if (colsum_out) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        acc[k].x += g[k].x; acc[k].y += g[k].y; acc[k].z += g[k].z; acc[k].w += g[k].w;
      }
    }
  }
  // block-level column reductions: pass -1 = colsum_out, pass j = grad_w row j
  for (int j = colsum_out ? -1 : 0; j < (grad_w ? n : 0); ++j) {
    float acc_b = 0.f;
    if (j >= 0) {
      r_zero(acc);
      for (int it = 0; it < rows_per_warp; ++it) {
        const long long row = first + it;
        if (row >= rows) break;
        const float out = score[row * n + j];
        const float dz = dscore[row * n + j] * act_bwd(out, act);
        r_load<32>(xf + row * width, width, lane, gw);
        acc_b += dz;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          acc[k].x += dz * gw[k].x; acc[k].y += dz * gw[k].y; acc[k].z += dz * gw[k].z; acc[k].w += dz * gw[k].w;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < NV; ++k) *reinterpret_cast<float4*>(&sh[wid][r_col<32>(lane, k)]) = acc[k];
    if (lane == 0) shb[wid] = acc_b;
    __syncthreads();
    // this block's slots (DetParts): colsum_out [block][width], grad_w [block][n][width], grad_wb [block][n]
    float* dst = j < 0 ? colsum_out + (long long)blockIdx.x * width : grad_w + ((long long)blockIdx.x * n + j) * width;
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
      float t = 0.f;
#pragma unroll
      for (int ww = 0; ww < ROWS_PER_BLOCK; ++ww) t += sh[ww][c];
      dst[c] = t;
    }
    if (j >= 0 && threadIdx.x == 0) {
      float t = 0.f;
      for (int ww = 0; ww < ROWS_PER_BLOCK; ++ww) t += shb[ww];
      grad_wb[(long long)blockIdx.x * n + j] = t;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ positional encoding
// x = sqrt(d) * x + pe[idx],  idx = padded ? last row : min(index, last row)     (allrank/models/positional.py:39-50,66-77)
__global__ void __launch_bounds__(256) pos_fwd_kernel(float* __restrict__ x, const long long* __restrict__ indices,
                                                      const uint8_t* __restrict__ mask, const float* __restrict__ pe,
                                                      int pe_rows, float scale, long long rows, int width) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int pad = pe_rows - 1;
  long long idx = mask[row] ? pad : indices[row];
  if (idx > pad) idx = pad;
  if (idx < 0) idx += pe_rows;                     // python-style negative index (only reachable for unmasked -1)
  if (idx < 0) idx = pad;                          // below -pe_rows: the padding row (the reference would raise)
  for (int c = lane * 4; c < width; c += 128) {
    float4 v = *reinterpret_cast<float4*>(x + row * width + c);
    const float4 p = *reinterpret_cast<const float4*>(pe + idx * width + c);
    v.x = scale * v.x + p.x; v.y = scale * v.y + p.y; v.z = scale * v.z + p.z; v.w = scale * v.w + p.w;
    *reinterpret_cast<float4*>(x + row * width + c) = v;
  }
}
// learned table: dpe[idx] += dx   (the padding row receives no gradient: nn.Embedding(padding_idx=-1), positional.py:64)
// Fixed order, no atomics: block k adds rows k * rows_per_block ... in ascending order into its own DetParts slot
// slot[k] [pad, width] (zeroed), each thread walking its columns row by row; the slots are then summed in order.
__global__ void __launch_bounds__(256) pos_bwd_kernel(const float* __restrict__ dx, const long long* __restrict__ indices,
                                                      const uint8_t* __restrict__ mask, float* __restrict__ slot,
                                                      int pe_rows, long long rows, int width, int rows_per_block) {
  const int pad = pe_rows - 1;
  float* const own = slot + (long long)blockIdx.x * pad * width;
  const long long r0 = (long long)blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
  for (long long row = r0; row < r1; ++row) {
    long long idx = mask[row] ? pad : indices[row];
    if (idx > pad) idx = pad;
    if (idx < 0) idx += pe_rows;
    if (idx < 0 || idx == pad) continue;
    for (int c = threadIdx.x; c < width; c += blockDim.x) own[idx * width + c] += dx[row * width + c];
  }
}

// ------------------------------------------------------------------------------------------------ FC-block activations
// FCModel applies dropout(activation(linear(x))) per layer (model.py:41-43).  ReLU / identity run inside the GEMM
// epilogue; the kernels below serve the other activations and the backward of every activation under dropout.
// Element index of the dropout counter = row * width + column (the same as the GEMM epilogue's).
// A layer of n columns that is not a multiple of 4 is stored at the pitch width = round_up(n, 4) (DESIGN.md 4.16): the
// counter then keeps the real layout, row * n + column, and the pad columns are written +0 (sigmoid(0) is not 0).
__global__ void __launch_bounds__(256) act_fwd_kernel(float* __restrict__ h, long long n4, int act, DropSite site,
                                                      const int* __restrict__ rows_dev, int width4, int n) {
  site.seed = drop_seed(site);
  if (rows_dev) n4 = min(n4, (long long)__ldg(rows_dev) * width4);
  const bool padded = n != 4 * width4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(h)[i];
    float* e = &v.x;
    if (padded) {
      const long long r = i / width4;
      const int c0 = int(i - r * width4) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float y = act_fwd(e[j], act);
        const bool real = c0 + j < n;
        e[j] = real && drop_keep((unsigned long long)r * n + c0 + j, site.seed, site.thresh) ? y * site.scale : 0.0f;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float y = act_fwd(e[j], act);
        e[j] = drop_keep((unsigned long long)i * 4 + j, site.seed, site.thresh) ? y * site.scale : 0.0f;
      }
    }
    reinterpret_cast<float4*>(h)[i] = v;
  }
}

// act'(z) of a kept element from its stored h = fl(y * scale).  The round trip y = h * (1 / scale) can land a saturated
// output (exactly 1 or 6) one ulp inside its bound, so the clamping activations compare h with fl(bound * scale),
// the very product the forward stored for a saturated y; lower bounds at 0 are decided by sign.
__device__ __forceinline__ float act_bwd_stored(float h, float inv_scale, float scale, int act) {
  switch (act) {
    case ARB_ACT_HARDTANH: return h > -scale && h < scale ? 1.0f : 0.0f;
    case ARB_ACT_RELU6: return h > 0.f && h < 6.0f * scale ? 1.0f : 0.0f;
    case ARB_ACT_HARDSIGMOID: return h > 0.f && h < scale ? 1.0f / 6.0f : 0.0f;
    default: return act_bwd(h * inv_scale, act);
  }
}

// dz = mul * dh * m/(1-p) * act'(y)  with y = act(z) recovered from the stored h = m y/(1-p); colsum_out += column sums
// of dz (the bias gradient of the linear that produced z).  dz may alias dh.  n < width: a padded layer as in
// act_fwd_kernel (dropout counter row * n + column; pad columns of dz +0).
__global__ void __launch_bounds__(256) act_bwd_kernel(const float* dh, const float* __restrict__ h, float* dz,
                                                      long long rows, int width, int act, DropSite site, float mul,
                                                      int tx_n, int rows_per_block, float* __restrict__ colsum_out,
                                                      const int* __restrict__ rows_dev, int n) {
  extern __shared__ float sh_cols[];     // [ty_n][width]: one row of column partials per row group
  site.seed = drop_seed(site);
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  if (rows_dev) rows = min(rows, (long long)__ldg(rows_dev));
  if (colsum_out) {
    for (int c = threadIdx.x; c < ty_n * width; c += blockDim.x) sh_cols[c] = 0.f;
    __syncthreads();
  }
  const int groups = width / 4;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  const float inv_scale = 1.0f / site.scale;
  for (int g = tx; g < groups; g += tx_n) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long r = r0 + ty; r < r1; r += ty_n) {
      const long long at = r * width + g * 4;
      const float4 hv = *reinterpret_cast<const float4*>(h + at);
      float4 gv = *reinterpret_cast<const float4*>(dh + at);
      const float* he = &hv.x;
      float* ge = &gv.x;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const bool keep = n == width ? drop_keep((unsigned long long)at + j, site.seed, site.thresh)
                                     : g * 4 + j < n && drop_keep((unsigned long long)r * n + g * 4 + j, site.seed,
                                                                  site.thresh);
        ge[j] = keep ? ge[j] * mul * site.scale * act_bwd_stored(he[j], inv_scale, site.scale, act) : 0.0f;
      }
      *reinterpret_cast<float4*>(dz + at) = gv;
      acc.x += gv.x; acc.y += gv.y; acc.z += gv.z; acc.w += gv.w;
    }
    if (colsum_out) *reinterpret_cast<float4*>(&sh_cols[ty * width + g * 4]) = acc;
  }
  if (colsum_out) {
    __syncthreads();
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
      float t = 0.f;
      for (int y = 0; y < ty_n; ++y) t += sh_cols[y * width + c];
      colsum_out[size_t(blockIdx.x) * width + c] = t;   // this block's slot (DetParts)
    }
  }
}

// ------------------------------------------------------------------------------------------------ host launchers
static int nv_for(int width) { return (width + 127) / 128; }

// NV of the one-row-per-warp kernels (column sums, multi-output head)
#define ARB_DISPATCH_NV(width, CALL)                                  \
  switch (nv_for(width)) {                                            \
    case 1: { constexpr int NV = 1; CALL; } break;                    \
    case 2: { constexpr int NV = 2; CALL; } break;                    \
    case 3: case 4: { constexpr int NV = 4; CALL; } break;            \
    case 5: case 6: case 7: case 8: { constexpr int NV = 8; CALL; } break; \
    default: arb_set_error("row kernels support widths up to 1024"); return ARB_E_UNSUPPORTED; \
  }

// Returns f(LPR, NJ, FILLED) with std::integral_constant arguments: the row layout of the LayerNorm and head kernels
// for `width`, and whether the width fills it.  A filled width is a compile-time constant of the kernel: its row
// statistics then divide by a constant, as kernels written for one width do (a run-time divisor costs registers and
// changes which products the compiler fuses into FMAs, and so the last bits of W = 128 / 256).
template <class F>
static int with_row_layout(int width, F&& f) {
  using std::integral_constant;
  auto layout = [&](auto LPR, auto NJ) {
    if (width == 4 * LPR * NJ) return f(LPR, NJ, std::true_type());
    return f(LPR, NJ, std::false_type());
  };
  if (width <= 128) return layout(integral_constant<int, 8>(), integral_constant<int, 4>());
  if (width <= 256) return layout(integral_constant<int, 16>(), integral_constant<int, 4>());
  if (width <= 512) return layout(integral_constant<int, 32>(), integral_constant<int, 4>());
  if (width <= 1024) return layout(integral_constant<int, 32>(), integral_constant<int, 8>());
  arb_set_error("row kernels support widths up to 1024");
  return ARB_E_UNSUPPORTED;
}
// steps per warp of the forward row kernels: 4 for large launches, 1 for small ones (more steps would leave SMs without
// a block -- B = 64 has 8 k live rows)
static inline int r_fwd_steps(long long rows) { return rows >= (1 << 17) ? 4 : 1; }
// rows per warp of the backward row kernels (a multiple of 4): the per-warp column reduction at the end costs 2 shuffles
// per accumulator element, so large launches amortise it over 32 rows; small ones keep every SM busy with 8
static inline int r_bwd_rows_per_warp(long long rows) { return rows >= (1 << 17) ? 32 : 8; }

// Accounting only (ProfScope): launches over packed rows process arb_row_frac() of the nominal rows.
static double live_rows(long long rows, const int* rows_dev) { return double(rows) * (rows_dev ? arb_row_frac() : 1.0); }

// ------------------------------------------------------------------------------------------------ packed rows
// Padding removal.  A slate of extent e (slate_extents: every item at or beyond e is padding) contributes its first
// e16 = round_up(e, 16) rows to the packed [rows, width] activation layout, slate after slate; the total is rounded up
// to a multiple of 128 (the GEMM tile height) with rows that belong to no item.  Every row-wise kernel and GEMM of the
// encoder then runs over plan[0] rows instead of B * S -- the count lives on the device, so nothing synchronises.
//   off[b]    first packed row of slate b (off[B] = plan[1])
//   plan[0]   packed rows, multiple of 128;  plan[1] = rows that belong to slates
//   rowmap[r] item index b * S + s of packed row r, or -1 (alignment row: zero features, no score)
__global__ void __launch_bounds__(1024) pack_scan_kernel(const int* __restrict__ ext, int B, int* __restrict__ off,
                                                         int* __restrict__ plan) {
  arb_pdl_wait();
  __shared__ int part[1024];
  const int t = threadIdx.x;
  const int per = (B + 1023) / 1024;
  const int b0 = min(B, t * per), b1 = min(B, b0 + per);
  int s = 0;
  for (int b = b0; b < b1; ++b) s += (ext[b] + 15) & ~15;
  part[t] = s;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {      // inclusive scan of the 1024 partial sums
    const int v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int run = part[t] - s;                    // exclusive prefix of this thread's chunk
  for (int b = b0; b < b1; ++b) { off[b] = run; run += (ext[b] + 15) & ~15; }
  if (t == 1023) {
    const int total = part[1023];
    off[B] = total;
    plan[0] = (total + 127) & ~127;
    plan[1] = total;
  }
}

// one block per slate (+ one for the tail alignment rows): row map and the packed copy of the features
__global__ void __launch_bounds__(256) pack_rows_kernel(const float* __restrict__ x, const int* __restrict__ ext,
                                                        const int* __restrict__ off, const int* __restrict__ plan,
                                                        int B, int S, int F, float* __restrict__ xc,
                                                        int* __restrict__ rowmap, int cap_rows) {
  arb_pdl_wait();
  const int b = blockIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int r0, n, src0;
  if (b < B) { r0 = off[b]; n = (ext[b] + 15) & ~15; src0 = b * S; }
  else { r0 = plan[1]; n = min(plan[0], cap_rows) - plan[1]; src0 = -1; }   // (the buffers hold cap_rows rows)
  // four rows of a warp in flight (a small batch has one block per slate and nothing else to hide the latency of a
  // row-at-a-time copy: 31 us at B = 64 for 4 MB)
  for (int s0 = wid; s0 < n; s0 += 32) {
    for (int c = lane * 4; c < F; c += 128) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int s = s0 + 8 * u;
        v[u] = (s < n && src0 >= 0 && s < S) ? *reinterpret_cast<const float4*>(x + (long long)(src0 + s) * F + c)
                                             : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int s = s0 + 8 * u;
        if (s < n) *reinterpret_cast<float4*>(xc + (long long)(r0 + s) * F + c) = v[u];
      }
    }
    if (lane < 4) {
      const int s = s0 + 8 * lane;
      if (s < n) rowmap[r0 + s] = (src0 >= 0 && s < S) ? src0 + s : -1;
    }
  }
}

// Rows the fused attention kernels may read beyond the packed rows (their 128-row boxes overrun the last slates) must
// be finite, and the alignment rows nobody writes must be zero before a product reads them.  Nothing else writes
// those rows during a call, so ONE launch at the start of a forward (backward) call zeroes them for every layer:
//   region.from == 0: `n` rows after the packed rows (plan[0]), capped at cap_rows;
//   region.from == 1: the alignment rows between the slates' rows (plan[1]) and the packed row count (plan[0]).
__global__ void __launch_bounds__(256) zero_rows_kernel(ZeroRegions z, const int* __restrict__ plan, long long cap_rows) {
  arb_pdl_wait();
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  for (int i = 0; i < z.count; ++i) {
    const ZeroRegion& g = z.r[i];
    const long long start = plan[g.from];
    const long long end = min(cap_rows, g.from == 0 ? start + g.n : (long long)plan[0]);
    const long long row = start + r;
    if (row >= end) continue;
    for (int c = lane * 4; c < g.width; c += 128)
      *reinterpret_cast<float4*>(g.p + row * g.pitch + c) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// The inverse of the feature packing: packed row r of src [rows, width] goes to dst[rowmap[r]] of the dense [B * S, width]
// tensor, which the caller has zero-filled (items beyond their slate's packed rows keep 0).  A warp per row, 128-bit
// accesses.
__global__ void __launch_bounds__(256) scatter_rows_kernel(const float* __restrict__ src, const int* __restrict__ plan,
                                                           const int* __restrict__ rowmap, long long cap_rows, int width,
                                                           float* __restrict__ dst) {
  arb_pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= min(cap_rows, (long long)plan[1])) return;      // (rows from plan[1] on are alignment rows)
  const long long to = rowmap[row];
  if (to < 0) return;
  for (int c = lane * 4; c < width; c += 128)
    *reinterpret_cast<float4*>(dst + to * width + c) = *reinterpret_cast<const float4*>(src + row * width + c);
}

int scatter_rows(const float* src, const int* plan, const int* rowmap, long long cap_rows, int width, float* dst,
                 cudaStream_t st) {
  if (width % 4) { arb_set_error("scatter_rows: the width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(cap_rows, plan) * 8.0 * width, st);
  return launch(scatter_rows_kernel, dim3(unsigned((cap_rows + 7) / 8)), dim3(256), 0, st, /*pdl=*/true, src, plan,
                rowmap, cap_rows, width, dst);
}

int pack_plan(const float* x, const int* ext, int B, int S, int F, int* off, int* plan, int* rowmap, float* xc,
              long long cap_rows, cudaStream_t st) {
  if (F % 4) { arb_set_error("packed rows: the feature count must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  {
    ProfScope ps(ARB_PROF_SCORER_SIMT, 8.0 * B, st, 0.0, "pack_scan");
    if (int rc = launch(pack_scan_kernel, dim3(1), dim3(1024), 0, st, /*pdl=*/true, ext, B, off, plan)) return rc;
  }
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(B) * S * arb_row_frac() * (8.0 * F + 4.0), st, 0.0, "pack_rows");
  return launch(pack_rows_kernel, dim3(unsigned(B + 1)), dim3(256), 0, st, /*pdl=*/true, x, ext,
                static_cast<const int*>(off), static_cast<const int*>(plan), B, S, F, xc, rowmap, int(cap_rows));
}

int zero_rows(const ZeroRegions& z, const int* plan, long long cap_rows, cudaStream_t st) {
  int n = 128;
  double bytes = 0.0;
  for (int i = 0; i < z.count; ++i) {
    if (z.r[i].width % 4 || z.r[i].pitch % 4) { arb_set_error("zero_rows: widths must be multiples of 4 floats"); return ARB_E_UNSUPPORTED; }
    if (z.r[i].from == 0) n = std::max(n, z.r[i].n);
    bytes += 4.0 * (z.r[i].from == 0 ? z.r[i].n : 64) * z.r[i].width;
  }
  ProfScope ps(ARB_PROF_SCORER_SIMT, bytes, st, 0.0, "zero_rows");
  return launch(zero_rows_kernel, dim3(unsigned((n + 7) / 8)), dim3(256), 0, st, /*pdl=*/true, z, plan, cap_rows);
}

int ln_forward(const float* x, const float* a, const float* b, float eps, long long rows, int width, float* y,
               float* mean, float* sd, cudaStream_t st, int torch_mode, void* y16, const int* rows_dev,
               const int* rowmap_out, int n) {
  if (rowmap_out && y16) { arb_set_error("ln_forward: a row-mapped output is fp32 only"); return ARB_E_INVALID_ARG; }
  if (width % 4) { arb_set_error("LayerNorm width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  if (n < 0) n = width;
  if (n > width || n <= width - 4 || (n != width && (rowmap_out || y16 || torch_mode))) {
    arb_set_error("ln_forward: a padded row needs n <= width < n + 4, fp32 dense rows and the reference's norm");
    return ARB_E_UNSUPPORTED;
  }
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * ((y16 ? 6.0 : 8.0) * width + 8), st);
  return with_row_layout(width, [&](auto LPR, auto NJ, auto FILLED) {
    const int steps = r_fwd_steps(rows), per_block = ROWS_PER_BLOCK * (32 / LPR) * steps;
    const unsigned nblk = unsigned((rows + per_block - 1) / per_block);
    return launch(n != width ? ln_fwd_kernel<LPR, NJ, false, false, true>
                  : rowmap_out ? ln_fwd_kernel<LPR, NJ, FILLED, true> : ln_fwd_kernel<LPR, NJ, FILLED, false>, dim3(nblk),
                  dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps, rows, width, y, mean, sd, torch_mode,
                  static_cast<uint16_t*>(y16), rows_dev, steps, rowmap_out, n);
  });
}

int ln_backward(const float* dy, const float* x, const float* a, const float* mean, const float* sd, float eps,
                const float* dres, long long rows, int width, float* dx, float* grad_a, float* grad_b,
                cudaStream_t st, float* dx_masked, DropSite site, float* colsum_out, int torch_mode,
                const void* dy16_in, void* dy16_out, const int* rows_dev, const int* rowmap_in, int n) {
  if (rowmap_in && dy16_in) { arb_set_error("ln_backward: a row-mapped gradient is fp32 only"); return ARB_E_INVALID_ARG; }
  if (n < 0) n = width;
  if (n > width || n <= width - 4 || (n != width && (rowmap_in || dy16_in || dy16_out || torch_mode))) {
    arb_set_error("ln_backward: a padded row needs n <= width < n + 4, fp32 dense rows and the reference's norm");
    return ARB_E_UNSUPPORTED;
  }
  if (site.thresh == 0 && site.scale == 1.0f) dx_masked = nullptr;
  if (dy16_out && dx_masked == nullptr && (site.thresh != 0 || site.scale != 1.0f)) {
    arb_set_error("ln_backward: a masked bf16 copy needs the masked fp32 buffer too"); return ARB_E_INVALID_ARG;
  }   // thresh 0 with a scale = pure rescale (positional encoding)
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * ((dres ? 16.0 : 12.0) * width + 8), st);
  return with_row_layout(width, [&](auto LPR, auto NJ, auto FILLED) {
    const int steps = r_bwd_rows_per_warp(rows) / (32 / LPR), per_block = ROWS_PER_BLOCK * (32 / LPR) * steps;
    const unsigned nblk = unsigned((rows + per_block - 1) / per_block);
    DetParts dp;
    dp.add(grad_a, nblk, 1, width, width); dp.add(grad_b, nblk, 1, width, width); dp.add(colsum_out, nblk, 1, width, width);
    if (int rc = dp.begin(st)) return rc;
    if (int rc = launch(n != width ? ln_bwd_kernel<LPR, NJ, false, false, true>
                        : rowmap_in ? ln_bwd_kernel<LPR, NJ, FILLED, true> : ln_bwd_kernel<LPR, NJ, FILLED, false>, dim3(nblk),
                        dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dy, x, a, mean, sd, eps, dres, rows, width,
                        steps, dx, grad_a, grad_b, dx_masked, site, colsum_out, torch_mode,
                        static_cast<const uint16_t*>(dy16_in), static_cast<uint16_t*>(dy16_out), rows_dev, rowmap_in, n))
      return rc;
    return dp.finish(st);
  });
}

int pos_forward(float* x, const long long* indices, const uint8_t* mask, const float* pe, int pe_rows, float scale,
                long long rows, int width, cudaStream_t st) {
  if (width % 4) { arb_set_error("positional encoding: width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * 12.0 * width, st);
  return launch(pos_fwd_kernel, dim3(unsigned((rows + 7) / 8)), dim3(256), 0, st, /*pdl=*/false, x, indices, mask, pe,
                pe_rows, scale, rows, width);
}

int pos_backward(const float* dx, const long long* indices, const uint8_t* mask, float* dpe, int pe_rows, long long rows,
                 int width, cudaStream_t st) {
  if (pe_rows < 2 || width <= 0) { arb_set_error("positional encoding: need >= 2 table rows and width > 0"); return ARB_E_INVALID_ARG; }
  if (rows == 0) return ARB_OK;
  // rows per block: a power of 2 from 64 on, the smallest whose slots (one [pe_rows - 1, width] table per block) fit
  // 2^24 floats
  const long long table = (long long)(pe_rows - 1) * width;
  long long rpb = 64;
  while (rpb < rows && (rows + rpb - 1) / rpb * table > (1LL << 24)) rpb *= 2;
  const unsigned blocks = unsigned((rows + rpb - 1) / rpb);
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * 8.0 * width, st);
  DetParts dp;
  dp.add(dpe, blocks, pe_rows - 1, width, width);     // (not the padding row: it stays as it is)
  if (int rc = dp.begin(st)) return rc;
  if (int rc = launch(pos_bwd_kernel, dim3(blocks), dim3(unsigned(std::min(256, (width + 31) / 32 * 32))), 0, st,
                      /*pdl=*/false, dx, indices, mask, dpe, pe_rows, rows, width, int(rpb)))
    return rc;
  return dp.finish(st);
}

int act_forward(float* h, long long rows, int width, int act, DropSite site, cudaStream_t st, const int* rows_dev,
                int n) {
  if (n < 0) n = width;
  if (width % 4 || n > width || n <= width - 4) { arb_set_error("activation: width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  const long long n4 = rows * width / 4;
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * 8.0 * width, st);
  const unsigned blocks = unsigned(std::min<long long>((n4 + 255) / 256, 132 * 16));
  return launch(act_fwd_kernel, dim3(blocks), dim3(256), 0, st, /*pdl=*/false, h, n4, act, site, rows_dev, width / 4,
                n);
}

int act_backward(const float* dh, const float* h, float* dz, long long rows, int width, int act, DropSite site, float mul,
                 float* colsum_out, cudaStream_t st, const int* rows_dev, int n) {
  if (n < 0) n = width;
  if (width % 4 || width > 8192 || n > width || n <= width - 4) { arb_set_error("activation: width must be a multiple of 4 and <= 8192"); return ARB_E_UNSUPPORTED; }
  int tx_n = 1;
  while (tx_n < width / 4 && tx_n < 256) tx_n *= 2;
  const int rpb = 64 * (256 / tx_n);
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * 12.0 * width, st);
  const unsigned blocks = unsigned((rows + rpb - 1) / rpb);
  DetParts dp;
  dp.add(colsum_out, blocks, 1, width, width);
  if (int rc = dp.begin(st)) return rc;
  if (int rc = launch(act_bwd_kernel, dim3(blocks), dim3(256), size_t(256 / tx_n) * width * 4, st, /*pdl=*/false, dh, h,
                      dz, rows, width, act, site, mul, tx_n, rpb, colsum_out, rows_dev, n))
    return rc;
  return dp.finish(st);
}

int softmax_forward(float* sc, const uint8_t* mask, int B, int h, int S, int pitch, cudaStream_t st, DropSite site) {
  if (S > 32 * 48) { arb_set_error("attention softmax supports slate_length <= 1536"); return ARB_E_UNSUPPORTED; }
  const long long rows = (long long)B * h * S;
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * 8.0 * S, st);
  return launch(site.thresh ? softmax_fwd_kernel<true> : softmax_fwd_kernel<false>, dim3(unsigned((rows + 7) / 8)),
                dim3(256), 0, st, /*pdl=*/false, sc, mask, B, h, S, pitch, site);
}

int softmax_backward(float* dp, float* prob, long long rows, int S, int pitch, cudaStream_t st, DropSite site) {
  if (S > 32 * 48) { arb_set_error("attention softmax supports slate_length <= 1536"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * (site.thresh ? 16.0 : 12.0) * S, st);
  return launch(site.thresh ? softmax_bwd_kernel<true> : softmax_bwd_kernel<false>, dim3(unsigned((rows + 7) / 8)),
                dim3(256), 0, st, /*pdl=*/false, dp, prob, rows, S, pitch, site);
}

int slate_extents(const uint8_t* mask, const float* dscores, int n_out, int B, int S, int* extent, cudaStream_t st) {
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(B) * S * (dscores ? 1.0 + 4.0 * n_out : 1.0), st);
  return launch(slate_extent_kernel, dim3(unsigned((B + 7) / 8)), dim3(256), 0, st, /*pdl=*/true, mask, dscores, n_out, B,
                S, extent);
}

int convert_to_bf16(const float* src, void* dst, long long n, cudaStream_t st) {
  const long long n4 = (n + 3) / 4;
  ProfScope ps(ARB_PROF_SCORER_SIMT, 6.0 * double(n), st);
  return launch(to_bf16_kernel, dim3(unsigned(std::max<long long>(1, std::min<long long>((n4 + 255) / 256, 132 * 8)))), dim3(256), 0, st,
                /*pdl=*/true, reinterpret_cast<const float4*>(src), static_cast<uint2*>(dst), n);
}

int tf32_weight_copy(const float* P, long long n, const WeightMats& m, int rnd, float* pr, float* pt, cudaStream_t st) {
  ProfScope ps(ARB_PROF_SCORER_SIMT, 12.0 * double(n), st);
  return launch(tf32_weight_copy_kernel, dim3(unsigned(std::max<long long>(1, std::min<long long>((n + 255) / 256, 132 * 8)))),
                dim3(256), 0, st, /*pdl=*/true, P, n, m, rnd, pr, pt);
}

int head_pad_copy(const float* pr, const float* P, const HeadPad& m, float* out, cudaStream_t st) {
  const long long n = m.size() * m.n_layers;
  ProfScope ps(ARB_PROF_SCORER_SIMT, 8.0 * double(n), st);
  return launch(head_pad_copy_kernel, dim3(unsigned(std::max<long long>(1, std::min<long long>((n + 255) / 256, 132 * 8)))),
                dim3(256), 0, st, /*pdl=*/true, pr, P, m, out);
}

int head_pad_grads(const float* gp, const HeadPad& m, int l, float* G, cudaStream_t st) {
  const long long n = 4LL * m.d * m.d + 3LL * m.d;
  ProfScope ps(ARB_PROF_SCORER_SIMT, 12.0 * double(n), st);
  return launch(head_pad_grads_kernel, dim3(unsigned(std::max<long long>(1, std::min<long long>((n + 255) / 256, 132 * 8)))),
                dim3(256), 0, st, /*pdl=*/true, gp, m, m.enc0 + l * m.enc_stride, G);
}

int colsum_accumulate(const float* in, long long rows, int width, long long ld, float* out, cudaStream_t st) {
  if (width % 4 || ld % 4) { arb_set_error("colsum: width and pitch must be multiples of 4"); return ARB_E_UNSUPPORTED; }
  const int rpb = 256;
  const unsigned blocks = unsigned((rows + rpb - 1) / rpb);
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * 4.0 * width, st);
  DetParts dp;
  dp.add(out, blocks, 1, width, width);
  int rc = dp.begin(st);
  if (rc) return rc;
  ARB_DISPATCH_NV(width, (rc = launch(colsum_kernel<NV>, dim3(blocks), dim3(256), 0, st, /*pdl=*/false, in, rows, width, ld, rpb, out)));
  if (rc) return rc;
  return dp.finish(st);
}

int head_forward(const float* x, const float* a, const float* b, float eps, const float* w, const float* wb,
                 int has_norm, int act, long long rows, int width, float* score, float* mean, float* sd,
                 cudaStream_t st, const int* rows_dev, const int* rowmap) {
  if (width % 4) { arb_set_error("model width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * (4.0 * width + 12), st);
  return with_row_layout(width, [&](auto LPR, auto NJ, auto FILLED) {
    const int steps = r_fwd_steps(rows), per_block = ROWS_PER_BLOCK * (32 / LPR) * steps;
    const unsigned nblk = unsigned((rows + per_block - 1) / per_block);
    return launch(head_fwd_kernel<LPR, NJ, FILLED>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps,
                  w, wb, has_norm, act, rows, width, score, mean, sd, rows_dev, rowmap, steps);
  });
}

int head_backward(const float* dscore, const float* score, const float* x, const float* a, const float* b,
                  const float* mean, const float* sd, float eps, const float* w, const float* wb, int has_norm,
                  int act, long long rows, int width, float* dx, float* grad_a, float* grad_b, float* grad_w,
                  float* grad_wb, cudaStream_t st, float* dx_masked, DropSite site, float* colsum_out, void* dy16_out,
                  const int* rows_dev, const int* rowmap) {
  if (site.thresh == 0) dx_masked = nullptr;
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * (8.0 * width + 16), st);
  return with_row_layout(width, [&](auto LPR, auto NJ, auto FILLED) {
    const int steps = r_bwd_rows_per_warp(rows) / (32 / LPR), per_block = ROWS_PER_BLOCK * (32 / LPR) * steps;
    const unsigned nblk = unsigned((rows + per_block - 1) / per_block);
    DetParts dp;
    if (has_norm) { dp.add(grad_a, nblk, 1, width, width); dp.add(grad_b, nblk, 1, width, width); }
    dp.add(grad_w, nblk, 1, width, width); dp.add(colsum_out, nblk, 1, width, width); dp.add(grad_wb, nblk, 1, 1, 1);
    if (int rc = dp.begin(st)) return rc;
    if (int rc = launch(head_bwd_kernel<LPR, NJ, FILLED>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dscore,
                        score, x, a, b, mean, sd, eps, w, has_norm, act, rows, width, steps, dx, grad_a, grad_b, grad_w,
                        grad_wb, dx_masked, site, colsum_out, static_cast<uint16_t*>(dy16_out), rows_dev, rowmap))
      return rc;
    return dp.finish(st);
  });
}

int head_multi_forward(const float* xf, const float* w, const float* wb, int act, long long rows, int width, int n,
                       float* score, cudaStream_t st) {
  if (width % 4) { arb_set_error("model width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  const unsigned blocks = unsigned((rows + ROWS_PER_BLOCK - 1) / ROWS_PER_BLOCK);
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * (4.0 * width + 4.0 * n), st);
  int rc;
  ARB_DISPATCH_NV(width, (rc = launch(head_multi_fwd_kernel<NV>, dim3(blocks), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/false, xf, w, wb, act, rows, width, n, score)));
  return rc;
}

int head_multi_backward(const float* dscore, const float* score, const float* xf, const float* w, int act,
                        long long rows, int width, int n, float* dxf, float* grad_w, float* grad_wb, cudaStream_t st,
                        float* dx_masked, DropSite site, float* colsum_out) {
  if (site.thresh == 0) dx_masked = nullptr;
  const int rpw = 8;    // rows per warp: more = fewer block slots of grad_w per byte moved
  const unsigned blocks = unsigned((rows + ROWS_PER_BLOCK * rpw - 1) / (ROWS_PER_BLOCK * rpw));
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * (8.0 * width + 8.0 * n), st);
  DetParts dp;
  dp.add(grad_w, blocks, 1, (long long)n * width, (long long)n * width); dp.add(grad_wb, blocks, 1, n, n);
  dp.add(colsum_out, blocks, 1, width, width);
  int rc = dp.begin(st);
  if (rc) return rc;
  ARB_DISPATCH_NV(width, (rc = launch(head_multi_bwd_kernel<NV>, dim3(blocks), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/false, dscore, score, xf, w, act, rows, width, n, rpw, dxf, grad_w, grad_wb, dx_masked, site, colsum_out)));
  if (rc) return rc;
  return dp.finish(st);
}

}  // namespace arb

// ------------------------------------------------------------------------------------------------ test entry points
// The row kernels on their own (include/allrank_b200.h): argument checks, then the launchers above, so that the steps
// per warp, the row layout and the DetParts slots are the ones the scorer gets for the same row count.
using namespace arb;

static int row_args(const char* what, bool ptrs_ok, long long rows, int width, float p) {
  if (!ptrs_ok) { arb_set_error((std::string(what) + ": null pointer").c_str()); return ARB_E_INVALID_ARG; }
  if (rows < 0) { arb_set_error((std::string(what) + ": rows must be >= 0").c_str()); return ARB_E_INVALID_ARG; }
  if (!(p >= 0.0f && p < 1.0f)) { arb_set_error((std::string(what) + ": dropout rate must be in [0, 1)").c_str()); return ARB_E_INVALID_ARG; }
  if (width <= 0 || width % 4 || width > 1024) {
    arb_set_error((std::string(what) + ": the width must be a positive multiple of 4, at most 1024").c_str());
    return ARB_E_UNSUPPORTED;
  }
  return ARB_OK;
}
#define ARB_ROW_ARGS(what, ptrs_ok, rows, width, p) \
  do { if (int rc__ = row_args(what, ptrs_ok, rows, width, p)) return rc__; if ((rows) == 0) return ARB_OK; } while (0)

static DropSite test_site(uint64_t seed, int layer, int site, float p) {
  return make_drop_site(CallSeed{seed, nullptr}, layer, site, p);
}

extern "C" int32_t arb_layernorm_forward(const float* x, const float* a, const float* b, float eps, int32_t torch_mode,
                                         int64_t rows, int32_t width, float* y, void* y16, float* mean, float* sd,
                                         const int32_t* rows_dev, const int32_t* rowmap, void* stream) {
  ARB_ROW_ARGS("arb_layernorm_forward", x && a && b && (y || y16) && mean && sd, rows, width, 0.0f);
  return ln_forward(x, a, b, eps, rows, width, y, mean, sd, static_cast<cudaStream_t>(stream), torch_mode, y16,
                    rows_dev, rowmap);
}

extern "C" int32_t arb_layernorm_backward(const float* dy, const void* dy16_in, const float* x, const float* a,
                                          const float* mean, const float* sd, float eps, int32_t torch_mode,
                                          const float* dres, int64_t rows, int32_t width, float* dx, float* grad_a,
                                          float* grad_b, float* dx_masked, void* dy16_out, float* colsum_out, float p,
                                          uint64_t seed, int32_t layer, int32_t site, const int32_t* rows_dev,
                                          const int32_t* rowmap, void* stream) {
  ARB_ROW_ARGS("arb_layernorm_backward", (dy || dy16_in) && x && a && mean && sd && dx, rows, width, p);
  return ln_backward(dy, x, a, mean, sd, eps, dres, rows, width, dx, grad_a, grad_b, static_cast<cudaStream_t>(stream),
                     dx_masked, test_site(seed, layer, site, p), colsum_out, torch_mode, dy16_in, dy16_out, rows_dev,
                     rowmap);
}

extern "C" int32_t arb_head_forward(const float* x, const float* a, const float* b, float eps, const float* w,
                                    const float* wb, int32_t has_norm, int32_t act, int64_t rows, int32_t width,
                                    float* score, float* mean, float* sd, const int32_t* rows_dev,
                                    const int32_t* rowmap, void* stream) {
  ARB_ROW_ARGS("arb_head_forward", act_known(act) && x && w && wb && score && (!has_norm || (a && b)) && !mean == !sd, rows, width, 0.0f);
  return head_forward(x, a, b, eps, w, wb, has_norm, act, rows, width, score, mean, sd,
                      static_cast<cudaStream_t>(stream), rows_dev, rowmap);
}

extern "C" int32_t arb_head_backward(const float* dscore, const float* score, const float* x, const float* a,
                                     const float* b, const float* mean, const float* sd, float eps, const float* w,
                                     int32_t has_norm, int32_t act, int64_t rows, int32_t width, float* dx,
                                     float* grad_a, float* grad_b, float* grad_w, float* grad_wb, float* dx_masked,
                                     void* dy16_out, float* colsum_out, float p, uint64_t seed, int32_t layer,
                                     int32_t site, const int32_t* rows_dev, const int32_t* rowmap, void* stream) {
  ARB_ROW_ARGS("arb_head_backward",
               act_known(act) && dscore && score && x && w && dx && (!has_norm || (a && b && mean && sd)),
               rows, width, p);
  return head_backward(dscore, score, x, a, b, mean, sd, eps, w, nullptr, has_norm, act, rows, width, dx, grad_a,
                       grad_b, grad_w, grad_wb, static_cast<cudaStream_t>(stream), dx_masked,
                       test_site(seed, layer, site, p), colsum_out, dy16_out, rows_dev, rowmap);
}

extern "C" int32_t arb_head_multi_forward(const float* xf, const float* w, const float* wb, int32_t act, int64_t rows,
                                          int32_t width, int32_t n, float* score, void* stream) {
  ARB_ROW_ARGS("arb_head_multi_forward", act_known(act) && xf && w && wb && score && n >= 1, rows, width, 0.0f);
  return head_multi_forward(xf, w, wb, act, rows, width, n, score, static_cast<cudaStream_t>(stream));
}

extern "C" int32_t arb_head_multi_backward(const float* dscore, const float* score, const float* xf, const float* w,
                                           int32_t act, int64_t rows, int32_t width, int32_t n, float* dxf,
                                           float* grad_w, float* grad_wb, float* dx_masked, float* colsum_out, float p,
                                           uint64_t seed, int32_t layer, int32_t site, void* stream) {
  ARB_ROW_ARGS("arb_head_multi_backward",
               act_known(act) && dscore && score && xf && w && dxf && n >= 1 && !grad_w == !grad_wb, rows, width, p);
  return head_multi_backward(dscore, score, xf, w, act, rows, width, n, dxf, grad_w, grad_wb,
                             static_cast<cudaStream_t>(stream), dx_masked, test_site(seed, layer, site, p), colsum_out);
}

extern "C" int32_t arb_column_sums(const float* in, int64_t rows, int32_t width, int64_t ld, float* out, void* stream) {
  ARB_ROW_ARGS("arb_column_sums", in && out && ld >= width, rows, width, 0.0f);
  return colsum_accumulate(in, rows, width, ld, out, static_cast<cudaStream_t>(stream));
}

static int softmax_args(const char* what, bool ptrs_ok, int S, int pitch, float p) {
  if (!ptrs_ok) { arb_set_error((std::string(what) + ": null pointer or no rows").c_str()); return ARB_E_INVALID_ARG; }
  if (S <= 0 || pitch < S) { arb_set_error((std::string(what) + ": S >= 1 and pitch >= S").c_str()); return ARB_E_INVALID_ARG; }
  if (!(p >= 0.0f && p < 1.0f)) { arb_set_error((std::string(what) + ": dropout rate must be in [0, 1)").c_str()); return ARB_E_INVALID_ARG; }
  return ARB_OK;
}

extern "C" int32_t arb_softmax_forward(float* scores, const uint8_t* mask, int32_t B, int32_t h, int32_t S,
                                       int32_t pitch, float p, uint64_t seed, int32_t layer, void* stream) {
  if (int rc = softmax_args("arb_softmax_forward", scores && mask && B >= 1 && h >= 1, S, pitch, p))
    return rc;
  return softmax_forward(scores, mask, B, h, S, pitch, static_cast<cudaStream_t>(stream),
                         test_site(seed, layer, SITE_ATTN_P, p));
}

extern "C" int32_t arb_softmax_backward(float* dprob, float* prob, int64_t rows, int32_t S, int32_t pitch, float p,
                                        uint64_t seed, int32_t layer, void* stream) {
  if (int rc = softmax_args("arb_softmax_backward", dprob && prob && rows >= 1, S, pitch, p)) return rc;
  return softmax_backward(dprob, prob, rows, S, pitch, static_cast<cudaStream_t>(stream),
                          test_site(seed, layer, SITE_ATTN_P, p));
}

// The activation, positional-encoding and packed-row kernels on their own (include/allrank_b200.h), through the
// scorer's launchers.
extern "C" int32_t arb_activation_forward(float* h, int64_t rows, int32_t width, int32_t act, float p, uint64_t seed,
                                          int32_t layer, const int32_t* rows_dev, void* stream) {
  if (!h || rows < 0 || width <= 0 || !act_known(act) || !(p >= 0.0f && p < 1.0f)) {
    arb_set_error("arb_activation_forward: null pointer or bad argument"); return ARB_E_INVALID_ARG;
  }
  if (rows == 0) return width % 4 ? ARB_E_UNSUPPORTED : ARB_OK;
  return act_forward(h, rows, width, act, test_site(seed, layer, SITE_FC, p), static_cast<cudaStream_t>(stream), rows_dev);
}

extern "C" int32_t arb_activation_backward(const float* dh, const float* h, float* dz, int64_t rows, int32_t width,
                                           int32_t act, float p, uint64_t seed, int32_t layer, float mul,
                                           float* colsum_out, const int32_t* rows_dev, void* stream) {
  if (!dh || !h || !dz || dz == h || rows < 0 || width <= 0 || !act_known(act) ||
      !(p >= 0.0f && p < 1.0f)) {
    arb_set_error("arb_activation_backward: null pointer, dz aliasing h, or bad argument"); return ARB_E_INVALID_ARG;
  }
  if (rows == 0) return ARB_OK;
  return act_backward(dh, h, dz, rows, width, act, test_site(seed, layer, SITE_FC, p), mul, colsum_out,
                      static_cast<cudaStream_t>(stream), rows_dev);
}

extern "C" int32_t arb_positional_forward(float* x, const int64_t* indices, const uint8_t* mask, const float* pe,
                                          int32_t pe_rows, float scale, int64_t rows, int32_t width, void* stream) {
  if (!x || !indices || !mask || !pe || pe_rows < 2 || rows < 0 || width <= 0) {
    arb_set_error("arb_positional_forward: null pointer or bad argument"); return ARB_E_INVALID_ARG;
  }
  if (rows == 0) return ARB_OK;
  return pos_forward(x, reinterpret_cast<const long long*>(indices), mask, pe, pe_rows, scale, rows, width,
                     static_cast<cudaStream_t>(stream));
}

extern "C" int32_t arb_positional_backward(const float* dx, const int64_t* indices, const uint8_t* mask, float* dpe,
                                           int32_t pe_rows, int64_t rows, int32_t width, void* stream) {
  if (!dx || !indices || !mask || !dpe || rows < 0) {
    arb_set_error("arb_positional_backward: null pointer or bad argument"); return ARB_E_INVALID_ARG;
  }
  return pos_backward(dx, reinterpret_cast<const long long*>(indices), mask, dpe, pe_rows, rows, width,
                      static_cast<cudaStream_t>(stream));
}

extern "C" int32_t arb_slate_extents(const uint8_t* mask, const float* dscores, int32_t n_out, int32_t B, int32_t S,
                                     int32_t* extent, void* stream) {
  if (!mask || !extent || B <= 0 || S <= 0 || (dscores && n_out < 1)) {
    arb_set_error("arb_slate_extents: null pointer or bad argument"); return ARB_E_INVALID_ARG;
  }
  return slate_extents(mask, dscores, n_out, B, S, extent, static_cast<cudaStream_t>(stream));
}

static int pack_args(const char* what, bool ptrs_ok, int B, int S, long long cap_rows) {
  if (!ptrs_ok || B <= 0 || S <= 0 || cap_rows < (long long)B * ((S + 15) / 16 * 16)) {
    arb_set_error((std::string(what) + ": null pointer, bad shape, or cap_rows below B * round_up(S, 16)").c_str());
    return ARB_E_INVALID_ARG;
  }
  return ARB_OK;
}

extern "C" int32_t arb_pack_plan(const float* x, const int32_t* ext, int32_t B, int32_t S, int32_t F, int32_t* off,
                                 int32_t* plan, int32_t* rowmap, float* xc, int64_t cap_rows, void* stream) {
  if (int rc = pack_args("arb_pack_plan", x && ext && off && plan && rowmap && xc && F > 0, B, S, cap_rows)) return rc;
  return pack_plan(x, ext, B, S, F, off, plan, rowmap, xc, cap_rows, static_cast<cudaStream_t>(stream));
}

extern "C" int32_t arb_zero_rows(float* p, int32_t pitch, int32_t width, int32_t from, int32_t n, const int32_t* plan,
                                 int64_t cap_rows, void* stream) {
  if (!p || !plan || width <= 0 || pitch < width || (from != 0 && from != 1) || n < 0 || cap_rows < 0) {
    arb_set_error("arb_zero_rows: null pointer or bad argument"); return ARB_E_INVALID_ARG;
  }
  ZeroRegions z;
  z.add(p, pitch, width, from, n);
  return zero_rows(z, plan, cap_rows, static_cast<cudaStream_t>(stream));
}

extern "C" int32_t arb_scatter_rows(const float* src, const int32_t* plan, const int32_t* rowmap, int64_t cap_rows,
                                    int32_t width, float* dst, void* stream) {
  if (!src || !plan || !rowmap || !dst || cap_rows <= 0 || width <= 0) {
    arb_set_error("arb_scatter_rows: null pointer or bad argument"); return ARB_E_INVALID_ARG;
  }
  return scatter_rows(src, plan, rowmap, cap_rows, width, dst, static_cast<cudaStream_t>(stream));
}
