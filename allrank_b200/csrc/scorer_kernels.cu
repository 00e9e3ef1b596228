// SIMT kernels of the scorer (everything that is not a tensor-core contraction):
//   row LayerNorm forward / backward (the reference's custom LayerNorm: unbiased std, eps added to the std,
//   allrank/models/transformer.py:59-81), key-masked row softmax forward / backward (transformer.py:148-153),
//   bias-gradient column sums, final LayerNorm + linear head forward / backward (model.py:111-117).
// All are one-warp-per-row, coalesced 128-bit accesses where the width allows, warp-shuffle reductions;
// they are HBM-bound (DESIGN.md section 3 lists bytes per row).
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#include "block_utils.cuh"
#include "common.h"
#include "defaults.h"
#include "dropout.cuh"
#include "scorer_kernels.h"

namespace arb {

constexpr int ROWS_PER_BLOCK = 8;   // 8 warps

// Each lane owns columns lane*4 + 128*k .. +3 (float4), k < NV; width must be a multiple of 4 and <= 128*NV.
template <int NV>
struct RowRegs {
  float4 v[NV];
};

template <int NV>
__device__ __forceinline__ void load_row(const float* __restrict__ p, int width, int lane, RowRegs<NV>& r) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane * 4 + 128 * k;
    r.v[k] = (c < width) ? *reinterpret_cast<const float4*>(p + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
template <int NV>
__device__ __forceinline__ void store_row(float* __restrict__ p, int width, int lane, const RowRegs<NV>& r) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane * 4 + 128 * k;
    if (c < width) *reinterpret_cast<float4*>(p + c) = r.v[k];
  }
}

// bf16 rows (the scorer's bf16 mode keeps GEMM operands -- LayerNorm outputs, hidden activations, the gradients that
// feed weight / input-gradient products -- as bfloat16): a lane's 4 elements are 8 bytes.
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
template <int NV>
__device__ __forceinline__ void load_row_bf16(const uint16_t* __restrict__ p, int width, int lane, RowRegs<NV>& r) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane * 4 + 128 * k;
    if (c < width) {
      const uint2 u = *reinterpret_cast<const uint2*>(p + c);
      r.v[k] = make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u),
                           __uint_as_float(u.y << 16), __uint_as_float(u.y & 0xffff0000u));
    } else {
      r.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}
template <int NV>
__device__ __forceinline__ void store_row_bf16(uint16_t* __restrict__ p, int width, int lane, const RowRegs<NV>& r) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane * 4 + 128 * k;
    if (c < width)
      *reinterpret_cast<uint2*>(p + c) = make_uint2(pack_bf16x2(r.v[k].x, r.v[k].y), pack_bf16x2(r.v[k].z, r.v[k].w));
  }
}

template <int NV>
__device__ __forceinline__ void apply_drop(RowRegs<NV>& r, long long row, int width, int lane, const DropSite& site) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int c = lane * 4 + 128 * k;
    float* v = &r.v[k].x;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const unsigned long long idx = (unsigned long long)row * (unsigned long long)width + (c + e);
      v[e] = drop_keep(idx, site.seed, site.thresh) ? v[e] * site.scale : 0.0f;
    }
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm fwd
// y = a * (x - mean) / (std_unbiased + eps) + b ; saves mean and std per row.
// A warp owns FWD_RPW consecutive rows and issues all their loads before the first reduction: one row per warp leaves
// only 512 B in flight per warp at d_model = 128, far too little to cover the HBM latency (Little's law).
constexpr int FWD_RPW = 4;
// ... and it walks FWD_NB such batches, the loads of the next batch issued before the arithmetic of the current one: a
// warp that retires after a single batch spends a third of its life waiting for its first loads and for a new block
// to be scheduled (ln_forward sat at 0.66 of the HBM roof, the head at 0.31).  Wide rows (NV > 2) keep one batch: two
// batches of them do not fit the register file.
template <int NV>
struct FwdBatches { static constexpr int value = NV <= 2 ? 4 : 1; };
// (small launches keep one batch per warp: more batches would leave SMs without a block -- B = 64 has 8 k live rows)
static inline int fwd_batches_for(int width, long long rows) { return (width <= 256 && rows >= (1 << 17)) ? 4 : 1; }

// MAP: packed rows with a row-mapped output (rowmap_out); a template flag so that the plain kernels compile unchanged
template <int NV, bool MAP>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) ln_fwd_kernel(const float* __restrict__ x,
                                                                    const float* __restrict__ a,
                                                                    const float* __restrict__ b, float eps,
                                                                    long long rows, int width,
                                                                    float* __restrict__ y, float* __restrict__ mean_o,
                                                                    float* __restrict__ std_o, int torch_mode,
                                                                    uint16_t* __restrict__ y16,
                                                                    const int* __restrict__ rows_dev, int n_batches,
                                                                    const int* __restrict__ rowmap_out) {
  arb_pdl_wait();
  constexpr int NBMAX = FwdBatches<NV>::value;
  const int NB = NBMAX > 1 ? n_batches : 1;
  const int lane = threadIdx.x & 31;
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5)) * (FWD_RPW * NB);
  if (base >= rows) return;
  // packed rows: the live row count lives on the device.  Its load is issued WITH the first row loads (every row below
  // the host-side bound is readable) and consulted afterwards.
  const long long live = rows_dev ? (long long)__ldg(rows_dev) : rows;
  // (a multi-batch warp amortises the wait for the count over 16 rows and must not fetch rows beyond it: the dead half
  // of a packed launch would otherwise read 12 % extra; a single-batch warp overlaps it with its only fetch)
  if (NB > 1) { rows = min(rows, live); if (base >= rows) return; }
  RowRegs<NV> r[FWD_RPW], rn[FWD_RPW], ga, gb;
  auto fetch = [&](long long r0, RowRegs<NV>(&dst)[FWD_RPW]) {
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) {
      if (r0 + q < rows) load_row<NV>(x + (r0 + q) * width, width, lane, dst[q]);
      else {
#pragma unroll
        for (int k = 0; k < NV; ++k) dst[q].v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  fetch(base, r);
  load_row<NV>(a, width, lane, ga);
  load_row<NV>(b, width, lane, gb);
  rows = min(rows, live);
#pragma unroll 1
  for (int nb = 0; nb < NB; ++nb) {
    const long long row0 = base + nb * FWD_RPW;
    if (row0 >= rows) break;
    if (NBMAX > 1 && nb + 1 < NB) fetch(row0 + FWD_RPW, rn);
    float mean[FWD_RPW], sd[FWD_RPW];
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) {
      float s = 0.f;
#pragma unroll
      for (int k = 0; k < NV; ++k) s += r[q].v[k].x + r[q].v[k].y + r[q].v[k].z + r[q].v[k].w;
      mean[q] = s;
    }
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) mean[q] = warp_sum(mean[q]) / float(width);
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) {
      float ss = 0.f;
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const int c = lane * 4 + 128 * k;
        if (c < width) {
          const float d0 = r[q].v[k].x - mean[q], d1 = r[q].v[k].y - mean[q], d2 = r[q].v[k].z - mean[q],
                      d3 = r[q].v[k].w - mean[q];
          ss += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
        }
      }
      sd[q] = ss;
    }
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) sd[q] = warp_sum(sd[q]);
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) {
      if (row0 + q >= rows) break;
      // torch_mode: nn.LayerNorm (biased variance, eps inside the root; FCModel's input_norm, model.py:27) -- the saved
      // "std" is then sqrt(var + eps) and the backward is called with eps = 0
      const float sdq = torch_mode ? sqrtf(sd[q] / float(width) + eps) : sqrtf(sd[q] / float(width - 1));
      // one reciprocal per row instead of a division per element: the kernel is bound by instruction issue as much as
      // by HBM (an IEEE division is ~10 instructions), and a * (x - mean) * (1 / (std + eps)) differs from the
      // reference's a * (x - mean) / (std + eps) by one rounding (6e-8 relative)
      const float rinv = 1.0f / (torch_mode ? sdq : sdq + eps);
      const float m = mean[q];
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        r[q].v[k].x = ga.v[k].x * (r[q].v[k].x - m) * rinv + gb.v[k].x;
        r[q].v[k].y = ga.v[k].y * (r[q].v[k].y - m) * rinv + gb.v[k].y;
        r[q].v[k].z = ga.v[k].z * (r[q].v[k].z - m) * rinv + gb.v[k].z;
        r[q].v[k].w = ga.v[k].w * (r[q].v[k].w - m) * rinv + gb.v[k].w;
      }
      if (y16) store_row_bf16<NV>(y16 + (row0 + q) * width, width, lane, r[q]);   // bf16 mode: the GEMM operand copy only
      else {   // packed rows with rowmap_out: row r goes to y[rowmap_out[r]] (alignment rows: nowhere)
        const long long yr = MAP ? (long long)rowmap_out[row0 + q] : row0 + q;
        if (!MAP || yr >= 0) store_row<NV>(y + yr * width, width, lane, r[q]);
      }
      if (lane == 0) { mean_o[row0 + q] = m; std_o[row0 + q] = sdq; }
    }
    if (NBMAX > 1) {
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) {
#pragma unroll
        for (int k = 0; k < NV; ++k) r[q].v[k] = rn[q].v[k];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm bwd
// dx = [dres +] r (dxh - mean(dxh)) - r^2 (sum_k dxh_k c_k) / ((d-1) std) * c,   dxh = dy * a, c = x - mean,
// r = 1/(std+eps).   grad_a += sum_rows dy * xhat,  grad_b += sum_rows dy  (block partials -> DetParts slots).
// MAP: packed rows reading a row-mapped gradient (rowmap_in); a template flag as in ln_fwd_kernel
template <int NV, bool MAP>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32, NV == 1 ? 4 : 1) ln_bwd_kernel(const float* __restrict__ dy,
                                                                    const float* __restrict__ x,
                                                                    const float* __restrict__ a,
                                                                    const float* __restrict__ mean_i,
                                                                    const float* __restrict__ std_i, float eps,
                                                                    const float* __restrict__ dres, long long rows,
                                                                    int width, int rows_per_warp,
                                                                    float* __restrict__ dx, float* __restrict__ grad_a,
                                                                    float* __restrict__ grad_b,
                                                                    float* __restrict__ dx_masked, DropSite site,
                                                                    float* __restrict__ colsum_out, int torch_mode,
                                                                    const uint16_t* __restrict__ dy16_in,
                                                                    uint16_t* __restrict__ dy16_out,
                                                                    const int* __restrict__ rows_dev,
                                                                    const int* __restrict__ rowmap_in) {
  arb_pdl_wait();
  if (rows_dev) {
    rows = min(rows, (long long)__ldg(rows_dev));
    if ((long long)blockIdx.x * ROWS_PER_BLOCK * rows_per_warp >= rows) return;   // whole block beyond the packed rows
  }
  __shared__ float sh[ROWS_PER_BLOCK][128 * NV + 4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  RowRegs<NV> ga, acc_a, acc_b, acc_c;
  load_row<NV>(a, width, lane, ga);
#pragma unroll
  for (int k = 0; k < NV; ++k) acc_a.v[k] = acc_b.v[k] = acc_c.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  const long long first = ((long long)blockIdx.x * ROWS_PER_BLOCK + wid) * rows_per_warp;
  // Software pipeline over the warp's rows: the loads of row it+1 (dy, x, residual gradient, statistics) are issued
  // before the reductions of row it, so two rows of traffic are in flight per warp.
  RowRegs<NV> g, xr, res, g_n, xr_n, res_n;
  float mean = 0.f, sd = 1.f, mean_n = 0.f, sd_n = 1.f;
  auto fetch = [&](long long row, RowRegs<NV>& gg, RowRegs<NV>& xx, RowRegs<NV>& rr, float& mm, float& ss) {
    if (dy16_in) load_row_bf16<NV>(dy16_in + row * width, width, lane, gg);
    else if (MAP) {   // packed rows: dy of row r is dy[rowmap_in[r]]; alignment rows have a zero gradient
      const long long src = rowmap_in[row];
      if (src >= 0) load_row<NV>(dy + src * width, width, lane, gg);
      else {
#pragma unroll
        for (int k = 0; k < NV; ++k) gg.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else load_row<NV>(dy + row * width, width, lane, gg);
    load_row<NV>(x + row * width, width, lane, xx);
    if (dres) load_row<NV>(dres + row * width, width, lane, rr);
    mm = mean_i[row]; ss = std_i[row];
  };
  if (first < rows) fetch(first, g, xr, res, mean, sd);
  for (int it = 0; it < rows_per_warp; ++it) {
    const long long row = first + it;
    if (row >= rows) break;
    const bool more = it + 1 < rows_per_warp && row + 1 < rows;
    if (more) fetch(row + 1, g_n, xr_n, res_n, mean_n, sd_n);
    const float r = 1.0f / (sd + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int c = lane * 4 + 128 * k;
      float* gv = &g.v[k].x;
      float* xv = &xr.v[k].x;
      const float* av = &ga.v[k].x;
      float* aa = &acc_a.v[k].x;
      float* ab = &acc_b.v[k].x;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float cc = (c < width) ? xv[e] - mean : 0.f;
        const float dyv = gv[e];
        aa[e] += dyv * cc * r;     // dy * xhat
        ab[e] += dyv;
        const float dxh = dyv * av[e];
        gv[e] = dxh;
        xv[e] = cc;
        s1 += dxh;
        s2 += dxh * cc;
      }
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    const float m1 = s1 / float(width);
    const float coef = torch_mode ? r * r * r * s2 / float(width)
                                  : ((sd > 0.f) ? r * r * s2 / (float(width - 1) * sd) : 0.f);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float* gv = &g.v[k].x;
      const float* xv = &xr.v[k].x;
      const float* rv = &res.v[k].x;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float o = r * (gv[e] - m1) - coef * xv[e];
        if (dres) o += rv[e];
        gv[e] = o;
      }
    }
    store_row<NV>(dx + row * width, width, lane, g);
    if (dx_masked) {   // the same gradient through the dropout of the sublayer below (mask regenerated)
      apply_drop<NV>(g, row, width, lane, site);
      store_row<NV>(dx_masked + row * width, width, lane, g);
    }
    // bf16 mode: the copy the weight / input-gradient GEMMs of the sublayer below read (after its dropout mask)
    if (dy16_out) store_row_bf16<NV>(dy16_out + row * width, width, lane, g);
    if (colsum_out) {  // bias gradient of the linear below = column sums of what that linear receives
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        acc_c.v[k].x += g.v[k].x; acc_c.v[k].y += g.v[k].y; acc_c.v[k].z += g.v[k].z; acc_c.v[k].w += g.v[k].w;
      }
    }
    if (more) {
#pragma unroll
      for (int k = 0; k < NV; ++k) { g.v[k] = g_n.v[k]; xr.v[k] = xr_n.v[k]; res.v[k] = res_n.v[k]; }
      mean = mean_n; sd = sd_n;
    }
  }
  // block-level reduction of the gain/bias gradients
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    float* dst = pass == 0 ? grad_a : (pass == 1 ? grad_b : colsum_out);
    if (!dst) continue;      // (no parameter gradients requested: grad_a / grad_b are null)
    const RowRegs<NV>& src = pass == 0 ? acc_a : (pass == 1 ? acc_b : acc_c);
#pragma unroll
    for (int k = 0; k < NV; ++k) *reinterpret_cast<float4*>(&sh[wid][lane * 4 + 128 * k]) = src.v[k];
    __syncthreads();
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < ROWS_PER_BLOCK; ++w) t += sh[w][c];
      dst[size_t(blockIdx.x) * width + c] = t;      // this block's slot (DetParts)
    }
    __syncthreads();
  }
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
  __shared__ float sh[8][128 * NV + 4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = min(rows, r0 + rows_per_block);
  RowRegs<NV> acc;
#pragma unroll
  for (int k = 0; k < NV; ++k) acc.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  long long r = r0 + wid;
  for (; r + 24 < r1; r += 32) {
    RowRegs<NV> a0, a1, a2, a3;
    load_row<NV>(in + r * ld, width, lane, a0);
    load_row<NV>(in + (r + 8) * ld, width, lane, a1);
    load_row<NV>(in + (r + 16) * ld, width, lane, a2);
    load_row<NV>(in + (r + 24) * ld, width, lane, a3);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      acc.v[k].x += (a0.v[k].x + a1.v[k].x) + (a2.v[k].x + a3.v[k].x);
      acc.v[k].y += (a0.v[k].y + a1.v[k].y) + (a2.v[k].y + a3.v[k].y);
      acc.v[k].z += (a0.v[k].z + a1.v[k].z) + (a2.v[k].z + a3.v[k].z);
      acc.v[k].w += (a0.v[k].w + a1.v[k].w) + (a2.v[k].w + a3.v[k].w);
    }
  }
  for (; r < r1; r += 8) {
    RowRegs<NV> a0;
    load_row<NV>(in + r * ld, width, lane, a0);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      acc.v[k].x += a0.v[k].x; acc.v[k].y += a0.v[k].y; acc.v[k].z += a0.v[k].z; acc.v[k].w += a0.v[k].w;
    }
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) *reinterpret_cast<float4*>(&sh[wid][lane * 4 + 128 * k]) = acc.v[k];
  __syncthreads();
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sh[w][c];
    out[size_t(blockIdx.x) * width + c] = t;        // this block's slot (DetParts)
  }
}

// ------------------------------------------------------------------------------------------------ head fwd
// score = act( w . LN(x) + bias )  (final encoder LayerNorm fused; has_norm = 0 for FC-only models)
__device__ __forceinline__ float act_fwd(float z, int act) {
  if (act == ARB_ACT_TANH) return tanhf(z);
  if (act == ARB_ACT_SIGMOID) return 1.0f / (1.0f + expf(-z));
  if (act == ARB_ACT_RELU) return fmaxf(z, 0.f);
  return z;
}
__device__ __forceinline__ float act_bwd(float out, float z, int act) {
  if (act == ARB_ACT_TANH) return 1.0f - out * out;
  if (act == ARB_ACT_SIGMOID) return out * (1.0f - out);
  if (act == ARB_ACT_RELU) return z > 0.f ? 1.0f : 0.0f;
  return 1.0f;
}

template <int NV>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) head_fwd_kernel(const float* __restrict__ x,
                                                                      const float* __restrict__ a,
                                                                      const float* __restrict__ b, float eps,
                                                                      const float* __restrict__ w,
                                                                      const float* __restrict__ wb, int has_norm,
                                                                      int act, long long rows, int width,
                                                                      float* __restrict__ score,
                                                                      float* __restrict__ mean_o,
                                                                      float* __restrict__ std_o,
                                                                      const int* __restrict__ rows_dev,
                                                                      const int* __restrict__ rowmap, int n_batches) {
  arb_pdl_wait();
  constexpr int NBMAX = FwdBatches<NV>::value;
  const int NB = NBMAX > 1 ? n_batches : 1;
  const int lane = threadIdx.x & 31;
  // n_batches batches of FWD_RPW rows per warp, the next batch's loads (rows and their row-map entries) issued before
  // the arithmetic of the current one (see ln_fwd_kernel); the device-side row count is loaded with the first batch
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5)) * (FWD_RPW * NB);
  if (base >= rows) return;
  const long long live = rows_dev ? (long long)__ldg(rows_dev) : rows;
  if (NB > 1) { rows = min(rows, live); if (base >= rows) return; }   // (see ln_fwd_kernel)
  RowRegs<NV> r[FWD_RPW], rn[FWD_RPW], ga, gb, gw;
  long long at[FWD_RPW], atn[FWD_RPW];
  auto fetch = [&](long long r0, RowRegs<NV>(&dst)[FWD_RPW], long long(&dat)[FWD_RPW]) {
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) {
      dat[q] = (rowmap && r0 + q < rows) ? (long long)rowmap[r0 + q] : r0 + q;
      if (r0 + q < rows) load_row<NV>(x + (r0 + q) * width, width, lane, dst[q]);
      else {
#pragma unroll
        for (int k = 0; k < NV; ++k) dst[q].v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  fetch(base, r, at);
  load_row<NV>(w, width, lane, gw);
  if (has_norm) {
    load_row<NV>(a, width, lane, ga);
    load_row<NV>(b, width, lane, gb);
  }
  const float bias = wb[0];
  rows = min(rows, live);
#pragma unroll 1
  for (int nb = 0; nb < NB; ++nb) {
    const long long row0 = base + nb * FWD_RPW;
    if (row0 >= rows) break;
    if (NBMAX > 1 && nb + 1 < NB) fetch(row0 + FWD_RPW, rn, atn);
    float mean[FWD_RPW], sd[FWD_RPW];
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) mean[q] = sd[q] = 0.f;
    if (has_norm) {
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) s += r[q].v[k].x + r[q].v[k].y + r[q].v[k].z + r[q].v[k].w;
        mean[q] = s;
      }
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) mean[q] = warp_sum(mean[q]) / float(width);
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) {
        float ss = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          const int c = lane * 4 + 128 * k;
          if (c < width) {
            const float d0 = r[q].v[k].x - mean[q], d1 = r[q].v[k].y - mean[q], d2 = r[q].v[k].z - mean[q],
                        d3 = r[q].v[k].w - mean[q];
            ss += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
          }
        }
        sd[q] = ss;
      }
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) sd[q] = sqrtf(warp_sum(sd[q]) / float(width - 1));
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) {
        const float rinv = 1.0f / (sd[q] + eps), m = mean[q];      // (one reciprocal per row: see ln_fwd_kernel)
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          r[q].v[k].x = ga.v[k].x * (r[q].v[k].x - m) * rinv + gb.v[k].x;
          r[q].v[k].y = ga.v[k].y * (r[q].v[k].y - m) * rinv + gb.v[k].y;
          r[q].v[k].z = ga.v[k].z * (r[q].v[k].z - m) * rinv + gb.v[k].z;
          r[q].v[k].w = ga.v[k].w * (r[q].v[k].w - m) * rinv + gb.v[k].w;
        }
      }
    }
    float dot[FWD_RPW];
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) {
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const int c = lane * 4 + 128 * k;
        if (c < width)
          t += r[q].v[k].x * gw.v[k].x + r[q].v[k].y * gw.v[k].y + r[q].v[k].z * gw.v[k].z + r[q].v[k].w * gw.v[k].w;
      }
      dot[q] = t;
    }
#pragma unroll
    for (int q = 0; q < FWD_RPW; ++q) dot[q] = warp_sum(dot[q]);
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) {
        if (row0 + q >= rows) break;
        // packed rows: the score goes to the item's place in the [B, S] tensor (alignment rows have none)
        if (at[q] >= 0) score[at[q]] = act_fwd(dot[q] + bias, act);
        if (has_norm && mean_o) { mean_o[row0 + q] = mean[q]; std_o[row0 + q] = sd[q]; }
      }
    }
    if (NBMAX > 1) {
#pragma unroll
      for (int q = 0; q < FWD_RPW; ++q) {
        at[q] = atn[q];
#pragma unroll
        for (int k = 0; k < NV; ++k) r[q].v[k] = rn[q].v[k];
      }
    }
  }
}

// head backward: dz = dscore * act'(z);  d xf = dz * w;  grad_w += dz * xf;  grad_wb += dz;  then LayerNorm bwd.
template <int NV>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) head_bwd_kernel(
    const float* __restrict__ dscore, const float* __restrict__ score, const float* __restrict__ x,
    const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ mean_i,
    const float* __restrict__ std_i, float eps, const float* __restrict__ w, const float* __restrict__ wb,
    int has_norm, int act, long long rows, int width, int rows_per_warp, float* __restrict__ dx,
    float* __restrict__ grad_a, float* __restrict__ grad_b, float* __restrict__ grad_w, float* __restrict__ grad_wb,
    float* __restrict__ dx_masked, DropSite site, float* __restrict__ colsum_out, uint16_t* __restrict__ dy16_out,
    const int* __restrict__ rows_dev, const int* __restrict__ rowmap) {
  arb_pdl_wait();
  if (rows_dev) {
    rows = min(rows, (long long)__ldg(rows_dev));
    if ((long long)blockIdx.x * ROWS_PER_BLOCK * rows_per_warp >= rows) return;
  }
  __shared__ float sh[ROWS_PER_BLOCK][128 * NV + 4];
  __shared__ float shb[ROWS_PER_BLOCK];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  RowRegs<NV> ga, gb, gw, acc_a, acc_b, acc_w, acc_c;
  load_row<NV>(w, width, lane, gw);
  if (has_norm) { load_row<NV>(a, width, lane, ga); load_row<NV>(b, width, lane, gb); }
#pragma unroll
  for (int k = 0; k < NV; ++k) acc_a.v[k] = acc_b.v[k] = acc_w.v[k] = acc_c.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  float acc_wb = 0.f;
  const long long first = ((long long)blockIdx.x * ROWS_PER_BLOCK + wid) * rows_per_warp;
  // The warp's rows go in batches of HB: the loads of a whole batch -- rows, row-map entries, statistics, then the
  // scores and their gradients -- are issued before the first row's arithmetic (one row at a time left 12 KB in flight
  // per SM at 73 registers).  Per-row arithmetic and accumulation order are unchanged.
  constexpr int HB = NV <= 2 ? 2 : 1;
#pragma unroll 1
  for (int it0 = 0; it0 < rows_per_warp; it0 += HB) {
    if (first + it0 >= rows) break;
    RowRegs<NV> xb[HB];
    long long atb[HB];
    float meanb[HB], sdb[HB], outb[HB], dsb[HB];
#pragma unroll
    for (int q = 0; q < HB; ++q) {
      const long long row = first + it0 + q;
      const bool ok = it0 + q < rows_per_warp && row < rows;
      atb[q] = -1;
      meanb[q] = 0.f; sdb[q] = 1.f;
      if (ok) {
        load_row<NV>(x + row * width, width, lane, xb[q]);
        // packed rows: score and its gradient sit at the item's place in the [B, S] tensors; alignment rows have neither
        atb[q] = rowmap ? (long long)rowmap[row] : row;
        if (has_norm) { meanb[q] = mean_i[row]; sdb[q] = std_i[row]; }
      }
    }
#pragma unroll
    for (int q = 0; q < HB; ++q) {
      outb[q] = atb[q] >= 0 ? score[atb[q]] : 0.f;
      dsb[q] = atb[q] >= 0 ? dscore[atb[q]] : 0.f;
    }
#pragma unroll
    for (int q = 0; q < HB; ++q) {
    const long long row = first + it0 + q;
    if (it0 + q >= rows_per_warp || row >= rows) break;
    RowRegs<NV>& xr = xb[q];
    RowRegs<NV> g;
    const float out = outb[q];
    float z = 0.f;
    if (act == ARB_ACT_RELU) z = out;   // relu: out > 0 <=> z > 0
    const float dz = atb[q] >= 0 ? dsb[q] * act_bwd(out, z, act) : 0.f;
    if (lane == 0) acc_wb += dz;
    if (!has_norm) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        const float* xv = &xr.v[k].x;
        const float* wv = &gw.v[k].x;
        float* gv = &g.v[k].x;
        float* aw = &acc_w.v[k].x;
#pragma unroll
        for (int e = 0; e < 4; ++e) { gv[e] = dz * wv[e]; aw[e] += dz * xv[e]; }
      }
      store_row<NV>(dx + row * width, width, lane, g);
      if (dx_masked) { apply_drop<NV>(g, row, width, lane, site); store_row<NV>(dx_masked + row * width, width, lane, g); }
      if (dy16_out) store_row_bf16<NV>(dy16_out + row * width, width, lane, g);
      if (colsum_out) {
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          acc_c.v[k].x += g.v[k].x; acc_c.v[k].y += g.v[k].y; acc_c.v[k].z += g.v[k].z; acc_c.v[k].w += g.v[k].w;
        }
      }
      continue;
    }
    const float mean = meanb[q], sd = sdb[q];
    const float r = 1.0f / (sd + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int c = lane * 4 + 128 * k;
      float* xv = &xr.v[k].x;
      const float* wv = &gw.v[k].x;
      const float* av = &ga.v[k].x;
      const float* bv = &gb.v[k].x;
      float* gv = &g.v[k].x;
      float* aa = &acc_a.v[k].x;
      float* ab = &acc_b.v[k].x;
      float* aw = &acc_w.v[k].x;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float cc = (c < width) ? xv[e] - mean : 0.f;
        const float xh = cc * r;
        const float xf = av[e] * xh + bv[e];     // the final norm's output, recomputed (xh = (x - mean) / (std + eps))
        const float dyv = dz * wv[e];          // d loss / d xf
        aw[e] += dz * xf;
        aa[e] += dyv * xh;
        ab[e] += dyv;
        const float dxh = dyv * av[e];
        gv[e] = dxh;
        xv[e] = cc;
        s1 += dxh;
        s2 += dxh * cc;
      }
    }
    s1 = warp_sum(s1);
    s2 = warp_sum(s2);
    const float m1 = s1 / float(width);
    const float coef = (sd > 0.f) ? r * r * s2 / (float(width - 1) * sd) : 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      float* gv = &g.v[k].x;
      const float* xv = &xr.v[k].x;
#pragma unroll
      for (int e = 0; e < 4; ++e) gv[e] = r * (gv[e] - m1) - coef * xv[e];
    }
    store_row<NV>(dx + row * width, width, lane, g);
    if (dx_masked) { apply_drop<NV>(g, row, width, lane, site); store_row<NV>(dx_masked + row * width, width, lane, g); }
    if (dy16_out) store_row_bf16<NV>(dy16_out + row * width, width, lane, g);
    if (colsum_out) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        acc_c.v[k].x += g.v[k].x; acc_c.v[k].y += g.v[k].y; acc_c.v[k].z += g.v[k].z; acc_c.v[k].w += g.v[k].w;
      }
    }
    }
  }
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    if (!has_norm && pass < 2) continue;
    float* dst = pass == 0 ? grad_a : (pass == 1 ? grad_b : (pass == 2 ? grad_w : colsum_out));
    if (!dst) continue;      // (no parameter gradients requested: the gradient outputs are null)
    const RowRegs<NV>& src = pass == 0 ? acc_a : (pass == 1 ? acc_b : (pass == 2 ? acc_w : acc_c));
#pragma unroll
    for (int k = 0; k < NV; ++k) *reinterpret_cast<float4*>(&sh[wid][lane * 4 + 128 * k]) = src.v[k];
    __syncthreads();
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
      float t = 0.f;
#pragma unroll
      for (int ww = 0; ww < ROWS_PER_BLOCK; ++ww) t += sh[ww][c];
      dst[size_t(blockIdx.x) * width + c] = t;      // this block's slot (DetParts)
    }
    __syncthreads();
  }
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
  RowRegs<NV> r, gw;
  load_row<NV>(xf + row * width, width, lane, r);
  for (int j = 0; j < n; ++j) {
    load_row<NV>(w + (long long)j * width, width, lane, gw);
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) dot += r.v[k].x * gw.v[k].x + r.v[k].y * gw.v[k].y + r.v[k].z * gw.v[k].z + r.v[k].w * gw.v[k].w;
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
  RowRegs<NV> acc, gw;
#pragma unroll
  for (int k = 0; k < NV; ++k) acc.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int it = 0; it < rows_per_warp; ++it) {
    const long long row = first + it;
    if (row >= rows) break;
    RowRegs<NV> g;
#pragma unroll
    for (int k = 0; k < NV; ++k) g.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < n; ++j) {
      const float out = score[row * n + j];
      const float dz = dscore[row * n + j] * act_bwd(out, out, act);   // relu: out > 0 <=> z > 0
      load_row<NV>(w + (long long)j * width, width, lane, gw);
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        g.v[k].x += dz * gw.v[k].x; g.v[k].y += dz * gw.v[k].y; g.v[k].z += dz * gw.v[k].z; g.v[k].w += dz * gw.v[k].w;
      }
    }
    store_row<NV>(dxf + row * width, width, lane, g);
    if (dx_masked) { apply_drop<NV>(g, row, width, lane, site); store_row<NV>(dx_masked + row * width, width, lane, g); }
    if (colsum_out) {
#pragma unroll
      for (int k = 0; k < NV; ++k) {
        acc.v[k].x += g.v[k].x; acc.v[k].y += g.v[k].y; acc.v[k].z += g.v[k].z; acc.v[k].w += g.v[k].w;
      }
    }
  }
  // block-level column reductions: pass -1 = colsum_out, pass j = grad_w row j
  for (int j = colsum_out ? -1 : 0; j < (grad_w ? n : 0); ++j) {
    float acc_b = 0.f;
    if (j >= 0) {
#pragma unroll
      for (int k = 0; k < NV; ++k) acc.v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int it = 0; it < rows_per_warp; ++it) {
        const long long row = first + it;
        if (row >= rows) break;
        const float out = score[row * n + j];
        const float dz = dscore[row * n + j] * act_bwd(out, out, act);
        load_row<NV>(xf + row * width, width, lane, gw);
        acc_b += dz;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          acc.v[k].x += dz * gw.v[k].x; acc.v[k].y += dz * gw.v[k].y; acc.v[k].z += dz * gw.v[k].z; acc.v[k].w += dz * gw.v[k].w;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < NV; ++k) *reinterpret_cast<float4*>(&sh[wid][lane * 4 + 128 * k]) = acc.v[k];
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
__global__ void __launch_bounds__(256) pos_bwd_kernel(const float* __restrict__ dx, const long long* __restrict__ indices,
                                                      const uint8_t* __restrict__ mask, float* __restrict__ dpe,
                                                      int pe_rows, long long rows, int width) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int pad = pe_rows - 1;
  long long idx = mask[row] ? pad : indices[row];
  if (idx > pad) idx = pad;
  if (idx < 0) idx += pe_rows;
  if (idx < 0 || idx == pad) return;
  for (int c = lane; c < width; c += 32) atomicAdd(dpe + idx * width + c, dx[row * width + c]);
}

// ------------------------------------------------------------------------------------------------ FC-block activations
// FCModel applies dropout(activation(linear(x))) per layer (model.py:41-43).  ReLU / identity run inside the GEMM
// epilogue; the kernels below serve the other activations and the backward of every activation under dropout.
// Element index of the dropout counter = row * width + column (the same as the GEMM epilogue's).
__global__ void __launch_bounds__(256) act_fwd_kernel(float* __restrict__ h, long long n4, int act, DropSite site,
                                                      const int* __restrict__ rows_dev, int width4) {
  if (rows_dev) n4 = min(n4, (long long)__ldg(rows_dev) * width4);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<float4*>(h)[i];
    float* e = &v.x;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float y = act_fwd(e[j], act);
      e[j] = drop_keep((unsigned long long)i * 4 + j, site.seed, site.thresh) ? y * site.scale : 0.0f;
    }
    reinterpret_cast<float4*>(h)[i] = v;
  }
}

// dz = mul * dh * m/(1-p) * act'(y)  with y = act(z) recovered from the stored h = m y/(1-p); colsum_out += column sums
// of dz (the bias gradient of the linear that produced z).  dz may alias dh.
__global__ void __launch_bounds__(256) act_bwd_kernel(const float* dh, const float* __restrict__ h, float* dz,
                                                      long long rows, int width, int act, DropSite site, float mul,
                                                      int tx_n, int rows_per_block, float* __restrict__ colsum_out,
                                                      const int* __restrict__ rows_dev) {
  extern __shared__ float sh_cols[];     // [ty_n][width]: one row of column partials per row group
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
        const bool keep = drop_keep((unsigned long long)at + j, site.seed, site.thresh);
        const float y = he[j] * inv_scale;
        ge[j] = keep ? ge[j] * mul * site.scale * act_bwd(y, y, act) : 0.0f;   // ReLU: y > 0 <=> z > 0
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

#define ARB_DISPATCH_NV(width, CALL)                                  \
  switch (nv_for(width)) {                                            \
    case 1: { constexpr int NV = 1; CALL; } break;                    \
    case 2: { constexpr int NV = 2; CALL; } break;                    \
    case 3: case 4: { constexpr int NV = 4; CALL; } break;            \
    case 5: case 6: case 7: case 8: { constexpr int NV = 8; CALL; } break; \
    default: arb_set_error("row kernels support widths up to 1024"); return ARB_E_UNSUPPORTED; \
  }

// rows per warp of the backward row kernels (LayerNorm, head): more rows per warp = fewer block-level reductions and
// block slots of the gain / bias gradients per byte moved.  ARB_ROWS_PER_WARP overrides (measurement knob).
static int bwd_rows_per_warp() {
  static int v = 0;
  if (!v) {
    const char* e = getenv("ARB_ROWS_PER_WARP");
    v = e ? std::max(1, std::min(256, atoi(e))) : 8;
  }
  return v;
}


// ------------------------------------------------------------------------------------------------ rows of 128 / 256
// "R" layout of the row kernels for the common model widths W = 128 (LPR = 8 lanes per row, 4 rows per warp step)
// and W = 256 (LPR = 16, 2 rows per step): a lane owns 16 elements of ONE row -- float4 j at column
// ((lane % LPR) + LPR * j) * 4, so that the LPR lanes of a row read LPR * 16 contiguous bytes per instruction --
// and a row reduction is log2(LPR) shuffle steps that serve all rows of the step at once (one row per warp needs five
// steps per row and reduction: ncu put ln_fwd at 75 % issue-active with shuffles and their adds a third of it).
// Same arithmetic per element as the generic kernels; the summation trees differ.
template <int LPR>
__device__ __forceinline__ int r_col(int lane, int j) { return ((lane % LPR) + LPR * j) * 4; }
template <int LPR>
__device__ __forceinline__ float r_sum(float v) {
#pragma unroll
  for (int off = 1; off < LPR; off <<= 1) v += __shfl_xor_sync(FULL, v, off);
  return v;
}
template <int LPR>
__device__ __forceinline__ void r_load(const float* __restrict__ row, int lane, float4 (&v)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = *reinterpret_cast<const float4*>(row + r_col<LPR>(lane, j));
}
template <int LPR>
__device__ __forceinline__ void r_load_bf16(const uint16_t* __restrict__ row, int lane, float4 (&v)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint2 u = *reinterpret_cast<const uint2*>(row + r_col<LPR>(lane, j));
    v[j] = make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xffff0000u));
  }
}
template <int LPR>
__device__ __forceinline__ void r_store(float* __restrict__ row, int lane, const float4 (&v)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(row + r_col<LPR>(lane, j)) = v[j];
}
template <int LPR>
__device__ __forceinline__ void r_store_bf16(uint16_t* __restrict__ row, int lane, const float4 (&v)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j)
    *reinterpret_cast<uint2*>(row + r_col<LPR>(lane, j)) = make_uint2(pack_bf16x2(v[j].x, v[j].y), pack_bf16x2(v[j].z, v[j].w));
}
__device__ __forceinline__ void r_zero(float4 (&v)[4]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
}
template <int LPR>
__device__ __forceinline__ void r_drop(float4 (&v)[4], long long row, int lane, const DropSite& site) {
  constexpr int W = 16 * LPR;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float* e = &v[j].x;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const unsigned long long idx = (unsigned long long)row * W + (r_col<LPR>(lane, j) + t);
      e[t] = drop_keep(idx, site.seed, site.thresh) ? e[t] * site.scale : 0.0f;
    }
  }
}
// sum the per-column accumulators of the warp's row groups, then over the block's warps, then into the block's slot of
// `dst` (DetParts)
template <int LPR>
__device__ __forceinline__ void r_reduce_columns(float4 (&acc)[4], float (*sh)[16 * LPR + 4], int lane, int wid,
                                                 float* __restrict__ dst) {
  constexpr int W = 16 * LPR;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float* e = &acc[j].x;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
#pragma unroll
      for (int off = LPR; off < 32; off <<= 1) e[t] += __shfl_xor_sync(FULL, e[t], off);
    }
  }
  if (lane < LPR) {
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<float4*>(&sh[wid][r_col<LPR>(lane, j)]) = acc[j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < W; c += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < ROWS_PER_BLOCK; ++w) t += sh[w][c];
    dst[size_t(blockIdx.x) * W + c] = t;            // this block's slot (DetParts)
  }
  __syncthreads();
}

template <int LPR, bool MAP>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) ln_fwd_r_kernel(const float* __restrict__ x,
                                                                      const float* __restrict__ a,
                                                                      const float* __restrict__ b, float eps,
                                                                      long long rows, float* __restrict__ y,
                                                                      float* __restrict__ mean_o,
                                                                      float* __restrict__ std_o, int torch_mode,
                                                                      uint16_t* __restrict__ y16,
                                                                      const int* __restrict__ rows_dev, int steps,
                                                                      const int* __restrict__ rowmap_out) {
  arb_pdl_wait();
  constexpr int RW = 32 / LPR, W = 16 * LPR;
  const int lane = threadIdx.x & 31, rg = lane / LPR;
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5)) * (RW * steps);
  if (base >= rows) return;
  if (rows_dev) { rows = min(rows, (long long)__ldg(rows_dev)); if (base >= rows) return; }
  float4 ga[4], gb[4], cur[4], nxt[4];
  r_load<LPR>(a, lane, ga);
  r_load<LPR>(b, lane, gb);
  if (base + rg < rows) r_load<LPR>(x + (base + rg) * W, lane, cur); else r_zero(cur);
#pragma unroll 1
  for (int s = 0; s < steps; ++s) {
    if (base + (long long)s * RW >= rows) break;
    const long long row = base + (long long)s * RW + rg;
    if (s + 1 < steps) { if (row + RW < rows) r_load<LPR>(x + (row + RW) * W, lane, nxt); else r_zero(nxt); }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) sum += cur[j].x + cur[j].y + cur[j].z + cur[j].w;
    const float m = r_sum<LPR>(sum) / float(W);
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float d0 = cur[j].x - m, d1 = cur[j].y - m, d2 = cur[j].z - m, d3 = cur[j].w - m;
      ss += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
    }
    ss = r_sum<LPR>(ss);
    // (torch_mode and the reciprocal: see ln_fwd_kernel)
    const float sdq = torch_mode ? sqrtf(ss / float(W) + eps) : sqrtf(ss / float(W - 1));
    const float rinv = 1.0f / (torch_mode ? sdq : sdq + eps);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      cur[j].x = ga[j].x * (cur[j].x - m) * rinv + gb[j].x;
      cur[j].y = ga[j].y * (cur[j].y - m) * rinv + gb[j].y;
      cur[j].z = ga[j].z * (cur[j].z - m) * rinv + gb[j].z;
      cur[j].w = ga[j].w * (cur[j].w - m) * rinv + gb[j].w;
    }
    if (row < rows) {
      if (y16) r_store_bf16<LPR>(y16 + row * W, lane, cur);
      else {   // (rowmap_out: see ln_fwd_kernel)
        const long long yr = MAP ? (long long)rowmap_out[row] : row;
        if (!MAP || yr >= 0) r_store<LPR>(y + yr * W, lane, cur);
      }
      if (lane % LPR == 0) { mean_o[row] = m; std_o[row] = sdq; }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) cur[j] = nxt[j];
  }
}

template <int LPR, bool MAP>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32, 2) ln_bwd_r_kernel(
    const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ a,
    const float* __restrict__ mean_i, const float* __restrict__ std_i, float eps, const float* __restrict__ dres,
    long long rows, int steps, float* __restrict__ dx, float* __restrict__ grad_a, float* __restrict__ grad_b,
    float* __restrict__ dx_masked, DropSite site, float* __restrict__ colsum_out, int torch_mode,
    const uint16_t* __restrict__ dy16_in, uint16_t* __restrict__ dy16_out, const int* __restrict__ rows_dev,
    const int* __restrict__ rowmap_in) {
  arb_pdl_wait();
  constexpr int RW = 32 / LPR, W = 16 * LPR;
  if (rows_dev) rows = min(rows, (long long)__ldg(rows_dev));
  if ((long long)blockIdx.x * ROWS_PER_BLOCK * RW * steps >= rows) return;      // whole block beyond the live rows
  __shared__ float sh[ROWS_PER_BLOCK][W + 4];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, rg = lane / LPR;
  float4 ga[4], acc_a[4], acc_b[4], acc_c[4];
  r_load<LPR>(a, lane, ga);
  r_zero(acc_a); r_zero(acc_b); r_zero(acc_c);
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + wid) * (RW * steps);
#pragma unroll 1
  for (int s = 0; s < steps; ++s) {
    if (base + (long long)s * RW >= rows) break;
    const long long row = base + (long long)s * RW + rg;
    const bool ok = row < rows;
    float4 g[4], xr[4], res[4];
    float mean = 0.f, sd = 1.f;
    r_zero(g); r_zero(xr); r_zero(res);
    if (ok) {
      if (dy16_in) r_load_bf16<LPR>(dy16_in + row * W, lane, g);
      else if (MAP) { const long long src = rowmap_in[row]; if (src >= 0) r_load<LPR>(dy + src * W, lane, g); }
      else r_load<LPR>(dy + row * W, lane, g);
      r_load<LPR>(x + row * W, lane, xr);
      if (dres) r_load<LPR>(dres + row * W, lane, res);
      mean = mean_i[row]; sd = std_i[row];
    }
    const float r = 1.0f / (sd + eps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float* gv = &g[j].x;
      float* xv = &xr[j].x;
      const float* av = &ga[j].x;
      float* aa = &acc_a[j].x;
      float* ab = &acc_b[j].x;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float cc = ok ? xv[t] - mean : 0.f;
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
    const float m1 = s1 / float(W);
    const float coef = torch_mode ? r * r * r * s2 / float(W) : ((sd > 0.f) ? r * r * s2 / (float(W - 1) * sd) : 0.f);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float* gv = &g[j].x;
      const float* xv = &xr[j].x;
      const float* rv = &res[j].x;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        float o = r * (gv[t] - m1) - coef * xv[t];
        if (dres) o += rv[t];
        gv[t] = o;
      }
    }
    if (ok) {
      r_store<LPR>(dx + row * W, lane, g);
      if (dx_masked) {   // the same gradient through the dropout of the sublayer below (mask regenerated)
        r_drop<LPR>(g, row, lane, site);
        r_store<LPR>(dx_masked + row * W, lane, g);
      }
      if (dy16_out) r_store_bf16<LPR>(dy16_out + row * W, lane, g);
      if (colsum_out) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc_c[j].x += g[j].x; acc_c[j].y += g[j].y; acc_c[j].z += g[j].z; acc_c[j].w += g[j].w; }
      }
    }
  }
  if (grad_a) r_reduce_columns<LPR>(acc_a, sh, lane, wid, grad_a);
  if (grad_b) r_reduce_columns<LPR>(acc_b, sh, lane, wid, grad_b);
  if (colsum_out) r_reduce_columns<LPR>(acc_c, sh, lane, wid, colsum_out);
}

template <int LPR>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32) head_fwd_r_kernel(
    const float* __restrict__ x, const float* __restrict__ a, const float* __restrict__ b, float eps,
    const float* __restrict__ w, const float* __restrict__ wb, int has_norm, int act, long long rows,
    float* __restrict__ score, float* __restrict__ mean_o, float* __restrict__ std_o,
    const int* __restrict__ rows_dev, const int* __restrict__ rowmap, int steps) {
  arb_pdl_wait();
  constexpr int RW = 32 / LPR, W = 16 * LPR;
  const int lane = threadIdx.x & 31, rg = lane / LPR;
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + (threadIdx.x >> 5)) * (RW * steps);
  if (base >= rows) return;
  if (rows_dev) { rows = min(rows, (long long)__ldg(rows_dev)); if (base >= rows) return; }
  float4 ga[4], gb[4], gw[4], cur[4], nxt[4];
  r_load<LPR>(w, lane, gw);
  if (has_norm) { r_load<LPR>(a, lane, ga); r_load<LPR>(b, lane, gb); } else { r_zero(ga); r_zero(gb); }
  const float bias = wb[0];
  long long at = -1, at_n = -1;
  if (base + rg < rows) {
    r_load<LPR>(x + (base + rg) * W, lane, cur);
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
        r_load<LPR>(x + (row + RW) * W, lane, nxt);
        at_n = rowmap ? (long long)rowmap[row + RW] : row + RW;
      } else {
        r_zero(nxt);
      }
    }
    float m = 0.f, sdv = 0.f;
    if (has_norm) {
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) sum += cur[j].x + cur[j].y + cur[j].z + cur[j].w;
      m = r_sum<LPR>(sum) / float(W);
      float ss = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float d0 = cur[j].x - m, d1 = cur[j].y - m, d2 = cur[j].z - m, d3 = cur[j].w - m;
        ss += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
      }
      sdv = sqrtf(r_sum<LPR>(ss) / float(W - 1));
      const float rinv = 1.0f / (sdv + eps);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        cur[j].x = ga[j].x * (cur[j].x - m) * rinv + gb[j].x;
        cur[j].y = ga[j].y * (cur[j].y - m) * rinv + gb[j].y;
        cur[j].z = ga[j].z * (cur[j].z - m) * rinv + gb[j].z;
        cur[j].w = ga[j].w * (cur[j].w - m) * rinv + gb[j].w;
      }
    }
    float dot = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) dot += cur[j].x * gw[j].x + cur[j].y * gw[j].y + cur[j].z * gw[j].z + cur[j].w * gw[j].w;
    dot = r_sum<LPR>(dot);
    if (row < rows && lane % LPR == 0) {
      // packed rows: the score goes to the item's place in the [B, S] tensor (alignment rows have none)
      if (at >= 0) score[at] = act_fwd(dot + bias, act);
      if (has_norm && mean_o) { mean_o[row] = m; std_o[row] = sdv; }
    }
    at = at_n;
#pragma unroll
    for (int j = 0; j < 4; ++j) cur[j] = nxt[j];
  }
}

template <int LPR>
__global__ void __launch_bounds__(ROWS_PER_BLOCK * 32, 2) head_bwd_r_kernel(
    const float* __restrict__ dscore, const float* __restrict__ score, const float* __restrict__ x,
    const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ mean_i,
    const float* __restrict__ std_i, float eps, const float* __restrict__ w, int has_norm, int act, long long rows,
    int steps, float* __restrict__ dx, float* __restrict__ grad_a, float* __restrict__ grad_b,
    float* __restrict__ grad_w, float* __restrict__ grad_wb, float* __restrict__ dx_masked, DropSite site,
    float* __restrict__ colsum_out, uint16_t* __restrict__ dy16_out, const int* __restrict__ rows_dev,
    const int* __restrict__ rowmap) {
  arb_pdl_wait();
  constexpr int RW = 32 / LPR, W = 16 * LPR;
  if (rows_dev) rows = min(rows, (long long)__ldg(rows_dev));
  if ((long long)blockIdx.x * ROWS_PER_BLOCK * RW * steps >= rows) return;
  __shared__ float sh[ROWS_PER_BLOCK][W + 4];
  __shared__ float shb[ROWS_PER_BLOCK];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, rg = lane / LPR;
  float4 ga[4], gb[4], gw[4], acc_a[4], acc_b[4], acc_w[4], acc_c[4];
  r_load<LPR>(w, lane, gw);
  if (has_norm) { r_load<LPR>(a, lane, ga); r_load<LPR>(b, lane, gb); } else { r_zero(ga); r_zero(gb); }
  r_zero(acc_a); r_zero(acc_b); r_zero(acc_w); r_zero(acc_c);
  float acc_wb = 0.f;
  const long long base = ((long long)blockIdx.x * ROWS_PER_BLOCK + wid) * (RW * steps);
#pragma unroll 1
  for (int s = 0; s < steps; ++s) {
    if (base + (long long)s * RW >= rows) break;
    const long long row = base + (long long)s * RW + rg;
    const bool ok = row < rows;
    float4 xr[4], g[4];
    r_zero(xr);
    long long at = -1;
    float mean = 0.f, sd = 1.f;
    if (ok) {
      r_load<LPR>(x + row * W, lane, xr);
      // packed rows: score and its gradient sit at the item's place in the [B, S] tensors; alignment rows have neither
      at = rowmap ? (long long)rowmap[row] : row;
      if (has_norm) { mean = mean_i[row]; sd = std_i[row]; }
    }
    const float out = at >= 0 ? score[at] : 0.f;
    float z = 0.f;
    if (act == ARB_ACT_RELU) z = out;   // relu: out > 0 <=> z > 0
    const float dz = at >= 0 ? dscore[at] * act_bwd(out, z, act) : 0.f;
    if (lane % LPR == 0) acc_wb += dz;
    if (!has_norm) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
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
      for (int j = 0; j < 4; ++j) {
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
          const float cc = ok ? xv[t] - mean : 0.f;
          const float xh = cc * r;
          const float xf = av[t] * xh + bv[t];     // the final norm's output, recomputed
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
      const float m1 = s1 / float(W);
      const float coef = (sd > 0.f) ? r * r * s2 / (float(W - 1) * sd) : 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float* gv = &g[j].x;
        const float* xv = &xr[j].x;
#pragma unroll
        for (int t = 0; t < 4; ++t) gv[t] = r * (gv[t] - m1) - coef * xv[t];
      }
    }
    if (ok) {
      r_store<LPR>(dx + row * W, lane, g);
      if (dx_masked) { r_drop<LPR>(g, row, lane, site); r_store<LPR>(dx_masked + row * W, lane, g); }
      if (dy16_out) r_store_bf16<LPR>(dy16_out + row * W, lane, g);
      if (colsum_out) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc_c[j].x += g[j].x; acc_c[j].y += g[j].y; acc_c[j].z += g[j].z; acc_c[j].w += g[j].w; }
      }
    }
  }
  if (has_norm && grad_a) r_reduce_columns<LPR>(acc_a, sh, lane, wid, grad_a);
  if (has_norm && grad_b) r_reduce_columns<LPR>(acc_b, sh, lane, wid, grad_b);
  if (grad_w) r_reduce_columns<LPR>(acc_w, sh, lane, wid, grad_w);
  if (colsum_out) r_reduce_columns<LPR>(acc_c, sh, lane, wid, colsum_out);
  acc_wb = warp_sum(acc_wb);
  if (lane == 0) shb[wid] = acc_wb;
  __syncthreads();
  if (threadIdx.x == 0 && grad_wb) {
    float t = 0.f;
    for (int ww = 0; ww < ROWS_PER_BLOCK; ++ww) t += shb[ww];
    grad_wb[blockIdx.x] = t;                        // this block's slot (DetParts)
  }
}

// Which row kernels use the layout above for W = 128 / 256 (else the generic one-row-per-warp kernels): bit 0 ln_fwd,
// bit 1 ln_bwd, bit 2 head_fwd, bit 3 head_bwd.  ARB_ROW_LAYOUT overrides (measurement knob).
enum { R_LN_FWD = 1, R_LN_BWD = 2, R_HEAD_FWD = 4, R_HEAD_BWD = 8 };
static int row_layout_r() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("ARB_ROW_LAYOUT"); v = e ? atoi(e) : ARB_DEFAULT_ROW_LAYOUT; }
  return v;
}
static inline int r_lpr(int width, int which) {
  return ((row_layout_r() & which) && (width == 128 || width == 256)) ? width / 16 : 0;
}
// steps per warp of the forward R kernels: 4 (16 / 8 rows per warp) for large launches, 1 for small ones
static inline int r_fwd_steps(long long rows) { return rows >= (1 << 17) ? 4 : 1; }
// rows per warp of the backward R kernels (a multiple of 4): the per-warp column reduction at the end costs 2 shuffles
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
               const int* rowmap_out) {
  if (rowmap_out && y16) { arb_set_error("ln_forward: a row-mapped output is fp32 only"); return ARB_E_INVALID_ARG; }
  if (width % 4) { arb_set_error("LayerNorm width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * ((y16 ? 6.0 : 8.0) * width + 8), st);
  if (const int lpr = r_lpr(width, R_LN_FWD)) {      // W = 128 / 256: several rows per warp step (see ln_fwd_r_kernel)
    const int steps = r_fwd_steps(rows), per_block = ROWS_PER_BLOCK * (32 / lpr) * steps;
    const unsigned nblk = unsigned((rows + per_block - 1) / per_block);
    if (lpr == 8) return launch(rowmap_out ? ln_fwd_r_kernel<8, true> : ln_fwd_r_kernel<8, false>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps, rows, y, mean, sd, torch_mode, static_cast<uint16_t*>(y16), rows_dev, steps, rowmap_out);
    return launch(rowmap_out ? ln_fwd_r_kernel<16, true> : ln_fwd_r_kernel<16, false>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps, rows, y, mean, sd, torch_mode, static_cast<uint16_t*>(y16), rows_dev, steps, rowmap_out);
  }
  const int nb = fwd_batches_for(width, rows);
  const int per_block = ROWS_PER_BLOCK * FWD_RPW * nb;
  const unsigned blocks = unsigned((rows + per_block - 1) / per_block);
  int rc;
  ARB_DISPATCH_NV(width, (rc = launch(rowmap_out ? ln_fwd_kernel<NV, true> : ln_fwd_kernel<NV, false>, dim3(blocks), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps, rows, width, y, mean, sd, torch_mode, static_cast<uint16_t*>(y16), rows_dev, nb, rowmap_out)));
  return rc;
}

int ln_backward(const float* dy, const float* x, const float* a, const float* mean, const float* sd, float eps,
                const float* dres, long long rows, int width, float* dx, float* grad_a, float* grad_b,
                cudaStream_t st, float* dx_masked, DropSite site, float* colsum_out, int torch_mode,
                const void* dy16_in, void* dy16_out, const int* rows_dev, const int* rowmap_in) {
  if (rowmap_in && dy16_in) { arb_set_error("ln_backward: a row-mapped gradient is fp32 only"); return ARB_E_INVALID_ARG; }
  if (site.thresh == 0 && site.scale == 1.0f) dx_masked = nullptr;
  if (dy16_out && dx_masked == nullptr && (site.thresh != 0 || site.scale != 1.0f)) {
    arb_set_error("ln_backward: a masked bf16 copy needs the masked fp32 buffer too"); return ARB_E_INVALID_ARG;
  }   // thresh 0 with a scale = pure rescale (positional encoding)
  const int rpw = bwd_rows_per_warp();
  const unsigned blocks = unsigned((rows + ROWS_PER_BLOCK * rpw - 1) / (ROWS_PER_BLOCK * rpw));
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * ((dres ? 16.0 : 12.0) * width + 8), st);
  const int lpr = r_lpr(width, R_LN_BWD);
  const int steps = lpr ? r_bwd_rows_per_warp(rows) / (32 / lpr) : 0;
  const unsigned nblk = lpr ? unsigned((rows + ROWS_PER_BLOCK * (32 / lpr) * steps - 1) / (ROWS_PER_BLOCK * (32 / lpr) * steps)) : blocks;
  DetParts dp;
  dp.add(grad_a, nblk, 1, width, width); dp.add(grad_b, nblk, 1, width, width); dp.add(colsum_out, nblk, 1, width, width);
  int rc = dp.begin(st);
  if (rc) return rc;
  if (lpr) {
    if (lpr == 8) rc = launch(rowmap_in ? ln_bwd_r_kernel<8, true> : ln_bwd_r_kernel<8, false>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dy, x, a, mean, sd, eps, dres, rows, steps, dx, grad_a, grad_b, dx_masked, site, colsum_out, torch_mode, static_cast<const uint16_t*>(dy16_in), static_cast<uint16_t*>(dy16_out), rows_dev, rowmap_in);
    else rc = launch(rowmap_in ? ln_bwd_r_kernel<16, true> : ln_bwd_r_kernel<16, false>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dy, x, a, mean, sd, eps, dres, rows, steps, dx, grad_a, grad_b, dx_masked, site, colsum_out, torch_mode, static_cast<const uint16_t*>(dy16_in), static_cast<uint16_t*>(dy16_out), rows_dev, rowmap_in);
  } else {
    ARB_DISPATCH_NV(width, (rc = launch(rowmap_in ? ln_bwd_kernel<NV, true> : ln_bwd_kernel<NV, false>, dim3(blocks), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dy, x, a, mean, sd, eps, dres, rows, width, rpw, dx, grad_a, grad_b, dx_masked, site, colsum_out, torch_mode, static_cast<const uint16_t*>(dy16_in), static_cast<uint16_t*>(dy16_out), rows_dev, rowmap_in)));
  }
  if (rc) return rc;
  return dp.finish(st);
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
  ProfScope ps(ARB_PROF_SCORER_SIMT, double(rows) * 8.0 * width, st);
  return launch(pos_bwd_kernel, dim3(unsigned((rows + 7) / 8)), dim3(256), 0, st, /*pdl=*/false, dx, indices, mask, dpe,
                pe_rows, rows, width);
}

int act_forward(float* h, long long rows, int width, int act, DropSite site, cudaStream_t st, const int* rows_dev) {
  if (width % 4) { arb_set_error("activation: width must be a multiple of 4"); return ARB_E_UNSUPPORTED; }
  const long long n4 = rows * width / 4;
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * 8.0 * width, st);
  const unsigned blocks = unsigned(std::min<long long>((n4 + 255) / 256, 132 * 16));
  return launch(act_fwd_kernel, dim3(blocks), dim3(256), 0, st, /*pdl=*/false, h, n4, act, site, rows_dev, width / 4);
}

int act_backward(const float* dh, const float* h, float* dz, long long rows, int width, int act, DropSite site, float mul,
                 float* colsum_out, cudaStream_t st, const int* rows_dev) {
  if (width % 4 || width > 8192) { arb_set_error("activation: width must be a multiple of 4 and <= 8192"); return ARB_E_UNSUPPORTED; }
  int tx_n = 1;
  while (tx_n < width / 4 && tx_n < 256) tx_n *= 2;
  const int rpb = 64 * (256 / tx_n);
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * 12.0 * width, st);
  const unsigned blocks = unsigned((rows + rpb - 1) / rpb);
  DetParts dp;
  dp.add(colsum_out, blocks, 1, width, width);
  if (int rc = dp.begin(st)) return rc;
  if (int rc = launch(act_bwd_kernel, dim3(blocks), dim3(256), size_t(256 / tx_n) * width * 4, st, /*pdl=*/false, dh, h,
                      dz, rows, width, act, site, mul, tx_n, rpb, colsum_out, rows_dev))
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
  if (const int lpr = r_lpr(width, R_HEAD_FWD)) {
    const int steps = r_fwd_steps(rows), per_block = ROWS_PER_BLOCK * (32 / lpr) * steps;
    const unsigned nblk = unsigned((rows + per_block - 1) / per_block);
    if (lpr == 8) return launch(head_fwd_r_kernel<8>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps, w, wb, has_norm, act, rows, score, mean, sd, rows_dev, rowmap, steps);
    return launch(head_fwd_r_kernel<16>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps, w, wb, has_norm, act, rows, score, mean, sd, rows_dev, rowmap, steps);
  }
  const int nb = fwd_batches_for(width, rows);
  const int per_block = ROWS_PER_BLOCK * FWD_RPW * nb;
  const unsigned blocks = unsigned((rows + per_block - 1) / per_block);
  int rc;
  ARB_DISPATCH_NV(width, (rc = launch(head_fwd_kernel<NV>, dim3(blocks), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, x, a, b, eps, w, wb, has_norm, act, rows, width, score, mean, sd, rows_dev, rowmap, nb)));
  return rc;
}

int head_backward(const float* dscore, const float* score, const float* x, const float* a, const float* b,
                  const float* mean, const float* sd, float eps, const float* w, const float* wb, int has_norm,
                  int act, long long rows, int width, float* dx, float* grad_a, float* grad_b, float* grad_w,
                  float* grad_wb, cudaStream_t st, float* dx_masked, DropSite site, float* colsum_out, void* dy16_out,
                  const int* rows_dev, const int* rowmap) {
  if (site.thresh == 0) dx_masked = nullptr;
  const int rpw = bwd_rows_per_warp();
  const unsigned blocks = unsigned((rows + ROWS_PER_BLOCK * rpw - 1) / (ROWS_PER_BLOCK * rpw));
  ProfScope ps(ARB_PROF_SCORER_SIMT, live_rows(rows, rows_dev) * (8.0 * width + 16), st);
  const int lpr = r_lpr(width, R_HEAD_BWD);
  const int steps = lpr ? r_bwd_rows_per_warp(rows) / (32 / lpr) : 0;
  const unsigned nblk = lpr ? unsigned((rows + ROWS_PER_BLOCK * (32 / lpr) * steps - 1) / (ROWS_PER_BLOCK * (32 / lpr) * steps)) : blocks;
  DetParts dp;
  if (has_norm) { dp.add(grad_a, nblk, 1, width, width); dp.add(grad_b, nblk, 1, width, width); }
  dp.add(grad_w, nblk, 1, width, width); dp.add(colsum_out, nblk, 1, width, width); dp.add(grad_wb, nblk, 1, 1, 1);
  int rc = dp.begin(st);
  if (rc) return rc;
  if (lpr) {
    if (lpr == 8) rc = launch(head_bwd_r_kernel<8>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dscore, score, x, a, b, mean, sd, eps, w, has_norm, act, rows, steps, dx, grad_a, grad_b, grad_w, grad_wb, dx_masked, site, colsum_out, static_cast<uint16_t*>(dy16_out), rows_dev, rowmap);
    else rc = launch(head_bwd_r_kernel<16>, dim3(nblk), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dscore, score, x, a, b, mean, sd, eps, w, has_norm, act, rows, steps, dx, grad_a, grad_b, grad_w, grad_wb, dx_masked, site, colsum_out, static_cast<uint16_t*>(dy16_out), rows_dev, rowmap);
  } else {
    ARB_DISPATCH_NV(width, (rc = launch(head_bwd_kernel<NV>, dim3(blocks), dim3(ROWS_PER_BLOCK * 32), 0, st, /*pdl=*/true, dscore, score, x, a, b, mean, sd, eps, w, wb, has_norm, act, rows, width, rpw, dx, grad_a, grad_b, grad_w, grad_wb, dx_masked, site, colsum_out, static_cast<uint16_t*>(dy16_out), rows_dev, rowmap)));
  }
  if (rc) return rc;
  return dp.finish(st);
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
  const int rpw = bwd_rows_per_warp();
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
