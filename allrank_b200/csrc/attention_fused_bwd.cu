// Fused self-attention backward for slates of up to 256 items and head width <= 32.
//
// Reference: autograd of attention() allrank/models/transformer.py:137-156.  Given d ctx it produces dQ, dK, dV
// without ever materialising the S x S probabilities in HBM: they are recomputed from Q, K and the row statistics
// (max, sum) the fused forward kernel saved.  See attn_bwd_kernel for the organisation.
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "attention_fused.h"
#include "block_utils.cuh"
#include "common.h"
#include "defaults.h"
#include "sm90_ptx.cuh"

namespace arb {

constexpr int BWD_THREADS = 256;          // 8 warps x 16 rows of a 128-row tile
constexpr int TILE_BYTES = 128 * 128;     // one [128 rows][128 B] operand tile

__device__ __forceinline__ float ex2_approx_b(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float round_tf32_b(float x) {
  // round-to-nearest (ties away) to tf32 as "+ half an ulp of the 10-bit mantissa, then let the tensor core ignore the
  // low 13 bits" -- one integer add instead of cvt.rna.tf32.f32.
  // Same result as cvt.rna for every finite value (probabilities and their gradients are finite).
  return __uint_as_float(__float_as_uint(x) + 0x1000u);
}

// delta[b,h,q] = sum_e dO[b,q,h,e] * O[b,q,h,e]: one warp per row of the [B*S, d_model] activations, 128-bit loads,
// segmented shuffle reduction over the dk/4 lanes that share a head (dk in {16, 32}: 4 or 8 lanes per head).
constexpr int DELTA_RPW = 4;     // rows per warp of the delta kernel
__global__ void __launch_bounds__(256) attn_delta_kernel(const float* __restrict__ d_o, const float* __restrict__ o,
                                                         long long pitch, int B, int S, int h, int dk,
                                                         float* __restrict__ delta, int o_bf16,
                                                         const int* __restrict__ rows_dev,
                                                         const int* __restrict__ rowmap, long long rows_cap) {
  arb_pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row0 = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * DELTA_RPW;
  // packed rows: the activations are indexed by the packed row, delta by the item (rows without an item are skipped);
  // rows at or beyond the device-side row count are not touched
  const long long rows = rows_dev ? min(rows_cap, (long long)__ldg(rows_dev)) : rows_cap;
  if (row0 >= rows) return;
  const int width = h * dk, lanes_per_head = dk >> 2;
  // a warp owns DELTA_RPW consecutive rows and issues all their loads (row-map entries included) up front
  long long item[DELTA_RPW];
#pragma unroll
  for (int q = 0; q < DELTA_RPW; ++q) item[q] = (row0 + q < rows) ? (rowmap ? (long long)rowmap[row0 + q] : row0 + q) : -1;
  for (int c0 = 0; c0 < width; c0 += 128) {
    const int c = c0 + lane * 4;
    float4 a[DELTA_RPW], bq[DELTA_RPW];
#pragma unroll
    for (int q = 0; q < DELTA_RPW; ++q) {
      a[q] = bq[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < width && row0 + q < rows) {
        const long long row = row0 + q;
        a[q] = *reinterpret_cast<const float4*>(d_o + row * pitch + c);
        if (o_bf16) {       // bf16 mode: the saved context is bfloat16
          const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(o) + row * pitch + c);
          bq[q] = make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                              __uint_as_float(u.y & 0xffff0000u));
        } else {
          bq[q] = *reinterpret_cast<const float4*>(o + row * pitch + c);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < DELTA_RPW; ++q) {
      float acc = a[q].x * bq[q].x + a[q].y * bq[q].y + a[q].z * bq[q].z + a[q].w * bq[q].w;
      for (int off = lanes_per_head >> 1; off > 0; off >>= 1) acc += __shfl_xor_sync(FULL, acc, off);
      if (item[q] >= 0 && c < width && (lane % lanes_per_head) == 0) {
        const int b = int(item[q] / S), qi = int(item[q] - (long long)b * S);
        delta[((long long)b * h + c / dk) * S + qi] = acc;
      }
    }
  }
}

struct BwdSmem {
  // operand tiles: Q, K, V, dO of the whole slate (up to 256 rows = two 128-row boxes each, DK <= 32 -> one 128-byte
  // row per item), then the output staging tiles dV | dK | dQ
  static constexpr int OPS = 4 * 2 * TILE_BYTES;
  static constexpr int OUT_OFF = OPS;
  static constexpr int STATS_OFF = OUT_OFF + 3 * TILE_BYTES;    // float2 {nm_q, delta_q} x 256
  static constexpr int BITS_OFF = STATS_OFF + 256 * 8;          // 8 words: key is a real item
  static constexpr int BARS_OFF = BITS_OFF + 64;
  static constexpr int BIAS_OFF = BARS_OFF + 64;                // float [3 * d_model]: this CTA's QKV bias gradient
  static int total(int d_model) { return BIAS_OFF + 12 * d_model + 1024; }
};

// One CTA walks the (slate, head) items item0, item0 + gridDim.x, ...  (one CTA per item, or -- persistent -- one per
// SM).  Per item, eight warps run two phases on the tensor cores (mma.sync m16n8k8 tf32), each keeping its products
// in registers:
//   phase 1, per 128-key tile (warp = 16 keys):  S^T = K Q^T, dP^T = V dO^T over 8-query blocks,
//            P^T = exp2(S^T c + nm_q) (key mask, dropout), dS^T = P^T * (dP^T - delta_q),
//            dV += P^T dO,  dK += dS^T Q   (P^T / dS^T go straight from the accumulators into the next product)
//   phase 2, per 128-query tile (warp = 16 queries):  S = Q K^T, dP = dO V^T over 8-key blocks, dS as above,
//            dQ += dS K
// with nm_q = -max_q c - log2 l_q from the forward's row statistics and c = log2(e) / sqrt(dk).  Outputs are staged in
// shared memory and TMA-stored (+ the QKV bias column sums).
template <int DK, bool DROP, bool OUT16 = false>
__global__ void __launch_bounds__(BWD_THREADS, 1) attn_bwd_kernel(
    const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
    const __grid_constant__ CUtensorMap tmDQ, const __grid_constant__ CUtensorMap tmDK,
    const __grid_constant__ CUtensorMap tmDV, const uint8_t* __restrict__ mask, const float* __restrict__ stat_max,
    const float* __restrict__ stat_sum, const float* __restrict__ delta, int S, int n_heads, float scale, DropSite drop,
    float* __restrict__ dbias_qkv, int d_model, const int* __restrict__ extent, const int* __restrict__ pack_off,
    int n_items, int rnd) {
  constexpr int KS = DK / 8;
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* q_s = smem;
  uint8_t* k_s = smem + 2 * TILE_BYTES;
  uint8_t* v_s = smem + 4 * TILE_BYTES;
  uint8_t* do_s = smem + 6 * TILE_BYTES;
  auto out_tile = [&](int which) { return smem + BwdSmem::OUT_OFF + which * TILE_BYTES; };   // 0 dV, 1 dK, 2 dQ
  float2* qstats = reinterpret_cast<float2*>(smem + BwdSmem::STATS_OFF);
  uint32_t* key_bits = reinterpret_cast<uint32_t*>(smem + BwdSmem::BITS_OFF);
  uint64_t* load_bar = reinterpret_cast<uint64_t*>(smem + BwdSmem::BARS_OFF);
  float* bias_acc = reinterpret_cast<float*>(smem + BwdSmem::BIAS_OFF);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  // Rows at or beyond a slate's extent are masked keys (probability exactly 0) whose d ctx rows are exactly zero:
  // neither their key tiles nor their query tiles contribute anything, and their dQ / dK / dV rows are zero.  Only
  // the tiles below the extent are processed; in the dense layout the rest is written as zeros.
  // Packed rows (see attn_fwd_kernel): slate b holds its first ext16 = round_up(extent, 16) rows at row pack_off[b] of
  // one long tensor.  Tiles that overrun the slate read other slates' rows: as keys they are masked, as queries their
  // probabilities are forced to zero (their statistics are -inf); outputs are stored in 16-row boxes that stop at the
  // slate's last packed row, and nothing is zero-filled.
  const int n_full = (S + 127) / 128;
  const float c_log2e = scale * 1.4426950408889634f;
  const bool packed = pack_off != nullptr;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ); ptx::prefetch_tmap(&tmK); ptx::prefetch_tmap(&tmV); ptx::prefetch_tmap(&tmDO);
    ptx::mbar_init(load_bar, 1);
    ptx::fence_barrier_init();
  }
  if (dbias_qkv != nullptr)
    for (int i = threadIdx.x; i < 3 * d_model; i += BWD_THREADS) bias_acc[i] = 0.f;
  arb_pdl_wait();
  __syncthreads();

  // one operand word: element (r, e) of a [256][32] operand (two 128-row boxes)
  auto op = [&](const uint8_t* base, int r, int e) -> uint32_t {
    const float x = ptx::ld_f32(base + (r >> 7) * TILE_BYTES, r & 127, e);
    return rnd ? ptx::cvt_tf32(x) : __float_as_uint(x);
  };
  auto key_live = [&](int key) { return (key_bits[key >> 5] >> (key & 31)) & 1u; };
  // stage rows r, r + 8 (tile-relative) of an accumulator [KS][4] (x mul) into output tile `which`
  auto stage_rows = [&](int which, int r, const float (&acc)[KS][4], float mul) {
    uint8_t* ot = out_tile(which);
#pragma unroll
    for (int nt = 0; nt < KS; ++nt) {
      const int e = 8 * nt + 2 * t;
      if constexpr (OUT16) {
        // bf16 mode: dQ / dK / dV only feed the QKV weight- and input-gradient products: dense bfloat16 rows of
        // 32 columns (64 bytes), unswizzled tensor maps
        *reinterpret_cast<uint32_t*>(ot + r * 64 + 2 * e) = ptx::pack_bf16(acc[nt][0] * mul, acc[nt][1] * mul);
        *reinterpret_cast<uint32_t*>(ot + (r + 8) * 64 + 2 * e) = ptx::pack_bf16(acc[nt][2] * mul, acc[nt][3] * mul);
      } else {
        *reinterpret_cast<float2*>(ot + ptx::sw128(r, 4 * e)) = make_float2(acc[nt][0] * mul, acc[nt][1] * mul);
        *reinterpret_cast<float2*>(ot + ptx::sw128(r + 8, 4 * e)) = make_float2(acc[nt][2] * mul, acc[nt][3] * mul);
      }
    }
  };
  // store output tiles [first, last] (staged by every warp) at tile row `tile` of item (b, head) and add their column
  // sums to the QKV bias gradient; returns with the staging free again
  auto flush = [&](int first, int last, int tile, int b, int head, int row_base, int ext16) {
    ptx::fence_proxy_async_smem();
    __syncthreads();
    const CUtensorMap* maps[3] = {&tmDV, &tmDK, &tmDQ};
    if (threadIdx.x == 0) {
      for (int w = first; w <= last; ++w) {
        if (packed) {      // 16-row boxes up to the slate's last packed row (staged rows are 128 / 64 bytes wide)
          constexpr int BOX = OUT16 ? 1024 : 2048;
          const int n16 = (min(128, ext16 - 128 * tile) + 15) >> 4;
          for (int i = 0; i < n16; ++i) ptx::tma_store_4d(maps[w], out_tile(w) + i * BOX, 0, row_base + 128 * tile + 16 * i, head, 0);
        } else {
          ptx::tma_store_4d(maps[w], out_tile(w), 0, 128 * tile, head, b);
        }
      }
      ptx::tma_store_commit();
    }
    if (dbias_qkv != nullptr) {
      // bias gradient of the QKV projection: column sums of the staged tiles (rows the slate does not have are 0), added
      // to the CTA's accumulator -- one thread per (tile, column), flushes ordered by the barriers around them
      const int which = first + int(threadIdx.x) / DK, cc = int(threadIdx.x) % DK;
      if (which <= last) {
        const uint8_t* tl = out_tile(which);
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < 128; ++r) {
          if constexpr (OUT16) s += __uint_as_float(uint32_t(*reinterpret_cast<const uint16_t*>(tl + r * 64 + cc * 2)) << 16);
          else s += *reinterpret_cast<const float*>(tl + ptx::sw128(r, 4 * cc));
        }
        bias_acc[(which == 0 ? 2 * d_model : (which == 1 ? d_model : 0)) + head * DK + cc] += s;
      }
    }
    if (threadIdx.x == 0) ptx::tma_store_wait_read();
    __syncthreads();
  };

  uint32_t phase = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int b = item / n_heads, head = item - b * n_heads;
    int e = extent ? __ldg(extent + b) : S;
    if (packed && e <= 0) continue;               // packed rows: an empty slate holds no rows
    e = max(1, min(S, e));
    const int n_kt = (e + 127) / 128;             // active key tiles == active query tiles
    const int ext16 = (e + 15) & ~15;
    const int q_lim = packed ? min(S, ext16) : S; // queries at or beyond it do not exist in this slate
    // queries at or beyond q_live contribute nothing (the dense layout's padding has zero d ctx rows; packed rows: the
    // slate has no such queries)
    const int q_live = packed ? q_lim : (extent ? e : S);
    const int row_base = packed ? __ldg(pack_off + b) : 0;
    const int bc = packed ? 0 : b;
    if (threadIdx.x == 0) {
      ptx::fence_proxy_async_smem();
      ptx::mbar_expect_tx(load_bar, 4 * n_kt * TILE_BYTES);
      for (int kt = 0; kt < n_kt; ++kt) {
        const int r = row_base + 128 * kt;
        ptx::tma_load_4d(q_s + kt * TILE_BYTES, &tmQ, load_bar, 0, r, head, bc);
        ptx::tma_load_4d(k_s + kt * TILE_BYTES, &tmK, load_bar, 0, r, head, bc);
        ptx::tma_load_4d(v_s + kt * TILE_BYTES, &tmV, load_bar, 0, r, head, bc);
        ptx::tma_load_4d(do_s + kt * TILE_BYTES, &tmDO, load_bar, 0, r, head, bc);
      }
    }
    {
      // per-query statistics (nm = -max*c - log2(sum); -inf for queries the slate does not have) and the key mask
      const int qi = threadIdx.x;
      float2 st = make_float2(-CUDART_INF_F, 0.f);
      if (qi < q_lim) {
        const size_t so = (size_t(b) * n_heads + head) * S + qi;
        st.x = -(stat_max[so] * c_log2e) - log2f(stat_sum[so]);
        st.y = delta[so];
      }
      qstats[qi] = st;
      const uint32_t w = __ballot_sync(FULL, qi < S && mask[size_t(b) * S + qi] == 0);
      if (lane == 0) key_bits[warp] = w;
    }
    if (!packed && n_kt < n_full) {
      // dense layout: zero rows of the skipped tiles -- one zero tile, TMA-stored over every skipped dQ / dK / dV tile
      // (TMA clips at S)
      for (int i = threadIdx.x; i < TILE_BYTES / 16; i += BWD_THREADS) reinterpret_cast<uint4*>(out_tile(0))[i] = make_uint4(0u, 0u, 0u, 0u);
      ptx::fence_proxy_async_smem();
      __syncthreads();
      if (threadIdx.x == 0) {
        for (int jt = n_kt; jt < n_full; ++jt) {
          ptx::tma_store_4d(&tmDQ, out_tile(0), 0, 128 * jt, head, b);
          ptx::tma_store_4d(&tmDK, out_tile(0), 0, 128 * jt, head, b);
          ptx::tma_store_4d(&tmDV, out_tile(0), 0, 128 * jt, head, b);
        }
        ptx::tma_store_commit();
        ptx::tma_store_wait_read();
      }
    }
    __syncthreads();
    ptx::mbar_wait(load_bar, phase & 1);
    ++phase;

    const unsigned long long dbase = (unsigned long long)(b * n_heads + head) * S;
    // ===== phase 1: dV, dK of each key tile (this warp: keys kA, kA + 8 of its 16)
    const int nq8 = (min(q_live, 128 * n_kt) + 7) & ~7;
    for (int jt = 0; jt < n_kt; ++jt) {
      const int kA = 128 * jt + 16 * warp + g, kB = kA + 8;
      const bool liveA = key_live(kA), liveB = key_live(kB);
      uint32_t ka[KS][4], va[KS][4];
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const int e0 = 8 * ks + t;
        ka[ks][0] = op(k_s, kA, e0); ka[ks][1] = op(k_s, kB, e0); ka[ks][2] = op(k_s, kA, e0 + 4); ka[ks][3] = op(k_s, kB, e0 + 4);
        va[ks][0] = op(v_s, kA, e0); va[ks][1] = op(v_s, kB, e0); va[ks][2] = op(v_s, kA, e0 + 4); va[ks][3] = op(v_s, kB, e0 + 4);
      }
      float dv[KS][4], dk[KS][4];
#pragma unroll
      for (int nt = 0; nt < KS; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) dv[nt][i] = dk[nt][i] = 0.f;
      for (int q0 = 0; q0 < nq8; q0 += 8) {
        float s[4] = {0.f, 0.f, 0.f, 0.f}, dp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
          const uint32_t qb[2] = {op(q_s, q0 + g, 8 * ks + t), op(q_s, q0 + g, 8 * ks + t + 4)};
          const uint32_t ob[2] = {op(do_s, q0 + g, 8 * ks + t), op(do_s, q0 + g, 8 * ks + t + 4)};
          ptx::mma_tf32(s, ka[ks], qb);
          ptx::mma_tf32(dp, va[ks], ob);
        }
        float pu[4], ds[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int q = q0 + 2 * t + (i & 1);
          const float2 st = qstats[q];
          const float p = (i < 2 ? liveA : liveB) ? ex2_approx_b(fmaf(s[i], c_log2e, st.x)) : 0.0f;
          float p_used = p, dpv = dp[i];
          if constexpr (DROP) {        // regenerate the forward's dropout mask on the probabilities
            const unsigned long long idx = (dbase + q) * (unsigned long long)S + (i < 2 ? kA : kB);
            const float m = drop_keep(idx, drop.seed, drop.thresh) ? drop.scale : 0.0f;
            p_used = p * m;
            dpv *= m;
          }
          pu[i] = round_tf32_b(p_used);
          ds[i] = round_tf32_b(p * (dpv - st.y));
        }
        uint32_t pa[4], dsa[4];
        ptx::acc_to_a_tf32(pu, pa, lane);
        ptx::acc_to_a_tf32(ds, dsa, lane);
#pragma unroll
        for (int nt = 0; nt < KS; ++nt) {
          const uint32_t ob[2] = {op(do_s, q0 + t, 8 * nt + g), op(do_s, q0 + t + 4, 8 * nt + g)};
          const uint32_t qb[2] = {op(q_s, q0 + t, 8 * nt + g), op(q_s, q0 + t + 4, 8 * nt + g)};
          ptx::mma_tf32(dv[nt], pa, ob);
          ptx::mma_tf32(dk[nt], dsa, qb);
        }
      }
      stage_rows(0, 16 * warp + g, dv, 1.0f);
      stage_rows(1, 16 * warp + g, dk, scale);
      flush(0, 1, jt, b, head, row_base, ext16);
    }
    // ===== phase 2: dQ of each query tile (this warp: queries qA, qA + 8 of its 16)
    const int nk8 = (e + 7) & ~7;          // keys at or beyond the extent are masked
    for (int qc = 0; qc < n_kt; ++qc) {
      const int qA = 128 * qc + 16 * warp + g, qB = qA + 8;
      const float2 stA = qstats[qA], stB = qstats[qB];
      uint32_t qa[KS][4], oa[KS][4];
#pragma unroll
      for (int ks = 0; ks < KS; ++ks) {
        const int e0 = 8 * ks + t;
        qa[ks][0] = op(q_s, qA, e0); qa[ks][1] = op(q_s, qB, e0); qa[ks][2] = op(q_s, qA, e0 + 4); qa[ks][3] = op(q_s, qB, e0 + 4);
        oa[ks][0] = op(do_s, qA, e0); oa[ks][1] = op(do_s, qB, e0); oa[ks][2] = op(do_s, qA, e0 + 4); oa[ks][3] = op(do_s, qB, e0 + 4);
      }
      float dq[KS][4];
#pragma unroll
      for (int nt = 0; nt < KS; ++nt) dq[nt][0] = dq[nt][1] = dq[nt][2] = dq[nt][3] = 0.f;
      if (128 * qc + 16 * warp < q_live) {
        for (int k0 = 0; k0 < nk8; k0 += 8) {
          float s[4] = {0.f, 0.f, 0.f, 0.f}, dp[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            const uint32_t kb2[2] = {op(k_s, k0 + g, 8 * ks + t), op(k_s, k0 + g, 8 * ks + t + 4)};
            const uint32_t vb[2] = {op(v_s, k0 + g, 8 * ks + t), op(v_s, k0 + g, 8 * ks + t + 4)};
            ptx::mma_tf32(s, qa[ks], kb2);
            ptx::mma_tf32(dp, oa[ks], vb);
          }
          float ds[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int key = k0 + 2 * t + (i & 1);
            const float2 st = i < 2 ? stA : stB;
            const float p = key_live(key) ? ex2_approx_b(fmaf(s[i], c_log2e, st.x)) : 0.0f;
            float dpv = dp[i];
            if constexpr (DROP) {
              const unsigned long long idx = (dbase + (i < 2 ? qA : qB)) * (unsigned long long)S + key;
              dpv *= drop_keep(idx, drop.seed, drop.thresh) ? drop.scale : 0.0f;
            }
            ds[i] = round_tf32_b(p * (dpv - st.y));
          }
          uint32_t dsa[4];
          ptx::acc_to_a_tf32(ds, dsa, lane);
#pragma unroll
          for (int nt = 0; nt < KS; ++nt) {
            const uint32_t kb2[2] = {op(k_s, k0 + t, 8 * nt + g), op(k_s, k0 + t + 4, 8 * nt + g)};
            ptx::mma_tf32(dq[nt], dsa, kb2);
          }
        }
      }
      stage_rows(2, 16 * warp + g, dq, scale);
      flush(2, 2, qc, b, head, row_base, ext16);
    }
  }
  if (dbias_qkv != nullptr) {
    // this CTA's slot of the bias gradient (its items in a fixed order; the slots are summed in order by DetParts)
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * d_model; i += BWD_THREADS) dbias_qkv[size_t(blockIdx.x) * 3 * d_model + i] = bias_acc[i];
  }
  if (threadIdx.x == 0) ptx::tma_store_wait_all();
}

static int g_attn_bwd_persistent = ARB_DEFAULT_ATTN_BWD_PERSISTENT;
void set_attn_bwd_persistent(int on) { g_attn_bwd_persistent = on; }

template <int DK>
static int launch_bwd_t(const AttnBwdArgs& a, cudaStream_t st) {
  alignas(64) CUtensorMap tQ, tK, tV, tDO, tDQ, tDK, tDV;
  int rc;
  const TmapBox box{{32, 128, 1, 1}};
  if ((rc = make_tmap_4d(&tQ, a.q, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tK, a.k, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tV, a.v, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tDO, a.d_o, box, 0))) return rc;
  const bool out16 = a.dq.bf16 != 0;
  if ((a.dk_.bf16 != 0) != out16 || (a.dv.bf16 != 0) != out16) { arb_set_error("attn_bwd: dQ, dK, dV must share an element type"); return ARB_E_INVALID_ARG; }
  const bool packed = a.pack_off != nullptr;
  if (packed && !(a.extent && a.rows_dev && a.rowmap)) { arb_set_error("attn_bwd: packed rows need the extents, the row count and the row map"); return ARB_E_INVALID_ARG; }
  const TmapBox obox{{32, packed ? 16u : 128u, 1, 1}};
  if ((rc = make_tmap_4d(&tDQ, a.dq, obox, out16 ? 1 : 0))) return rc;
  if ((rc = make_tmap_4d(&tDK, a.dk_, obox, out16 ? 1 : 0))) return rc;
  if ((rc = make_tmap_4d(&tDV, a.dv, obox, out16 ? 1 : 0))) return rc;
  const double rf = packed ? arb_row_frac() : 1.0;
  {
    ProfScope ps(ARB_PROF_SCORER_SIMT, rf * double(a.B) * a.S * (8.0 * a.h * a.dk + 4.0 * a.h), st, 0.0, "attn_delta_kernel");
    const long long rows = packed ? (long long)a.q.dim[1] : (long long)a.B * a.S;   // packed: the buffers' row count
    arb_launch(attn_delta_kernel, dim3(unsigned((rows + 8 * DELTA_RPW - 1) / (8 * DELTA_RPW))), dim3(256), 0, st, a.do_ptr,
               static_cast<const float*>(a.o_ptr), (long long)a.o_pitch, a.B, a.S, a.h, a.dk, a.delta, a.o_bf16, a.rows_dev,
               a.rowmap, rows);
  }
  arb_count_launch();
  const bool drop = a.drop.thresh != 0;
  auto kern = out16 ? (drop ? attn_bwd_kernel<DK, true, true> : attn_bwd_kernel<DK, false, true>)
                    : (drop ? attn_bwd_kernel<DK, true> : attn_bwd_kernel<DK, false>);
  static int configured[ARB_MAX_DEVICES][4] = {};      // dynamic shared memory limit set so far
  const int dev = arb_device_slot();
  const int cslot = (drop ? 1 : 0) + (out16 ? 2 : 0);
  const int smem = BwdSmem::total(a.dbias_qkv ? a.d_model : 0);
  if (configured[dev][cslot] < smem) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      arb_set_error("attn_bwd: cannot raise the dynamic shared memory limit");
      return ARB_E_CUDA;
    }
    configured[dev][cslot] = smem;
  }
  // one CTA per (slate, head), or -- persistent (default) -- one per SM walking the items head-fastest
  const int n_items = a.h * a.B;
  int n_ctas = n_items;
  if (g_attn_bwd_persistent) {
    static int n_sm_of[ARB_MAX_DEVICES] = {};
    if (!n_sm_of[dev]) {
      int id = 0, n = 132;
      cudaGetDevice(&id);
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, id);
      n_sm_of[dev] = n;
    }
    n_ctas = std::min(n_items, n_sm_of[dev]);
  }
  dim3 grid(n_ctas);
  // the QKV bias gradient: one slot per CTA, summed in CTA order afterwards
  float* dbias = a.dbias_qkv;
  DetParts dp;
  dp.add(dbias, n_ctas, 1, 3LL * a.d_model, 3LL * a.d_model);
  if ((rc = dp.begin(st))) return rc;
  {
    ProfScope ps(ARB_PROF_GEMM, (a.extent ? arb_attn_frac() : 1.0) * 10.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
                 rf * 4.0 * double(a.B) * a.h * a.S * (7.0 * a.dk + 3.0), "attn_bwd_kernel");
    arb_launch(kern, grid, dim3(BWD_THREADS), size_t(smem), st, tQ, tK, tV, tDO, tDQ, tDK, tDV, a.mask,
               a.stat_max, a.stat_sum, a.delta, a.S, a.h, a.scale, a.drop, dbias, a.d_model, a.extent, a.pack_off,
               n_items, tf32_round_on_load());
  }
  arb_count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { arb_set_error(cudaGetErrorString(e)); return ARB_E_CUDA; }
  return dp.finish(st);
}

bool attn_fused_bwd_supported(int S, int dk) { return S >= 1 && S <= 256 && (dk == 16 || dk == 32); }

int launch_attn_bwd(const AttnBwdArgs& a, cudaStream_t st) {
  if (!attn_fused_bwd_supported(a.S, a.dk)) { arb_set_error("fused attention backward: unsupported shape"); return ARB_E_UNSUPPORTED; }
  return a.dk == 16 ? launch_bwd_t<16>(a, st) : launch_bwd_t<32>(a, st);
}

}  // namespace arb
