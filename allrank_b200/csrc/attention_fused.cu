// Fused self-attention core for slates of up to 256 items:  ctx = softmax(mask(Q K^T / sqrt(dk))) V
// in ONE kernel, the [S,S] score / probability tile living only in registers.
//
// Reference: attention() allrank/models/transformer.py:137-156 (+ the head split / concat of
// MultiHeadedAttention.forward :193-202, which here are just TMA coordinates).
//
// One CTA = one (slate b, head, 128-query tile).  Q (128 x dk), K and V (up to 256 x dk, in 128-key boxes) are staged
// by TMA straight out of the packed [B*S, 3*d_model] QKV activation (4-D tensor maps: dk, item, head, slate).
// Eight warps, each owning 16 query rows, run the whole attention on the tensor cores (mma.sync m16n8k8 tf32):
//   pass A  S = Q K^T, one 8-key block at a time, keeping only the masked row maximum;
//   pass B  the same blocks again: P = exp2((S - max) / sqrt(dk) * log2 e) (key mask, dropout), rounded to tf32 and
//           fed straight from the accumulator registers into O += P V.
// The O epilogue (1/rowsum) is staged in swizzled shared memory and TMA-stored into the concatenated-heads layout.
// Nothing of size S^2 touches HBM or shared memory: per (slate, head) the kernel reads 3*S*dk*4 bytes and writes
// S*dk*4 (+ 8*S of softmax statistics for the backward pass) -- versus ~5*S^2*4 bytes for the unfused sequence.
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "attention_fused.h"
#include "common.h"
#include "sm90_ptx.cuh"

namespace arb {

constexpr int ATT_THREADS = 256;               // 8 warps x 16 query rows

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float round_tf32(float x) {
  // round-to-nearest (ties away) to tf32 as "+ half an ulp of the 10-bit mantissa, then let the tensor core ignore the
  // low 13 bits" -- one integer add instead of cvt.rna.tf32.f32.  Same result as cvt.rna for every finite value
  // (probabilities are finite).
  return __uint_as_float(__float_as_uint(x) + 0x1000u);
}

template <int DK>
struct AttFwdSmem {
  static constexpr int NKB = (DK + 31) / 32;            // 32-wide column blocks of the head (one 128-byte row each)
  static constexpr int TILE = 128 * 128;                // one [128 rows][128 B] box
  static constexpr int Q_BYTES = NKB * TILE;            // [kb]
  static constexpr int KV_BYTES = 2 * NKB * TILE;       // [128-key chunk][kb]
  static constexpr int O_BYTES = NKB * TILE;            // staging [kb][128 rows][128 B]
  static constexpr int total() { return Q_BYTES + 2 * KV_BYTES + O_BYTES + 256 + 1024; }
};

template <int DK, bool DROP, bool OUT16 = false>
__global__ void __launch_bounds__(ATT_THREADS) attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ,
                                                               const __grid_constant__ CUtensorMap tmK,
                                                               const __grid_constant__ CUtensorMap tmV,
                                                               const __grid_constant__ CUtensorMap tmO,
                                                               const uint8_t* __restrict__ mask,
                                                               float* __restrict__ stat_max,
                                                               float* __restrict__ stat_sum, int S, int n_heads,
                                                               float scale_log2e, DropSite drop,
                                                               const int* __restrict__ extent,
                                                               const int* __restrict__ pack_off, int rnd) {
  using L = AttFwdSmem<DK>;
  constexpr int NKB = L::NKB;
  constexpr int KS = DK / 8;                 // k8 steps over the head width
  static_assert(!OUT16 || DK <= 32, "bf16 context: one 64-byte row per query");
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* q_s = smem;
  uint8_t* k_s = q_s + L::Q_BYTES;
  uint8_t* v_s = k_s + L::KV_BYTES;
  uint8_t* o_s = v_s + L::KV_BYTES;
  uint64_t* load_bar = reinterpret_cast<uint64_t*>(o_s + L::O_BYTES);
  uint32_t* mask_bits = reinterpret_cast<uint32_t*>(load_bar + 1);   // 8 words: bit j of word w = key 32w+j is real

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.x * 128, head = blockIdx.y, b = blockIdx.z;
  // Packed rows (pack_off != nullptr): the activations hold only the first round_up(extent, 16) rows of every slate,
  // slate b starting at row pack_off[b] of one long [rows, h, dk] tensor (TMA coordinates (.., row, head, 0)).  Boxes
  // that overrun the slate read the next slates' rows (finite; their keys are masked, their query rows never stored);
  // the output is stored in 16-row boxes that stop at the slate's last packed row.  extent / pack_off were written by
  // kernels at least two launches upstream, so they may be read before the PDL wait.
  const bool packed = pack_off != nullptr;
  const int row_base = packed ? __ldg(pack_off + b) : 0;
  const int bc = packed ? 0 : b;
  if (packed && m0 >= ((__ldg(extent + b) + 15) & ~15)) return;   // no packed query rows in this tile (or an empty slate)
  // keys at or beyond the slate's extent are all masked (probability exactly 0): the products, the softmax and the
  // K / V loads stop there.  At least one key block is always processed, so an all-padded slate still produces the
  // reference's NaN rows.
  const int kext = extent ? max(1, min(S, __ldg(extent + b))) : S;
  const int S8 = (kext + 7) & ~7;
  const int nkc = (S8 + 127) / 128;          // 128-key chunks

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ); ptx::prefetch_tmap(&tmK); ptx::prefetch_tmap(&tmV); ptx::prefetch_tmap(&tmO);
    ptx::mbar_init(load_bar, 1);
    ptx::fence_barrier_init();
  }
  arb_pdl_wait();
  if (threadIdx.x == 0) {
    ptx::mbar_expect_tx(load_bar, L::Q_BYTES + nkc * 2 * NKB * L::TILE);
    for (int kb = 0; kb < NKB; ++kb) {
      ptx::tma_load_4d(q_s + kb * L::TILE, &tmQ, load_bar, 32 * kb, row_base + m0, head, bc);
      for (int kc = 0; kc < nkc; ++kc) {
        ptx::tma_load_4d(k_s + (kc * NKB + kb) * L::TILE, &tmK, load_bar, 32 * kb, row_base + 128 * kc, head, bc);
        ptx::tma_load_4d(v_s + (kc * NKB + kb) * L::TILE, &tmV, load_bar, 32 * kb, row_base + 128 * kc, head, bc);
      }
    }
  }
  {                     // key mask as 8 words: one key per thread, one ballot per warp
    const int key = threadIdx.x;
    const uint32_t w = __ballot_sync(0xffffffffu, key < S && mask[size_t(b) * S + key] == 0);
    if (lane == 0) mask_bits[warp] = w;
  }
  __syncthreads();
  ptx::mbar_wait(load_bar, 0);

  const int g = lane >> 2, t = lane & 3;
  const int rA = 16 * warp + g, rB = rA + 8;        // this thread's two query rows of the tile
  auto kv_at = [&](const uint8_t* base, int key, int e) -> uint32_t {
    const float x = ptx::ld_f32(base + ((key >> 7) * NKB + (e >> 5)) * L::TILE, key & 127, e & 31);
    return rnd ? ptx::cvt_tf32(x) : __float_as_uint(x);
  };
  uint32_t qa[KS][4];
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const int e0 = 8 * ks + t, e1 = e0 + 4;
    const uint8_t* qt = q_s + (e0 >> 5) * L::TILE;
    auto qv = [&](int r, int e) { const float x = ptx::ld_f32(qt, r, e & 31); return rnd ? ptx::cvt_tf32(x) : __float_as_uint(x); };
    qa[ks][0] = qv(rA, e0); qa[ks][1] = qv(rB, e0); qa[ks][2] = qv(rA, e1); qa[ks][3] = qv(rB, e1);
  }
  // raw scores of keys 8j + 2t, 8j + 2t + 1 for rows rA, rB
  auto scores = [&](int j, float (&s)[4]) {
    s[0] = s[1] = s[2] = s[3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      const uint32_t kb2[2] = {kv_at(k_s, 8 * j + g, 8 * ks + t), kv_at(k_s, 8 * j + g, 8 * ks + t + 4)};
      ptx::mma_tf32(s, qa[ks], kb2);
    }
  };
  const int nj = S8 / 8;
  // ---- pass A: masked row maxima
  float mxA = -CUDART_INF_F, mxB = -CUDART_INF_F;
  for (int j = 0; j < nj; ++j) {
    float s[4];
    scores(j, s);
    const int k0 = 8 * j + 2 * t;
    const uint32_t bits = mask_bits[k0 >> 5] >> (k0 & 31);
    if (bits & 1u) { mxA = fmaxf(mxA, s[0]); mxB = fmaxf(mxB, s[2]); }
    if (bits & 2u) { mxA = fmaxf(mxA, s[1]); mxB = fmaxf(mxB, s[3]); }
  }
  mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 1)); mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 2));
  mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 1)); mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 2));
  // ---- pass B: probabilities and O = P V
  const float mxsA = mxA * scale_log2e, mxsB = mxB * scale_log2e;
  const int qA = m0 + rA, qB = m0 + rB;
  float sumA = 0.f, sumB = 0.f;
  float o[KS][4];
#pragma unroll
  for (int nt = 0; nt < KS; ++nt) o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f;
  for (int j = 0; j < nj; ++j) {
    float s[4];
    scores(j, s);
    const int k0 = 8 * j + 2 * t;
    const uint32_t bits = mask_bits[k0 >> 5] >> (k0 & 31);
    // exp((s - max)/sqrt(dk)) as exp2; padded keys contribute exactly 0.  An all-padded slate gives
    // (-inf) - (-inf) = NaN like the reference (quirk Q2).
    float p[4];
    p[0] = (bits & 1u) ? ex2_approx(fmaf(s[0], scale_log2e, -mxsA)) : 0.0f;
    p[1] = (bits & 2u) ? ex2_approx(fmaf(s[1], scale_log2e, -mxsA)) : 0.0f;
    p[2] = (bits & 1u) ? ex2_approx(fmaf(s[2], scale_log2e, -mxsB)) : 0.0f;
    p[3] = (bits & 2u) ? ex2_approx(fmaf(s[3], scale_log2e, -mxsB)) : 0.0f;
    sumA += p[0] + p[1];                 // softmax normalises BEFORE dropout (transformer.py:153-155)
    sumB += p[2] + p[3];
    if constexpr (DROP) {
      const unsigned long long base = (unsigned long long)(b * n_heads + head) * S;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned long long idx = (base + (i < 2 ? qA : qB)) * (unsigned long long)S + (k0 + (i & 1));
        p[i] = drop_keep(idx, drop.seed, drop.thresh) ? p[i] * drop.scale : 0.0f;
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) p[i] = round_tf32(p[i]);
    uint32_t pa[4];
    ptx::acc_to_a_tf32(p, pa, lane);
#pragma unroll
    for (int nt = 0; nt < KS; ++nt) {
      const uint32_t vb[2] = {kv_at(v_s, 8 * j + t, 8 * nt + g), kv_at(v_s, 8 * j + t + 4, 8 * nt + g)};
      ptx::mma_tf32(o[nt], pa, vb);
    }
  }
  sumA += __shfl_xor_sync(0xffffffffu, sumA, 1); sumA += __shfl_xor_sync(0xffffffffu, sumA, 2);
  sumB += __shfl_xor_sync(0xffffffffu, sumB, 1); sumB += __shfl_xor_sync(0xffffffffu, sumB, 2);
  if (t == 0) {
    const size_t so = (size_t(b) * n_heads + head) * S;
    if (qA < S) { stat_max[so + qA] = mxA; stat_sum[so + qA] = sumA; }
    if (qB < S) { stat_max[so + qB] = mxB; stat_sum[so + qB] = sumB; }
  }
  const float invA = 1.0f / sumA, invB = 1.0f / sumB;
#pragma unroll
  for (int nt = 0; nt < KS; ++nt) {
    const int e = 8 * nt + 2 * t;
    if constexpr (OUT16) {
      // bf16 mode: the context only feeds the output projection -- stage it as dense bfloat16 rows (32 columns =
      // 64 bytes, unswizzled tensor map)
      *reinterpret_cast<uint32_t*>(o_s + rA * 64 + 2 * e) = ptx::pack_bf16(o[nt][0] * invA, o[nt][1] * invA);
      *reinterpret_cast<uint32_t*>(o_s + rB * 64 + 2 * e) = ptx::pack_bf16(o[nt][2] * invB, o[nt][3] * invB);
    } else {
      uint8_t* ot = o_s + (e >> 5) * L::TILE;
      *reinterpret_cast<float2*>(ot + ptx::sw128(rA, 4 * (e & 31))) = make_float2(o[nt][0] * invA, o[nt][1] * invA);
      *reinterpret_cast<float2*>(ot + ptx::sw128(rB, 4 * (e & 31))) = make_float2(o[nt][2] * invB, o[nt][3] * invB);
    }
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();
  if (threadIdx.x == 0) {
    constexpr int OSLABS = OUT16 ? 1 : NKB;
    for (int sl = 0; sl < OSLABS; ++sl) {
      if (packed) {       // 16-row boxes up to the slate's last packed row (the staged rows are 128 / 64 bytes wide)
        const int ext16 = (__ldg(extent + b) + 15) & ~15;
        const int n16 = (min(128, ext16 - m0) + 15) >> 4;
        for (int i = 0; i < n16; ++i)
          ptx::tma_store_4d(&tmO, o_s + sl * L::TILE + i * (OUT16 ? 1024 : 2048), 32 * sl, row_base + m0 + 16 * i, head, 0);
      } else {
        ptx::tma_store_4d(&tmO, o_s + sl * L::TILE, 32 * sl, m0, head, b);
      }
    }
    ptx::tma_store_commit();
    ptx::tma_store_wait_all();
  }
}

// Both settings run attn_fwd_kernel; the switch is kept for the C ABI (arb_set_attention_fwd_two_pass).
void set_attn_fwd_two_pass(int) {}

template <int DK>
static int launch_fwd_t(const AttnFwdArgs& a, cudaStream_t st) {
  using L = AttFwdSmem<DK>;
  alignas(64) CUtensorMap tQ, tK, tV, tO;
  int rc;
  if ((rc = make_tmap_4d(&tQ, a.q, TmapBox{{32, 128, 1, 1}}, 0))) return rc;
  if ((rc = make_tmap_4d(&tK, a.k, TmapBox{{32, 128, 1, 1}}, 0))) return rc;
  if ((rc = make_tmap_4d(&tV, a.v, TmapBox{{32, 128, 1, 1}}, 0))) return rc;
  const bool out16 = a.o.bf16 != 0;
  if (out16 && DK > 32) { arb_set_error("attn_fwd: a bf16 context needs head width <= 32"); return ARB_E_UNSUPPORTED; }
  const bool packed = a.pack_off != nullptr;
  if (packed && !a.extent) { arb_set_error("attn_fwd: packed rows need the slate extents"); return ARB_E_UNSUPPORTED; }
  if ((rc = make_tmap_4d(&tO, a.o, TmapBox{{32, packed ? 16u : 128u, 1, 1}}, out16 ? 1 : 0))) return rc;
  const bool drop = a.drop.thresh != 0;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, const uint8_t*, float*, float*, int, int, float,
               DropSite, const int*, const int*, int);
  if constexpr (DK <= 32) {
    if (out16) kern = drop ? attn_fwd_kernel<DK, true, true> : attn_fwd_kernel<DK, false, true>;
    else kern = drop ? attn_fwd_kernel<DK, true> : attn_fwd_kernel<DK, false>;
  } else {
    kern = drop ? attn_fwd_kernel<DK, true> : attn_fwd_kernel<DK, false>;
  }
  dim3 grid((a.S + 127) / 128, a.h, a.B);
  ProfScope ps(ARB_PROF_GEMM, (a.extent ? arb_attn_frac() : 1.0) * 4.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
               (packed ? arb_row_frac() : 1.0) * 4.0 * double(a.B) * a.h * a.S * ((out16 ? 3.5 : 4.0) * a.dk + 2.0),
               "attn_fwd_kernel");
  return launch(kern, grid, dim3(ATT_THREADS), size_t(L::total()), st, /*pdl=*/true, tQ, tK, tV, tO, a.mask, a.stat_max,
                a.stat_sum, a.S, a.h, a.scale * 1.4426950408889634f, a.drop, a.extent, a.pack_off, tf32_round_on_load());
}

bool attn_fused_supported(int S, int dk) { return S >= 1 && S <= 256 && (dk == 16 || dk == 32 || dk == 64); }

int launch_attn_fwd(const AttnFwdArgs& a, cudaStream_t st) {
  if (!attn_fused_supported(a.S, a.dk)) { arb_set_error("fused attention: unsupported shape"); return ARB_E_UNSUPPORTED; }
  switch (a.dk) {
    case 16: return launch_fwd_t<16>(a, st);
    case 32: return launch_fwd_t<32>(a, st);
    default: return launch_fwd_t<64>(a, st);
  }
}

}  // namespace arb
