// Batched TF32 GEMM on the Hopper tensor cores:  C[M,N] = epilogue(alpha * A * B^T)
//
//   * operands staged by TMA (cp.async.bulk.tensor, 128-byte swizzle) into a STAGES-deep shared-memory ring,
//   * fp32 operands that are both K-major (every forward and input-gradient linear) run on warpgroup MMA: the four
//     consumer warps issue wgmma m64nNk8 with A in registers (ldmatrix, rounded to nearest tf32) and B read by the
//     tensor core straight from the swizzled ring.  fp32 operands that are both MN-major (the split-K weight
//     gradients) run on wgmma as well, with both operands read from shared memory: the warpgroup rewrites each ring
//     stage K-major (and rounded) into one of two on-chip stages, and the MMAs of one stage run while it rewrites the
//     next.  The mixed fp32 pairs and bf16 run warp-level mma.sync (m16n8k8 tf32 / m16n8k16 bf16), each warp owning 32
//     rows of the 128-row tile.  The fp32 accumulator stays in registers either way,
//   * the epilogue turns each 32-column chunk of a warp's accumulator into one row per thread (through a small
//     per-warp transpose buffer), applies bias / ReLU / residual / ReLU-mask, stages the tile in swizzled shared
//     memory and writes it with one TMA store per 32-column slab (TMA clips ragged edges, so a 240-row slate or a
//     136-wide feature matrix needs no masking code),
//   * either operand may be "K-major" (rows of K contiguous, e.g. nn.Linear weights [out,in]) or "MN-major"
//     (the transpose), which is what the backward GEMMs dX = dY W and dW = dY^T X need; the mma.sync fragment loads
//     address either layout directly,
//   * split-K for the weight gradients (K = all rows of the batch): every split stores its tile into a slot of its own
//     and the slots are summed in split order (DetParts), so results do not depend on the order splits finish in.
//
// Warp roles (192 threads): warps 0-3 = MMA + epilogue (one aligned warpgroup, as wgmma needs), warp 4 = TMA producer,
// warp 5 = idle.
//
// This one kernel is the tensor-core workhorse of the scorer: every nn.Linear forward/backward and the
// generic (unfused) attention contractions go through it.  Reference ops replaced: aten::addmm / aten::bmm
// issued from allrank/models/transformer.py:148,156,193-195,203,227 and allrank/models/model.py:41-44,117.
#include <cstdio>
#include <cstring>
#include <cuda.h>
#include <cuda_runtime.h>

#include "common.h"
#include "defaults.h"
#include "gemm_tf32.h"
#include "sm90_ptx.cuh"

namespace arb {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;                    // 32 fp32 = one 128-byte swizzle row
// bf16 operands keep the BYTE geometry: a k-block is still one 128-byte swizzle row (64 bf16), so ring stages and
// K-major tiles are shared; only MN-major tiles differ (SWIZZLE_128B slabs of 64 MN-elements x 64 k-rows instead of
// 32 x 32).
constexpr int BLOCK_K_BF16 = 64;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 4;   // 16 KB
constexpr int GEMM_EPI_GROUPS = 1;            // consumer warps per 32-row quarter of the tile
constexpr int GEMM_EPI_THREADS = 128 * GEMM_EPI_GROUPS;
constexpr int GEMM_THREADS = 64 + GEMM_EPI_THREADS;
constexpr int XPOSE_BYTES = 32 * 33 * 4;      // per-warp accumulator transpose buffer (32 rows x 32 columns, padded)

struct GemmParams {
  int M, N, K;
  int nb2;
  int a_b2, a_b3, b_b2, b_b3, c_b2, c_b3;
  int flags;
  int kb_per_split;   // k-blocks per split (split-K), or total k-blocks
  int rnd;            // round fp32 operands to tf32 (nearest) before the MMA; else the tensor core truncates them
  int rnd_b;          // wgmma path: round the B stages in place (rnd, unless B arrives rounded already)
  float alpha;
  int atomic_ld;         // EPI_ATOMIC: the row pitch of atomic_out; EPI_DROPOUT (never with EPI_ATOMIC): the row
                         // width of the dropout counter (GemmDesc::drop_n) -- one field keeps GemmParams in 128 bytes
  const float* bias;
  float* atomic_out;     // split-K: the splits' slots [split][M][atomic_ld] (DetParts), summed in order afterwards
  DropSite drop;
  float* colsum_out;
  const int* rows_dev;   // packed rows: device-resident live row count -- bounds M, or K for the split-K weight gradients
  uint32_t* bits;        // EPI_RELU_BITS / EPI_MASK_BITS: [M, N / 32] words
};
// The compiler keeps a kernel's by-value parameter struct of up to 128 bytes in registers; a larger GemmParams is
// read through its address instead, which costs most GEMM kernels registers and several of them spills.
static_assert(sizeof(GemmParams) <= 128, "GemmParams must stay within 128 bytes");

// ---- MMA main loop ------------------------------------------------------------------------------------------------
// One 32-bit operand word of a ring stage: an fp32 element (tf32 mode) or the bf16 pair (k, k+1) (k even) of row /
// column `rc`.  K-major tiles are [rows][128 B]; MN-major tiles are slabs of [k-rows][128 B] (32 fp32 / 64 bf16
// MN-elements per slab row).
template <bool MN, bool IN16>
__device__ __forceinline__ uint32_t op_word(const uint8_t* s, int rc, int k, int rnd) {
  if constexpr (IN16) {
    if constexpr (MN) {
      const uint8_t* slab = s + (rc >> 6) * 8192;
      const uint32_t lo = *reinterpret_cast<const uint16_t*>(slab + ptx::sw128(k, 2 * (rc & 63)));
      const uint32_t hi = *reinterpret_cast<const uint16_t*>(slab + ptx::sw128(k + 1, 2 * (rc & 63)));
      return lo | (hi << 16);
    } else {
      return *reinterpret_cast<const uint32_t*>(s + ptx::sw128(rc, 2 * k));
    }
  } else {
    const float x = MN ? ptx::ld_f32(s + (rc >> 5) * 4096, k, rc & 31) : ptx::ld_f32(s, rc, k);
    return rnd ? ptx::cvt_tf32(x) : __float_as_uint(x);
  }
}

// acc[mt][nt] += rows row0 + 16 mt .. of A  x  columns col(nt) .. +7 of B over one k-block of the ring.
// col(nt) = 32 * (slab0 + slab_step * (nt / 4)) + 8 * (nt % 4): the warp's 32-column slabs of the tile.
template <int NT, bool A_MN, bool B_MN, bool IN16>
__device__ __forceinline__ void warp_mma_kblock(float (&acc)[2][NT][4], const uint8_t* a_s, const uint8_t* b_s, int row0,
                                                int slab0, int slab_step, int rnd) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    // tf32: k8 steps (k = 8 ks + t, +4); bf16: k16 steps (pairs at k = 16 ks + 2t, +8)
    const int k0 = IN16 ? 16 * ks + 2 * t : 8 * ks + t;
    const int kh = IN16 ? 8 : 4;
    uint32_t a[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const int r = row0 + 16 * mt + g;
      a[mt][0] = op_word<A_MN, IN16>(a_s, r, k0, rnd);
      a[mt][1] = op_word<A_MN, IN16>(a_s, r + 8, k0, rnd);
      a[mt][2] = op_word<A_MN, IN16>(a_s, r, k0 + kh, rnd);
      a[mt][3] = op_word<A_MN, IN16>(a_s, r + 8, k0 + kh, rnd);
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int n = 32 * (slab0 + slab_step * (nt >> 2)) + 8 * (nt & 3) + g;
      const uint32_t b[2] = {op_word<B_MN, IN16>(b_s, n, k0, rnd), op_word<B_MN, IN16>(b_s, n, k0 + kh, rnd)};
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        if constexpr (IN16) ptx::mma_bf16(acc[mt][nt], a[mt], b);
        else ptx::mma_tf32(acc[mt][nt], a[mt], b);
      }
    }
  }
}

// fp32 operands with both A and B K-major run on warpgroup MMA (wgmma) instead: the consumer warps form one warpgroup
// per 128 x WG_N(BLOCK_N) block of the output.  Both kernels issue the same instruction shapes in the same k order, so the
// one-tile and the persistent kernel give bit-identical results.  fp32 operands that are both MN-major (the split-K
// weight gradients, some batched attention products) run on wgmma too, in the one-tile kernel only: the warpgroup
// first rewrites each ring stage K-major (wg_kmajor_stage).
template <int A_MN, int B_MN, bool IN16>
constexpr bool use_wgmma() { return A_MN == B_MN && !IN16; }
template <int A_MN, int B_MN, bool IN16>
constexpr bool wgmma_transposed() { return A_MN == 1 && B_MN == 1 && !IN16; }
template <int BLOCK_N>
constexpr int wg_cols() { return BLOCK_N == 128 ? 64 : 32; }

// acc[mt][nt] += rows 64 mt + 16 w .. +15 of A (w: the warp's rank in its warpgroup)  x  columns col0 + 8 nt .. +7 of
// B over one k-block of the ring, issued by the calling warp's whole warpgroup (128 threads, named barrier `bar`).
// The A fragments come from ptx::load_a_tf32 (ldmatrix + round to nearest in registers); with rnd_b, the warpgroup first
// rounds its B rows in place (wgmma reads B from shared memory and would truncate it).  Returns with the MMAs of this
// k-block complete, so the caller may release the stage.
template <int NT, int WN>
__device__ __forceinline__ void wg_mma_kblock(float (&acc)[2][NT][4], const uint8_t* a_s, uint8_t* b_s, int col0,
                                              int rnd, int rnd_b, int bar) {
  const int w = (threadIdx.x >> 5) & 3;
  if (rnd_b) {
    float4* b4 = reinterpret_cast<float4*>(b_s + col0 * 128);
#pragma unroll
    for (int i = threadIdx.x & 127; i < NT * 8 * 8; i += 128) {
      float4 v = b4[i];
      v.x = __uint_as_float(ptx::cvt_tf32(v.x)); v.y = __uint_as_float(ptx::cvt_tf32(v.y));
      v.z = __uint_as_float(ptx::cvt_tf32(v.z)); v.w = __uint_as_float(ptx::cvt_tf32(v.w));
      b4[i] = v;
    }
    ptx::fence_proxy_async_smem();
    ptx::named_bar_sync(bar, 128);
  }
  uint32_t a[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) ptx::load_a_tf32(a[mt], a_s, 64 * mt + 16 * w, rnd);
  const uint64_t desc = ptx::wgmma_desc_sw128(b_s + col0 * 128);
  ptx::wgmma_fence_acc(acc[0]);
  ptx::wgmma_fence_acc(acc[1]);
  ptx::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const uint64_t d = desc + 2 * ks;                     // +32 bytes (8 tf32) per k8 step
      if constexpr (WN == 64) {
        ptx::wgmma_m64n64k8_tf32<0>(acc[mt], a[mt][ks], d);
        if constexpr (NT == 16) ptx::wgmma_m64n64k8_tf32<8>(acc[mt], a[mt][ks], d + 64 * 128 / 16);
      } else {
        ptx::wgmma_m64n32k8_tf32<0>(acc[mt], a[mt][ks], d);
        if constexpr (NT == 8) ptx::wgmma_m64n32k8_tf32<4>(acc[mt], a[mt][ks], d + 32 * 128 / 16);
      }
    }
  ptx::wgmma_commit();
  ptx::wgmma_wait0();
  ptx::wgmma_fence_acc(acc[0]);
  ptx::wgmma_fence_acc(acc[1]);
}

// Both operands MN-major: tf32 wgmma reads only K-major tiles from shared memory, so the warpgroup (128 threads)
// rewrites a ring stage K-major into `kt`, rounded to nearest tf32 on the way when `rnd` (else the tensor core
// truncates).  The stage is NSLAB slabs (4 of A, then those of B) of 32 k-rows x 128 bytes, element (k, m) of a slab at
// sw128(k, 4 m).  In `kt` slab sl becomes rows 32 sl .. 32 sl + 31 of 128 bytes, element (m, k) at sw128(m, 4 k) of the
// slab's 4 KB: the A tile (rows 0..127) and then the B tile, both in the layout TMA gives K-major operands.
//
// A thread moves 4 x 4 blocks: k-rows 4 kc .. 4 kc + 3 of 16-byte chunk c (MN-elements 4 c .. 4 c + 3) come in as four
// 16-byte loads, and the rows m = 4 c .. 4 c + 3 of 16-byte chunk kc go out as four 16-byte stores.  Bank conflicts: a
// warp's 16-byte access is served 8 lanes (128 bytes) at a time, conflict-free when those 8 lanes touch the 8 distinct
// 16-byte bank groups of a 128-byte row.  Lane l (0..7) of each 8-lane group takes kc = l and c = l ^ d, d being the
// group's diagonal of the slab's 8 x 8 blocks.  Load j (k = 4 l + j) hits bank group c ^ (k & 7) = P(l) ^ d ^ j, store j
// (m = 4 c + j) hits kc ^ (m & 7) = P(l) ^ 4 (d & 1) ^ j, with P(l) = l ^ 4 (l & 1) a permutation of 0..7: 8 distinct
// groups either way.  The 16 groups of a warpgroup walk the 8 NSLAB (slab, diagonal) pairs.
template <int NSLAB>
__device__ __forceinline__ void wg_kmajor_stage(const uint8_t* ring, uint8_t* kt, int rnd) {
  constexpr int TASKS = 8 * NSLAB, PER = (TASKS + 15) / 16;
  const int l = threadIdx.x & 7, grp = (threadIdx.x & 127) >> 3;
  const uint32_t src0 = ptx::smem_u32(ring), dst0 = ptx::smem_u32(kt);
  float v[PER][4][4];                       // [task][k][m]
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    const int task = grp + 16 * u;
    if (TASKS % 16 != 0 && task >= TASKS) continue;
    const uint32_t src = src0 + (task >> 3) * 4096;
    const int c = l ^ (task & 7);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int k = 4 * l + j;
      const float4 x = ptx::lds128(src + k * 128 + ((c ^ (k & 7)) << 4));
      v[u][j][0] = x.x; v[u][j][1] = x.y; v[u][j][2] = x.z; v[u][j][3] = x.w;
    }
  }
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    const int task = grp + 16 * u;
    if (TASKS % 16 != 0 && task >= TASKS) continue;
    const uint32_t dst = dst0 + (task >> 3) * 4096;
    const int c = l ^ (task & 7);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = 4 * c + j;
      float o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) o[e] = rnd ? __uint_as_float(ptx::cvt_tf32(v[u][e][j])) : v[u][e][j];
      ptx::sts128(dst + m * 128 + ((l ^ (m & 7)) << 4), make_float4(o[0], o[1], o[2], o[3]));
    }
  }
}

// acc += the K-major stage `kt` written by wg_kmajor_stage (A: rows 0..127, B: the BLOCK_N rows after them), both
// operands read by the tensor core from shared memory; same instruction shapes, accumulator layout and k8 order as
// wg_mma_kblock.  Issued and committed, not waited for.
template <int NT, int WN>
__device__ __forceinline__ void wg_mma_kmajor(float (&acc)[2][NT][4], const uint8_t* kt) {
  const uint64_t da = ptx::wgmma_desc_sw128(kt), db = ptx::wgmma_desc_sw128(kt + A_STAGE_BYTES);
  ptx::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const uint64_t a = da + mt * (64 * 128 / 16) + 2 * ks, b = db + 2 * ks;
      if constexpr (WN == 64) {
        ptx::wgmma_m64n64k8_tf32_ss<0>(acc[mt], a, b);
        if constexpr (NT == 16) ptx::wgmma_m64n64k8_tf32_ss<8>(acc[mt], a, b + 64 * 128 / 16);
      } else {
        ptx::wgmma_m64n32k8_tf32_ss<0>(acc[mt], a, b);
        if constexpr (NT == 8) ptx::wgmma_m64n32k8_tf32_ss<4>(acc[mt], a, b + 32 * 128 / 16);
      }
    }
  ptx::wgmma_commit();
}

// The 32 accumulator values of chunk `c` (n-tiles 4c .. 4c+3) of the warp's accumulator row `lane` (fragment row
// 16 mt + g), one row per thread: the fragments go through the warp's transpose buffer `xp`.
template <int NT>
__device__ __forceinline__ void acc_chunk_row(const float (&acc)[2][NT][4], int c, float* xp, uint32_t (&v)[32]) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  __syncwarp();
#pragma unroll
  for (int cc = 0; cc < NT / 4; ++cc) {
    if (cc != c) continue;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float* r0 = xp + (16 * mt + g) * 33 + 8 * j + 2 * t;
        r0[0] = acc[mt][4 * cc + j][0];
        r0[1] = acc[mt][4 * cc + j][1];
        r0[8 * 33] = acc[mt][4 * cc + j][2];
        r0[8 * 33 + 1] = acc[mt][4 * cc + j][3];
      }
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(xp[lane * 33 + j]);
}

// ---- epilogue element transform -----------------------------------------------------------------------------------
// One thread turns its 32 accumulator values of a 32-column chunk into the staged fp32 output row piece by piece.
// The flags are COMPILE-TIME here: with run-time flags the unrolled loop carries a test per element and flag (about
// 20 instructions per element), and the epilogue bounds the short-K linears.  epi_chunk_dispatch picks the
// instantiation once per chunk; unusual flag combinations take the generic run-time path.
// `word`: the chunk's 32 mask bits of this row (EPI_MASK_BITS); returns the chunk's ReLU bits (EPI_RELU_BITS, else 0).
template <int F>
__device__ __forceinline__ uint32_t epi_chunk_f32(const uint32_t (&v)[32], uint8_t* slab_row, int row, const float* bias_c,
                                                  float alpha, uint32_t word = 0u) {
  uint32_t out_bits = 0u;
#pragma unroll
  for (int piece = 0; piece < 8; ++piece) {
    float4* dst = reinterpret_cast<float4*>(slab_row + ((piece ^ (row & 7)) << 4));
    float4 o = make_float4(__uint_as_float(v[piece * 4 + 0]) * alpha, __uint_as_float(v[piece * 4 + 1]) * alpha,
                           __uint_as_float(v[piece * 4 + 2]) * alpha, __uint_as_float(v[piece * 4 + 3]) * alpha);
    if constexpr ((F & EPI_BIAS) != 0) {
      const float4 bv = *reinterpret_cast<const float4*>(bias_c + 4 * piece);
      o.x += bv.x; o.y += bv.y; o.z += bv.z; o.w += bv.w;
    }
    if constexpr ((F & EPI_RELU) != 0) {
      o.x = fmaxf(o.x, 0.0f); o.y = fmaxf(o.y, 0.0f); o.z = fmaxf(o.z, 0.0f); o.w = fmaxf(o.w, 0.0f);
    }
    if constexpr ((F & (EPI_ADD_AUX | EPI_MASK_AUX)) != 0) {
      const float4 a = *dst;
      if constexpr ((F & EPI_ADD_AUX) != 0) { o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w; }
      if constexpr ((F & EPI_MASK_AUX) != 0) {
        o.x = a.x > 0.f ? o.x : 0.f; o.y = a.y > 0.f ? o.y : 0.f; o.z = a.z > 0.f ? o.z : 0.f; o.w = a.w > 0.f ? o.w : 0.f;
      }
    }
    if constexpr ((F & EPI_MASK_BITS) != 0) {
      o.x = (word >> (4 * piece + 0)) & 1u ? o.x : 0.f; o.y = (word >> (4 * piece + 1)) & 1u ? o.y : 0.f;
      o.z = (word >> (4 * piece + 2)) & 1u ? o.z : 0.f; o.w = (word >> (4 * piece + 3)) & 1u ? o.w : 0.f;
    }
    if constexpr ((F & EPI_RELU_BITS) != 0) {
      out_bits |= (o.x > 0.f ? 1u : 0u) << (4 * piece + 0) | (o.y > 0.f ? 1u : 0u) << (4 * piece + 1) |
                  (o.z > 0.f ? 1u : 0u) << (4 * piece + 2) | (o.w > 0.f ? 1u : 0u) << (4 * piece + 3);
    }
    *dst = o;
  }
  return out_bits;
}
// returns false when the flag combination has no specialisation (caller runs the generic loop); `bits_at`: this row's
// word of the chunk in the bit-mask array (written for EPI_RELU_BITS; nullptr: out of range); word_in: the same word,
// already loaded, for EPI_MASK_BITS
__device__ __forceinline__ bool epi_chunk_dispatch(int flags, const uint32_t (&v)[32], uint8_t* slab_row, int row,
                                                   const float* bias_c, float alpha, uint32_t* bits_at = nullptr,
                                                   uint32_t word_in = 0u) {
  switch (flags & (EPI_BIAS | EPI_RELU | EPI_ADD_AUX | EPI_MASK_AUX | EPI_DROPOUT | EPI_ATOMIC | EPI_RELU_BITS | EPI_MASK_BITS)) {
    case 0: epi_chunk_f32<0>(v, slab_row, row, bias_c, alpha); return true;
    case EPI_BIAS: epi_chunk_f32<EPI_BIAS>(v, slab_row, row, bias_c, alpha); return true;
    case EPI_BIAS | EPI_RELU: epi_chunk_f32<EPI_BIAS | EPI_RELU>(v, slab_row, row, bias_c, alpha); return true;
    case EPI_BIAS | EPI_ADD_AUX: epi_chunk_f32<EPI_BIAS | EPI_ADD_AUX>(v, slab_row, row, bias_c, alpha); return true;
    case EPI_MASK_AUX: epi_chunk_f32<EPI_MASK_AUX>(v, slab_row, row, bias_c, alpha); return true;
    case EPI_BIAS | EPI_RELU | EPI_RELU_BITS: {
      const uint32_t w = epi_chunk_f32<EPI_BIAS | EPI_RELU | EPI_RELU_BITS>(v, slab_row, row, bias_c, alpha);
      if (bits_at) *bits_at = w;
      return true;
    }
    case EPI_MASK_BITS:
      epi_chunk_f32<EPI_MASK_BITS>(v, slab_row, row, bias_c, alpha, word_in);   // (fetched one chunk ahead by the caller)
      return true;
    default: return false;
  }
}

// ---- TMA producer loads -------------------------------------------------------------------------------------------
// One k-block (elements k0 ..) of A (tile rows m0 ..) and B (tile rows n0 ..) of batch (b2, b3) into the ring stage at
// a_s (B after the A_STAGE_BYTES of A), completing on `bar`.  An MN-major operand comes as slabs of 32 fp32 / 64 bf16
// MN-elements x one k-block; a K-major one as one box of 128-byte rows.
template <int A_MN, int B_MN, bool IN16, int BLOCK_N>
__device__ __forceinline__ void load_stage(uint8_t* a_s, uint64_t* bar, const CUtensorMap* tmA, const CUtensorMap* tmB,
                                           const GemmParams& p, int m0, int n0, int k0, int b2, int b3) {
  constexpr int MN_SLAB = IN16 ? 64 : 32;                     // MN-elements per MN-major slab (128 bytes)
  constexpr int MN_SLAB_BYTES = MN_SLAB * 128;                // the k-block's 32 / 64 k-rows of 128 bytes: 4096 / 8192
  uint8_t* b_s = a_s + A_STAGE_BYTES;
  ptx::mbar_expect_tx(bar, A_STAGE_BYTES + BLOCK_N * 128);
  if (A_MN) {
    for (int c = 0; c < BLOCK_M / MN_SLAB; ++c)
      ptx::tma_load_4d(a_s + c * MN_SLAB_BYTES, tmA, bar, m0 + MN_SLAB * c, k0, b2 * p.a_b2, b3 * p.a_b3);
  } else {
    ptx::tma_load_4d(a_s, tmA, bar, k0, m0, b2 * p.a_b2, b3 * p.a_b3);
  }
  if (B_MN) {
    for (int c = 0; c < BLOCK_N / MN_SLAB; ++c)
      ptx::tma_load_4d(b_s + c * MN_SLAB_BYTES, tmB, bar, n0 + MN_SLAB * c, k0, b2 * p.b_b2, b3 * p.b_b3);
  } else {
    ptx::tma_load_4d(b_s, tmB, bar, k0, n0, b2 * p.b_b2, b3 * p.b_b3);
  }
}
// The residual / ReLU-mask tile of output tile (m0, n0) into the staging slabs, completing on `bar`.  It has the
// output's element type: 128-byte slab rows hold 32 fp32 or 64 bf16 columns.
template <int BLOCK_N, bool OUT16>
__device__ __forceinline__ void load_aux_tile(uint8_t* staging, uint64_t* bar, const CUtensorMap* tmAux,
                                              const GemmParams& p, int m0, int n0, int b2, int b3) {
  constexpr int OUT_COLS = OUT16 ? 64 : 32, OUT_SLABS = BLOCK_N / OUT_COLS;
  ptx::mbar_expect_tx(bar, OUT_SLABS * BLOCK_M * 128);
  for (int c = 0; c < OUT_SLABS; ++c)
    ptx::tma_load_4d(staging + c * (BLOCK_M * 128), tmAux, bar, n0 + OUT_COLS * c, m0, b2 * p.c_b2, b3 * p.c_b3);
}

template <int BLOCK_N, int NST = 2, bool KM = false>
struct SmemLayout {
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 4;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGING_BYTES = BLOCK_M * BLOCK_N * 4;
  // Two stages: the contraction is short (K = 32..512) and latency is hidden by co-resident CTAs instead.
  // weight-gradient GEMMs (both operands MN-major, K = all rows of the batch) run a long K loop per CTA: 4 stages
  static constexpr int stages() { return NST; }
  static constexpr int pipe_bytes() { return stages() * STAGE_BYTES; }
  // KM (fp32, both operands MN-major): after the ring, the two K-major stages wgmma reads (wg_kmajor_stage)
  static constexpr int kmajor_bytes() { return KM ? 2 * STAGE_BYTES : 0; }
  // The output staging tile (and the residual / mask tile, fetched only after the last MMA) aliases the operand
  // ring: both are touched only once every consumer warp has finished reading it.
  static constexpr int body_bytes() {
    return pipe_bytes() + kmajor_bytes() > STAGING_BYTES ? pipe_bytes() + kmajor_bytes() : STAGING_BYTES;
  }
  static constexpr int XPOSE_OFF = 256 + BLOCK_N * 4;     // after the barriers and the bias row, in the tail
  static constexpr int total() { return body_bytes() + XPOSE_OFF + (GEMM_EPI_THREADS / 32) * XPOSE_BYTES + 1024; }
};

template <int BLOCK_N, int A_MN, int B_MN, bool DROP, int NST, bool IN16 = false, bool OUT16 = false>
__global__ void __launch_bounds__(GEMM_THREADS) gemm_tf32_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                 const __grid_constant__ CUtensorMap tmB,
                                                                 const __grid_constant__ CUtensorMap tmC,
                                                                 const __grid_constant__ CUtensorMap tmAux,
                                                                 const GemmParams p) {
  constexpr bool WG = use_wgmma<A_MN, B_MN, IN16>();
  constexpr bool WG_T = wgmma_transposed<A_MN, B_MN, IN16>();
  using L = SmemLayout<BLOCK_N, NST, WG_T>;
  constexpr int STAGES = L::stages();
  constexpr int N_SLABS = BLOCK_N / 32;                       // 32-column accumulator chunks
  constexpr int NT = BLOCK_N / 8;                             // 8-column MMA tiles per warp
  constexpr int N_CONSUMERS = GEMM_EPI_THREADS / 32;          // warps 0 .. N_CONSUMERS-1; the next one is the producer
  static_assert(!WG_T || N_CONSUMERS == 4, "the K-major rewrite is one warpgroup's");
  constexpr int OUT_COLS = OUT16 ? 64 : 32;                   // output columns per 128-byte staging slab row
  constexpr int OUT_SLABS = (BLOCK_N + OUT_COLS - 1) / OUT_COLS;
  static_assert(!OUT16 || BLOCK_N >= 64, "bf16 outputs need at least one full 128-byte slab row");

  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  const bool has_aux = (p.flags & (EPI_ADD_AUX | EPI_MASK_AUX)) != 0;
  uint8_t* staging = smem;
  uint8_t* tail = smem + L::body_bytes();
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* ring_done_bar = empty_bar + STAGES;   // every consumer warp has read its last k-block
  uint64_t* aux_bar = ring_done_bar + 1;
  float* bias_s = reinterpret_cast<float*>(tail + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BLOCK_N, m0 = blockIdx.y * BLOCK_M;
  const bool split = (p.flags & EPI_ATOMIC) != 0;
  const int b2 = split ? 0 : int(blockIdx.z) % p.nb2, b3 = split ? 0 : int(blockIdx.z) / p.nb2;
  constexpr int KELEMS = IN16 ? BLOCK_K_BF16 : BLOCK_K;       // elements of K per k-block (128 bytes either way)
  // Packed rows: the live row count is on the device (written at least two launches upstream, so it may be read
  // before the PDL wait).  It bounds M -- CTAs of tiles beyond it leave at once -- or, for the split-K weight gradients,
  // K, which is then divided evenly over the grid's splits here.
  const bool dev_rows = p.rows_dev != nullptr;
  if (dev_rows && !split && m0 >= __ldg(p.rows_dev)) return;
  const int k_live = (dev_rows && split) ? min(p.K, __ldg(p.rows_dev)) : p.K;
  const int total_kb = (k_live + KELEMS - 1) / KELEMS;
  const int kb_per = (dev_rows && split) ? (total_kb + int(gridDim.z) - 1) / int(gridDim.z) : p.kb_per_split;
  const int kb_begin = split ? int(blockIdx.z) * kb_per : 0;
  const int kb_end = split ? min(total_kb, kb_begin + kb_per) : total_kb;
  const int nkb = max(0, kb_end - kb_begin);

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    if (!split) ptx::prefetch_tmap(&tmC);
    if (has_aux) ptx::prefetch_tmap(&tmAux);
    for (int s = 0; s < STAGES; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], N_CONSUMERS); }
    ptx::mbar_init(ring_done_bar, N_CONSUMERS);
    ptx::mbar_init(aux_bar, 1);
    ptx::fence_barrier_init();
  }
  arb_pdl_wait();          // everything above overlaps the previous kernel's tail; global memory is touched below
  __syncthreads();

  if (warp == N_CONSUMERS) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES, round = i / STAGES;
        if (round > 0) ptx::mbar_wait(&empty_bar[s], (round - 1) & 1);
        load_stage<A_MN, B_MN, IN16, BLOCK_N>(smem + s * L::STAGE_BYTES, &full_bar[s], &tmA, &tmB, p, m0, n0,
                                              (kb_begin + i) * KELEMS, b2, b3);
      }
      if (has_aux) {
        // the residual / ReLU-mask tile goes into the staging area, i.e. over the operand ring: wait until every
        // consumer warp has finished reading it
        if (nkb > 0) ptx::mbar_wait(ring_done_bar, 0);
        load_aux_tile<BLOCK_N, OUT16>(staging, aux_bar, &tmAux, p, m0, n0, b2, b3);
      }
    }
  } else if (warp < N_CONSUMERS) {
    // ===================== MMA + epilogue (warps 0..N_CONSUMERS-1) =====================
    const int q = warp & 3;                 // mma.sync: 32-row quarter of the tile; wgmma: rank in the warpgroup
    // row of the tile owned by this thread in the epilogue (wgmma: the warp computes rows 16q.. and 64+16q.., 16 each)
    const int row = WG ? 64 * (lane >> 4) + 16 * q + (lane & 15) : 32 * q + lane;
    const int et = threadIdx.x;             // 0..GEMM_EPI_THREADS-1
    const int grp = warp >> 2;              // which chunks: grp, grp + GEMM_EPI_GROUPS, ...
    float* xp = reinterpret_cast<float*>(tail + L::XPOSE_OFF) + warp * (XPOSE_BYTES / 4);
    if (p.flags & EPI_BIAS) {
      for (int j = et; j < BLOCK_N; j += GEMM_EPI_THREADS) bias_s[j] = (n0 + j < p.N) ? p.bias[n0 + j] : 0.0f;
    }
    // EPI_MASK_BITS: this row's mask word of a chunk is fetched one chunk ahead (a global load per row and chunk); the
    // first one goes out before the main loop
    auto mask_word = [&](int c) -> uint32_t {
      return ((p.flags & EPI_MASK_BITS) && c < N_SLABS && m0 + row < p.M && n0 + 32 * c < p.N)
                 ? p.bits[(long long)(m0 + row) * (p.N >> 5) + ((n0 >> 5) + c)] : 0u;
    };
    uint32_t word_next = mask_word(grp);
    float acc[2][NT][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.f;
    if constexpr (WG_T) {
      // ring stage i -> K-major stage i & 1 (which frees the ring stage at once); the MMAs of stage i then run while
      // the warpgroup rewrites stage i + 1.  Each warp waits for its MMAs of stage i - 1 before the barrier of stage i,
      // so no warp rewrites a K-major stage that the tensor core may still read.
      uint8_t* kmajor = smem + L::pipe_bytes();
      for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES, round = i / STAGES;
        ptx::mbar_wait(&full_bar[s], round & 1);
        uint8_t* kt = kmajor + (i & 1) * L::STAGE_BYTES;
        wg_kmajor_stage<4 + N_SLABS>(smem + s * L::STAGE_BYTES, kt, p.rnd);
        ptx::fence_proxy_async_smem();                     // generic-proxy writes -> the tensor core's reads
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty_bar[s]);
        ptx::wgmma_wait0();
        ptx::wgmma_fence_acc(acc[0]);
        ptx::wgmma_fence_acc(acc[1]);
        ptx::named_bar_sync(1, GEMM_EPI_THREADS);
        wg_mma_kmajor<NT, wg_cols<BLOCK_N>()>(acc, kt);
      }
      ptx::wgmma_wait0();
      ptx::wgmma_fence_acc(acc[0]);
      ptx::wgmma_fence_acc(acc[1]);
    } else {
      for (int i = 0; i < nkb; ++i) {
        const int s = i % STAGES, round = i / STAGES;
        ptx::mbar_wait(&full_bar[s], round & 1);
        uint8_t* a_s = smem + s * L::STAGE_BYTES;
        if constexpr (WG) wg_mma_kblock<NT, wg_cols<BLOCK_N>()>(acc, a_s, a_s + A_STAGE_BYTES, 0, p.rnd, p.rnd_b, 1);
        else warp_mma_kblock<NT, A_MN, B_MN, IN16>(acc, a_s, a_s + A_STAGE_BYTES, 32 * q, 0, 1, p.rnd);
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty_bar[s]);      // this warp is done with the stage
      }
    }
    if (lane == 0) ptx::mbar_arrive(ring_done_bar);
    // the staging tile aliases the ring: no warp writes it before every warp has finished its MMAs (this barrier also
    // publishes the bias row)
    ptx::named_bar_sync(1, GEMM_EPI_THREADS);
    if (has_aux) ptx::mbar_wait(aux_bar, 0);
    const uint32_t drop_s = DROP ? drop_seed(p.drop) : 0u;
#pragma unroll 1
    for (int c = grp; c < N_SLABS; c += GEMM_EPI_GROUPS) {
      const uint32_t word_in = word_next;
      word_next = mask_word(c + GEMM_EPI_GROUPS);
      uint32_t v[32];
      acc_chunk_row<NT>(acc, c, xp, v);
      if constexpr (OUT16) {
        // bf16 output: a 128-byte staging row holds 64 columns; this 32-column chunk fills 16-byte pieces
        // 4*(c&1) .. +3 of slab c/2.  The aux (ReLU-mask) tile has the same layout and type.
        uint8_t* slab_row = staging + (c >> 1) * (BLOCK_M * 128) + row * 128;
#pragma unroll
        for (int piece = 0; piece < 4; ++piece) {
          uint4* dst = reinterpret_cast<uint4*>(slab_row + ((((c & 1) * 4 + piece) ^ (row & 7)) << 4));
          float o[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int j = piece * 8 + e;
            float x = __uint_as_float(v[j]) * p.alpha;
            if (p.flags & EPI_BIAS) x += bias_s[32 * c + j];
            if (p.flags & EPI_RELU) x = fmaxf(x, 0.0f);
            if constexpr (DROP) {
              const unsigned long long idx = (unsigned long long)(m0 + row) * (unsigned long long)p.atomic_ld + (n0 + 32 * c + j);
              x = drop_keep(idx, drop_s, p.drop.thresh) ? x * p.drop.scale : 0.0f;
            }
            o[e] = x;
          }
          if (has_aux) {                       // bf16 aux: bit 15 clear and non-zero <=> value > 0
            const uint4 a = *dst;
            const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              const uint32_t h = (w[e >> 1] >> ((e & 1) * 16)) & 0xffffu;
              const float av = __uint_as_float(h << 16);
              if (p.flags & EPI_ADD_AUX) o[e] += av;
              if (p.flags & EPI_MASK_AUX) o[e] = av > 0.f ? o[e] : 0.f;
            }
          }
          uint4 pk;
          pk.x = ptx::pack_bf16(o[0], o[1]); pk.y = ptx::pack_bf16(o[2], o[3]);
          pk.z = ptx::pack_bf16(o[4], o[5]); pk.w = ptx::pack_bf16(o[6], o[7]);
          *dst = pk;
        }
        continue;
      }
      uint8_t* slab_row = staging + c * (BLOCK_M * 128) + row * 128;
      if constexpr (!DROP) {
        uint32_t* bits_at = (p.bits && m0 + row < p.M && n0 + 32 * c < p.N)
                                ? p.bits + (long long)(m0 + row) * (p.N >> 5) + ((n0 >> 5) + c) : nullptr;
        if (epi_chunk_dispatch(p.flags, v, slab_row, row, bias_s + 32 * c, p.alpha, bits_at, word_in)) continue;
      }
#pragma unroll
      for (int piece = 0; piece < 8; ++piece) {
        float4* dst = reinterpret_cast<float4*>(slab_row + ((piece ^ (row & 7)) << 4));
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = piece * 4 + e;
          float x = __uint_as_float(v[j]) * p.alpha;
          if (p.flags & EPI_BIAS) x += bias_s[32 * c + j];
          if (p.flags & EPI_RELU) x = fmaxf(x, 0.0f);
          if constexpr (DROP) {
            const unsigned long long idx = (unsigned long long)(m0 + row) * (unsigned long long)p.atomic_ld + (n0 + 32 * c + j);
            x = drop_keep(idx, drop_s, p.drop.thresh) ? x * p.drop.scale : 0.0f;
          }
          o[e] = x;
        }
        if (has_aux) {
          const float4 a = *dst;
          if (p.flags & EPI_ADD_AUX) { o[0] += a.x; o[1] += a.y; o[2] += a.z; o[3] += a.w; }
          if (p.flags & EPI_MASK_AUX) {
            o[0] = a.x > 0.f ? o[0] : 0.f; o[1] = a.y > 0.f ? o[1] : 0.f;
            o[2] = a.z > 0.f ? o[2] : 0.f; o[3] = a.w > 0.f ? o[3] : 0.f;
          }
        }
        if (split) {
          // this split's slot of the weight gradient (summed over the splits in order by DetParts::finish)
          const int gm = m0 + row, gn = n0 + 32 * c + piece * 4;
          if (gm < p.M && gn < p.N) {
            float* dstg = p.atomic_out + (long long)blockIdx.z * p.M * p.atomic_ld + (long long)gm * p.atomic_ld + gn;
            if (gn + 3 < p.N && (p.atomic_ld & 3) == 0) {
              *reinterpret_cast<float4*>(dstg) = make_float4(o[0], o[1], o[2], o[3]);
            } else {
#pragma unroll
              for (int e = 0; e < 4; ++e)
                if (gn + e < p.N) dstg[e] = o[e];
            }
          }
        } else {
          *dst = make_float4(o[0], o[1], o[2], o[3]);
        }
      }
    }
    if (!split) {
      ptx::fence_proxy_async_smem();
      ptx::named_bar_sync(1, GEMM_EPI_THREADS);
      if (et == 0) {
        for (int c = 0; c < OUT_SLABS; ++c)
          ptx::tma_store_4d(&tmC, staging + c * (BLOCK_M * 128), n0 + OUT_COLS * c, m0, b2 * p.c_b2, b3 * p.c_b3);
        ptx::tma_store_commit();
      }
      if ((p.flags & EPI_COLSUM) && et < BLOCK_N && n0 + et < p.N) {
        // bias gradient fused into the epilogue: thread = output column, walks the 128 staged rows (conflict-free
        // under the 128B swizzle).  Rows past M hold exact zeros (zero-filled operands / mask tile).  A bf16 output
        // is summed as staged (bf16-rounded terms, fp32 sum).
        float t = 0.f;
        if constexpr (OUT16) {
          const uint8_t* slab = staging + (et >> 6) * (BLOCK_M * 128);
          const int cc = et & 63;
#pragma unroll 8
          for (int r = 0; r < BLOCK_M; ++r) {
            const uint16_t hv = *reinterpret_cast<const uint16_t*>(slab + r * 128 + ((((cc >> 3) ^ (r & 7)) << 4) | ((cc & 7) << 1)));
            t += __uint_as_float(uint32_t(hv) << 16);
          }
        } else {
          const uint8_t* slab = staging + (et >> 5) * (BLOCK_M * 128);
          const int cc = et & 31;
#pragma unroll 8
          for (int r = 0; r < BLOCK_M; ++r)
            t += *reinterpret_cast<const float*>(slab + r * 128 + ((((cc >> 2) ^ (r & 7)) << 4) | ((cc & 3) << 2)));
        }
        p.colsum_out[((long long)blockIdx.z * gridDim.y + blockIdx.y) * p.N + n0 + et] = t;   // this tile's slot
      }
      if (et == 0) ptx::tma_store_wait_read();   // smem may be released once the TMA engine has read it
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ persistent variant
// Same maths and epilogues as gemm_tf32_kernel, restructured as a persistent pipeline: one CTA per SM walks a static
// round-robin list of output tiles; the TMA producer keeps a deep operand ring full ACROSS tile boundaries, so the
// next tile's loads are in flight while the consumer warps run the current tile's epilogue (the non-persistent kernel
// has no loads in flight during its epilogue).
template <int BLOCK_N>
struct PersistLayout {
  static constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 4;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES = BLOCK_N <= 64 ? 6 : 3;
  static constexpr int STAGING_BYTES = BLOCK_M * BLOCK_N * 4;
  static constexpr int RING_BYTES = STAGES * STAGE_BYTES;
  static constexpr int XPOSE_OFF = RING_BYTES + STAGING_BYTES + 512 + BLOCK_N * 4;
  static constexpr int total();
};

constexpr int EPI_GROUPS = 2;                 // consumer groups of four warps (one warp per 32-row quarter)
constexpr int EPI_THREADS = 128 * EPI_GROUPS;
constexpr int PERSIST_THREADS = 64 + EPI_THREADS;
template <int BLOCK_N>
constexpr int PersistLayout<BLOCK_N>::total() { return XPOSE_OFF + (EPI_THREADS / 32) * XPOSE_BYTES + 1024; }

template <int BLOCK_N, int A_MN, int B_MN>
__global__ void __launch_bounds__(PERSIST_THREADS, 1) gemm_tf32_persistent(const __grid_constant__ CUtensorMap tmA,
                                                                        const __grid_constant__ CUtensorMap tmB,
                                                                        const __grid_constant__ CUtensorMap tmC,
                                                                        const __grid_constant__ CUtensorMap tmAux,
                                                                        const GemmParams p, int n_tiles_n,
                                                                        int n_tiles_m, int n_z) {
  using L = PersistLayout<BLOCK_N>;
  constexpr int STAGES = L::STAGES;
  constexpr int N_SLABS = BLOCK_N / 32;
  constexpr int NGA = N_SLABS < EPI_GROUPS ? N_SLABS : EPI_GROUPS;   // active consumer groups
  constexpr int SLABS_PER_GROUP = N_SLABS / NGA;
  constexpr int NT = 4 * SLABS_PER_GROUP;                            // 8-column MMA tiles per warp
  constexpr bool WG = use_wgmma<A_MN, B_MN, false>();
  static_assert(!wgmma_transposed<A_MN, B_MN, false>(), "both operands MN-major: one-tile kernel only");
  static_assert(!WG || 32 * SLABS_PER_GROUP == wg_cols<BLOCK_N>(), "a group's columns are one wgmma instruction wide");
  constexpr int PRODUCER_WARP = EPI_THREADS / 32;                   // after the consumer warps (whole warpgroups)

  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* staging = smem + L::RING_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + L::STAGING_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;        // 4 * NGA consumer-warp arrivals
  uint64_t* aux_full = empty_bar + STAGES;        // aux tile landed in staging
  uint64_t* stage_free = aux_full + 1;            // staging free again (store has read it), one arrival per group
  float* bias_s = reinterpret_cast<float*>(staging + L::STAGING_BYTES + 512);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool split = (p.flags & EPI_ATOMIC) != 0;
  const bool has_aux = (p.flags & (EPI_ADD_AUX | EPI_MASK_AUX)) != 0;
  const bool dev_rows = p.rows_dev != nullptr;     // packed rows: see gemm_tf32_kernel
  if (dev_rows && !split) n_tiles_m = min(n_tiles_m, (__ldg(p.rows_dev) + BLOCK_M - 1) / BLOCK_M);
  const int total_kb = (((dev_rows && split) ? min(p.K, __ldg(p.rows_dev)) : p.K) + BLOCK_K - 1) / BLOCK_K;
  const int kb_per = (dev_rows && split) ? (total_kb + n_z - 1) / n_z : p.kb_per_split;
  const int n_tiles = n_tiles_n * n_tiles_m * n_z;

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    if (!split) ptx::prefetch_tmap(&tmC);
    if (has_aux) ptx::prefetch_tmap(&tmAux);
    for (int s = 0; s < STAGES; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], 4 * NGA); }
    ptx::mbar_init(aux_full, 1);
    ptx::mbar_init(stage_free, NGA);
    ptx::fence_barrier_init();
  }
  arb_pdl_wait();          // everything above overlaps the previous kernel's tail; global memory is touched below
  __syncthreads();

  auto decode = [&](int t, int& n0, int& m0, int& z) {
    const int nt = t % n_tiles_n;
    const int rest = t / n_tiles_n;
    n0 = nt * BLOCK_N;
    m0 = (rest % n_tiles_m) * BLOCK_M;
    z = rest / n_tiles_m;
  };
  auto k_range = [&](int z, int& kb0, int& nkb) {
    if (split) {
      kb0 = z * kb_per;
      nkb = min(total_kb, kb0 + kb_per) - kb0;
      if (nkb < 0) nkb = 0;
    } else {
      kb0 = 0;
      nkb = total_kb;
    }
  };

  if (warp == PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      uint32_t it = 0;          // running k-block counter across tiles (ring position)
      int local = 0;            // tiles processed by this CTA
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++local) {
        int n0, m0, z, kb0, nkb;
        decode(t, n0, m0, z);
        k_range(z, kb0, nkb);
        const int b2 = split ? 0 : z % p.nb2, b3 = split ? 0 : z / p.nb2;
        for (int i = 0; i < nkb; ++i, ++it) {
          const int s = it % STAGES;
          const uint32_t round = it / STAGES;
          if (round > 0) ptx::mbar_wait(&empty_bar[s], (round - 1) & 1);
          load_stage<A_MN, B_MN, false, BLOCK_N>(smem + s * L::STAGE_BYTES, &full_bar[s], &tmA, &tmB, p, m0, n0,
                                                 (kb0 + i) * BLOCK_K, b2, b3);
        }
        if (has_aux) {
          // the residual / mask tile goes into the staging area, which is reused tile after tile: wait until the
          // previous tile's TMA store has read it (issued AFTER this tile's operand loads so the ring never stalls
          // behind the epilogue)
          if (local > 0) ptx::mbar_wait(stage_free, (local - 1) & 1);
          load_aux_tile<BLOCK_N, false>(staging, aux_full, &tmAux, p, m0, n0, b2, b3);
        }
      }
    }
  } else if (warp < PRODUCER_WARP) {
    // ===================== MMA + epilogue (warps 0..7) =====================
    // NGA = min(EPI_GROUPS, slabs) groups of four warps (warpgroups) are active, group g owning the 32-column slabs
    // g * SLABS_PER_GROUP .. +SLABS_PER_GROUP-1 of the tile (mma.sync: each warp 32 rows of them; wgmma: see row).  A group turns a slab registers -> swizzled staging and its leader
    // immediately issues that slab's TMA store; the staging slab is reclaimed lazily (cp.async.bulk.wait_group.read)
    // right before the group writes it again one tile later.  No barrier spans more than the 128 threads of a group.
    const int q = warp & 3;
    const int row = WG ? 64 * (lane >> 4) + 16 * q + (lane & 15) : 32 * q + lane;   // as in gemm_tf32_kernel
    const int grp = warp >> 2;                          // 0 .. EPI_GROUPS-1
    const int gt = threadIdx.x - 128 * grp;             // 0..127 inside the group
    const bool leader = gt == 0;
    float* xp = reinterpret_cast<float*>(smem + L::XPOSE_OFF) + warp * (XPOSE_BYTES / 4);
    if (grp < NGA) {
      uint32_t it = 0;
      int local = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++local) {
        int n0, m0, z, kb0, nkb;
        decode(t, n0, m0, z);
        k_range(z, kb0, nkb);
        const int b2 = split ? 0 : z % p.nb2, b3 = split ? 0 : z / p.nb2;
        ptx::named_bar_sync(1 + grp, 128);            // the group's previous epilogue is done with the bias row
        if (p.flags & EPI_BIAS) {                     // this group's columns only (ordered by the group barriers)
          for (int j = gt; j < 32 * SLABS_PER_GROUP; j += 128) {
            const int col = 32 * (grp * SLABS_PER_GROUP + (j >> 5)) + (j & 31);
            bias_s[col] = (n0 + col < p.N) ? p.bias[n0 + col] : 0.0f;
          }
        }
        // EPI_MASK_BITS: this row's mask words of the group's slabs, fetched before the main loop
        uint32_t mword[2] = {0u, 0u};
        if ((p.flags & EPI_MASK_BITS) && m0 + row < p.M) {
#pragma unroll
          for (int ci = 0; ci < (SLABS_PER_GROUP < 2 ? SLABS_PER_GROUP : 2); ++ci) {
            const int c = grp * SLABS_PER_GROUP + ci;
            if (n0 + 32 * c < p.N) mword[ci] = p.bits[(long long)(m0 + row) * (p.N >> 5) + ((n0 >> 5) + c)];
          }
        }
        float acc[2][NT][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) acc[mt][nt][0] = acc[mt][nt][1] = acc[mt][nt][2] = acc[mt][nt][3] = 0.f;
        for (int i = 0; i < nkb; ++i, ++it) {
          const int s = it % STAGES;
          const uint32_t round = it / STAGES;
          ptx::mbar_wait(&full_bar[s], round & 1);
          uint8_t* a_s = smem + s * L::STAGE_BYTES;
          if constexpr (WG)
            wg_mma_kblock<NT, wg_cols<BLOCK_N>()>(acc, a_s, a_s + A_STAGE_BYTES, 32 * SLABS_PER_GROUP * grp, p.rnd, p.rnd_b,
                                                  1 + grp);
          else warp_mma_kblock<NT, A_MN, B_MN, false>(acc, a_s, a_s + A_STAGE_BYTES, 32 * q, SLABS_PER_GROUP * grp, 1, p.rnd);
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(&empty_bar[s]);
        }
        if (has_aux) ptx::mbar_wait(aux_full, local & 1);
#pragma unroll 1
        for (int ci = 0; ci < SLABS_PER_GROUP; ++ci) {
          const int c = grp * SLABS_PER_GROUP + ci;
          // reclaim the slab: every store this leader committed except the most recent (SLABS_PER_GROUP - 1) ones has
          // been read out of shared memory -- in particular the one that used slab c a tile ago.  With an aux tile
          // the leader already drained its stores before the producer refilled the staging area.
          if (!split && !has_aux && leader && local > 0) {
            if constexpr (SLABS_PER_GROUP == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            else ptx::tma_store_wait_read();
          }
          ptx::named_bar_sync(1 + grp, 128);
          uint32_t v[32];
          acc_chunk_row<NT>(acc, ci, xp, v);
          uint8_t* slab_row = staging + c * (BLOCK_M * 128) + row * 128;
          uint32_t* bits_at = (p.bits && m0 + row < p.M && n0 + 32 * c < p.N)
                                  ? p.bits + (long long)(m0 + row) * (p.N >> 5) + ((n0 >> 5) + c) : nullptr;
          const uint32_t word_in = ci == 0 ? mword[0] : mword[1];
          if (!epi_chunk_dispatch(p.flags, v, slab_row, row, bias_s + 32 * c, p.alpha, bits_at, word_in)) {
          const uint32_t drop_s = (p.flags & EPI_DROPOUT) ? drop_seed(p.drop) : 0u;
#pragma unroll
          for (int piece = 0; piece < 8; ++piece) {
            float4* dst = reinterpret_cast<float4*>(slab_row + ((piece ^ (row & 7)) << 4));
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int j = piece * 4 + e;
              float x = __uint_as_float(v[j]) * p.alpha;
              if (p.flags & EPI_BIAS) x += bias_s[32 * c + j];
              if (p.flags & EPI_RELU) x = fmaxf(x, 0.0f);
              if (p.flags & EPI_DROPOUT) {
                const unsigned long long idx = (unsigned long long)(m0 + row) * (unsigned long long)p.atomic_ld + (n0 + 32 * c + j);
                x = drop_keep(idx, drop_s, p.drop.thresh) ? x * p.drop.scale : 0.0f;
              }
              o[e] = x;
            }
            if (has_aux) {
              const float4 a = *dst;
              if (p.flags & EPI_ADD_AUX) { o[0] += a.x; o[1] += a.y; o[2] += a.z; o[3] += a.w; }
              if (p.flags & EPI_MASK_AUX) {
                o[0] = a.x > 0.f ? o[0] : 0.f; o[1] = a.y > 0.f ? o[1] : 0.f;
                o[2] = a.z > 0.f ? o[2] : 0.f; o[3] = a.w > 0.f ? o[3] : 0.f;
              }
            }
            if (split) {
              const int gm = m0 + row, gn = n0 + 32 * c + piece * 4;
              if (gm < p.M && gn < p.N) {
                float* dstg = p.atomic_out + (long long)z * p.M * p.atomic_ld + (long long)gm * p.atomic_ld + gn;
                if (gn + 3 < p.N && (p.atomic_ld & 3) == 0) {
                  *reinterpret_cast<float4*>(dstg) = make_float4(o[0], o[1], o[2], o[3]);
                } else {
#pragma unroll
                  for (int e = 0; e < 4; ++e)
                    if (gn + e < p.N) dstg[e] = o[e];
                }
              }
            } else {
              *dst = make_float4(o[0], o[1], o[2], o[3]);
            }
          }
          }
          if (!split) {
            ptx::fence_proxy_async_smem();
            ptx::named_bar_sync(1 + grp, 128);
            if (leader) {
              ptx::tma_store_4d(&tmC, staging + c * (BLOCK_M * 128), n0 + 32 * c, m0, b2 * p.c_b2, b3 * p.c_b3);
              ptx::tma_store_commit();
            }
            if (p.flags & EPI_COLSUM) {
              // bias gradient fused into the epilogue: 4 threads per output column, 32 staged rows each (conflict-free
              // under the 128B swizzle), combined by shuffles.  Rows past M hold exact zeros.  The slab is not
              // rewritten before this group's next barrier.
              const int cc = gt >> 2, seg = gt & 3;
              const uint8_t* slab = staging + c * (BLOCK_M * 128);
              float tsum = 0.f;
#pragma unroll 8
              for (int r = 32 * seg; r < 32 * seg + 32; ++r)
                tsum += *reinterpret_cast<const float*>(slab + r * 128 + ((((cc >> 2) ^ (r & 7)) << 4) | ((cc & 3) << 2)));
              tsum += __shfl_xor_sync(0xffffffffu, tsum, 1);
              tsum += __shfl_xor_sync(0xffffffffu, tsum, 2);
              if (seg == 0 && n0 + 32 * c + cc < p.N)      // this tile's slot
                p.colsum_out[((long long)z * ((p.M + BLOCK_M - 1) / BLOCK_M) + m0 / BLOCK_M) * p.N + n0 + 32 * c + cc] = tsum;
            }
          }
        }
        if (!split && has_aux && leader) {     // the producer refills the staging area with the next aux tile
          ptx::tma_store_wait_read();
          ptx::mbar_arrive(stage_free);
        }
      }
      if (!split && leader) ptx::tma_store_wait_read();
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) != cudaSuccess || !sym)
      return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(sym);
  }
  return fn;
}

// MMA operands are rounded fp32 -> tf32 (nearest even) as the kernels load them from shared memory, instead of letting the
// tensor core truncate the mantissa: this removes the systematic bias truncation puts on gradients (DESIGN.md 5).
static int g_round_on_load = 1;
void set_tf32_round_on_load(int enable) { g_round_on_load = enable; }
int tf32_round_on_load() { return g_round_on_load; }

int make_tmap_4d(void* out, const TRef& t, TmapBox box, int unswizzled) {
  EncodeTiledFn enc = get_encode();
  if (!enc) { arb_set_error("cuTensorMapEncodeTiled is not available from this driver"); return ARB_E_CUDA; }
  const int64_t esz = t.bf16 ? 2 : 4;
  const int64_t per16 = 16 / esz;                 // elements per 16 bytes
  cuuint64_t gdim[4], gstride[3];
  cuuint32_t bx[4], estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) { gdim[i] = cuuint64_t(t.dim[i] > 0 ? t.dim[i] : 1); bx[i] = box.b[i]; }
  for (int i = 1; i < 4; ++i) {
    // a broadcast / unused dimension (extent 1) still needs a legal (multiple of 16 B) stride
    int64_t s = t.stride[i];
    if (gdim[i] == 1 && (s <= 0 || (s * esz) % 16 != 0))
      s = int64_t(gdim[0]) * esz >= 16 ? ((int64_t(gdim[0]) + per16 - 1) / per16) * per16 : per16;
    gstride[i - 1] = cuuint64_t(s) * esz;
    if (gstride[i - 1] % 16 != 0) { arb_set_error("tensor map: strides must be multiples of 16 bytes"); return ARB_E_INVALID_ARG; }
  }
  if ((reinterpret_cast<uintptr_t>(t.ptr) & 15) != 0) { arb_set_error("tensor map: base must be 16-byte aligned"); return ARB_E_INVALID_ARG; }
  const CUtensorMapDataType dt = t.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = enc(reinterpret_cast<CUtensorMap*>(out), dt, 4, const_cast<void*>(t.ptr),
                   gdim, gstride, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   unswizzled ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[256];
    std::snprintf(msg, sizeof msg, "cuTensorMapEncodeTiled failed (%d): dim=(%llu,%llu,%llu,%llu) box=(%u,%u,%u,%u)", int(r),
                  (unsigned long long)gdim[0], (unsigned long long)gdim[1], (unsigned long long)gdim[2],
                  (unsigned long long)gdim[3], bx[0], bx[1], bx[2], bx[3]);
    arb_set_error(msg);
    return ARB_E_CUDA;
  }
  return ARB_OK;
}

// launch name for the per-kernel profile table: shape, operand layouts and what the epilogue does
static void gemm_prof_name(char (&out)[56], const GemmDesc& d, const char* variant) {
  const char* kind = (d.flags & EPI_ATOMIC) ? "wgrad" : (d.nb2 * d.nb3 > 1 ? "batched" : (d.b_mn || d.dgrad ? "dgrad" : "fwd"));
  std::snprintf(out, sizeof out, "gemm_%s%s[%s M%d N%d K%d%s%s%s]", variant, d.A.bf16 ? (d.C.bf16 ? "_bf16o" : "_bf16") : "",
                kind, d.M, d.N, d.K, (d.flags & EPI_RELU) ? " relu" : "", (d.flags & EPI_ADD_AUX) ? " +res" : "",
                (d.flags & EPI_MASK_AUX) ? " mask" : "");
}

// accounting only: a launch over packed rows (rows_dev) processes arb_row_frac() of its nominal M (or K, split-K)
static double live_m(const GemmDesc& d) { return double(d.M) * ((d.rows_dev && !(d.flags & EPI_ATOMIC)) ? arb_row_frac() : 1.0); }
static double live_k(const GemmDesc& d) { return double(d.K) * ((d.rows_dev && (d.flags & EPI_ATOMIC)) ? arb_row_frac() : 1.0); }
// the profile record of one GEMM launch: 2 M N K flops per batch; bytes: both operands once, the output and any aux
// tile, at their element sizes
static ProfScope gemm_prof(const GemmDesc& d, const char* variant, cudaStream_t st) {
  const double nb = double(d.nb2) * double(d.nb3), dM = live_m(d), dK = live_k(d);
  const double isz = d.A.bf16 ? 2.0 : 4.0, osz = d.C.bf16 ? 2.0 : 4.0;
  const double has_x = (d.flags & (EPI_ADD_AUX | EPI_MASK_AUX)) ? 1.0 : 0.0;
  char pname[56];
  gemm_prof_name(pname, d, variant);
  return ProfScope(ARB_PROF_GEMM, 2.0 * dM * double(d.N) * dK * nb, st,
                   nb * (isz * (dM * dK + double(d.N) * dK) + osz * (1.0 + has_x) * dM * d.N), pname);
}
static int g_persistent = ARB_DEFAULT_GEMM_PERSISTENT;   // 0: never, 1: wherever supported, 2: auto
void set_gemm_persistent(int on) { g_persistent = on; }

template <int BLOCK_N, int A_MN, int B_MN>
static int launch_persistent_t(const GemmDesc& d, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC,
                               const CUtensorMap& tX, const GemmParams& p, dim3 tiles, cudaStream_t st) {
  const long long n_tiles = (long long)tiles.x * tiles.y * tiles.z;
  const int grid = int(std::min<long long>(n_tiles, sm_count()));
  const ProfScope ps = gemm_prof(d, "persist", st);
  return launch(gemm_tf32_persistent<BLOCK_N, A_MN, B_MN>, dim3(grid), dim3(PERSIST_THREADS),
                PersistLayout<BLOCK_N>::total(), st, /*pdl=*/true, tA, tB, tC, tX, p, int(tiles.x), int(tiles.y),
                int(tiles.z));
}

// bf16 operands (mma m16n8k16): the one-tile-per-CTA kernel; 4-stage ring for the split-K weight gradients, else 3 stages
// (a k-block is 64 elements, so K = 256 is four blocks); fp32 or bf16 output.
template <int BLOCK_N, int A_MN, int B_MN>
static int launch_bf16_t(const GemmDesc& d, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC,
                         const CUtensorMap& tX, const GemmParams& p, dim3 grid, cudaStream_t st) {
  constexpr bool WGRAD = (A_MN == 1 && B_MN == 1);
  const bool drop = (p.flags & EPI_DROPOUT) != 0;   // (K-major operands only: launch_gemm_tf32)
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, GemmParams) = nullptr;
  int smem = 0;
  if constexpr (WGRAD) {
    kern = gemm_tf32_kernel<BLOCK_N, 1, 1, false, 4, true, false>; smem = SmemLayout<BLOCK_N, 4>::total();
  } else if constexpr (BLOCK_N >= 64) {
    constexpr bool CAN_DROP = (A_MN == 0 && B_MN == 0);
    if (d.C.bf16) {
      if (drop) kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, CAN_DROP, 3, true, true>;
      else      kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, false, 3, true, true>;
    } else {
      if (drop) kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, CAN_DROP, 3, true, false>;
      else      kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, false, 3, true, false>;
    }
    smem = SmemLayout<BLOCK_N, 3>::total();
  }
  if (!kern) { arb_set_error("gemm_bf16: block_n must be 64 or 128"); return ARB_E_UNSUPPORTED; }
  const ProfScope ps = gemm_prof(d, "tile", st);
  return launch(kern, grid, dim3(GEMM_THREADS), smem, st, /*pdl=*/true, tA, tB, tC, tX, p);
}

template <int BLOCK_N, int A_MN, int B_MN>
static int launch_t(const GemmDesc& d, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tC,
                    const CUtensorMap& tX, const GemmParams& p, dim3 grid, cudaStream_t st) {
  if (d.A.bf16) return launch_bf16_t<BLOCK_N, A_MN, B_MN>(d, tA, tB, tC, tX, p, grid, st);
  // Mode 1: the persistent pipeline for every shape it supports, i.e. all but those with both operands MN-major, which
  // always take the one-tile kernel (its K-major rewrite for wgmma).
  // Mode 2 (default): the persistent pipeline for every unbatched, non-split shape EXCEPT short-K products with a
  // residual / mask tile, whose aux load it can only issue once the previous tile's stores have left the staging area.
  // Mode 3 (measurement): as 2, but the short-K products with an aux tile go to the persistent kernel too (under packed
  // rows half of a one-tile grid are CTAs of dead tiles that only exit; the persistent kernel has none).
  constexpr bool WGRAD = (A_MN == 1 && B_MN == 1);
  if constexpr (!WGRAD) {
    const bool has_aux_tile = (p.flags & (EPI_ADD_AUX | EPI_MASK_AUX)) != 0;
    const bool pick = !(p.flags & EPI_ATOMIC) && d.nb2 == 1 && d.nb3 == 1 &&
                      (d.K >= 256 || !has_aux_tile || g_persistent == 3);
    if (g_persistent == 1 || (g_persistent >= 2 && pick))
      return launch_persistent_t<BLOCK_N, A_MN, B_MN>(d, tA, tB, tC, tX, p, grid, st);
  }
  // dropout epilogue is a separate instantiation (forward linears only) so the common path carries no mask code;
  // ring depth: 4 stages for the long split-K loops of the weight gradients (1 CTA/SM), 3 for K >= 256
  // (2 CTAs/SM), 2 for the short contractions (3-4 CTAs/SM)
  constexpr bool CAN_DROP = (A_MN == 0 && B_MN == 0);
  const bool drop = (p.flags & EPI_DROPOUT) != 0;   // (K-major operands only: launch_gemm_tf32)
  const bool deep = !WGRAD && d.K >= 256;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, GemmParams);
  int smem;
  if constexpr (WGRAD) {
    kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, false, 4>; smem = SmemLayout<BLOCK_N, 4, true>::total();
  } else if (drop) {
    if (deep) { kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, CAN_DROP, 3>; smem = SmemLayout<BLOCK_N, 3>::total(); }
    else      { kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, CAN_DROP, 2>; smem = SmemLayout<BLOCK_N, 2>::total(); }
  } else {
    if (deep) { kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, false, 3>; smem = SmemLayout<BLOCK_N, 3>::total(); }
    else      { kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, false, 2>; smem = SmemLayout<BLOCK_N, 2>::total(); }
  }
  const ProfScope ps = gemm_prof(d, "tile", st);
  return launch(kern, grid, dim3(GEMM_THREADS), smem, st, /*pdl=*/true, tA, tB, tC, tX, p);
}

int launch_gemm_tf32(const GemmDesc& d, cudaStream_t st) {
  if (d.M <= 0 || d.N <= 0 || d.K < 0) { arb_set_error("gemm_tf32: bad shape"); return ARB_E_INVALID_ARG; }
  if (d.block_n != 32 && d.block_n != 64 && d.block_n != 128) { arb_set_error("gemm_tf32: block_n must be 32/64/128"); return ARB_E_INVALID_ARG; }
  const bool split = (d.flags & EPI_ATOMIC) != 0;
  if (split && (d.nb2 != 1 || d.nb3 != 1 || !d.atomic_out)) { arb_set_error("gemm_tf32: split-K needs an unbatched problem and atomic_out"); return ARB_E_INVALID_ARG; }
  if (!split && d.split_k != 1) { arb_set_error("gemm_tf32: split_k > 1 needs EPI_ATOMIC"); return ARB_E_INVALID_ARG; }
  const bool in16 = d.A.bf16 != 0, out16 = d.C.bf16 != 0;
  if ((d.B.bf16 != 0) != in16) { arb_set_error("gemm: A and B must have the same element type"); return ARB_E_INVALID_ARG; }
  if (out16 && (!in16 || split || d.block_n < 64)) { arb_set_error("gemm: a bf16 output needs bf16 operands, no split-K and block_n >= 64"); return ARB_E_INVALID_ARG; }
  if ((d.flags & (EPI_ADD_AUX | EPI_MASK_AUX)) && (d.Aux.bf16 != 0) != out16) { arb_set_error("gemm: the aux tile must have the output's element type"); return ARB_E_INVALID_ARG; }
  if (in16 && d.block_n < 64) { arb_set_error("gemm: bf16 operands need block_n >= 64 (a 128-byte row holds 64 elements)"); return ARB_E_INVALID_ARG; }
  if (in16 && (d.nb2 != 1 || d.nb3 != 1)) { arb_set_error("gemm: bf16 operands serve the unbatched linears only"); return ARB_E_UNSUPPORTED; }
  // (the bf16 kernel for two MN-major operands is the weight gradients' and stages an fp32 tile only)
  if (out16 && d.a_mn && d.b_mn) { arb_set_error("gemm: a bf16 output needs a K-major operand"); return ARB_E_UNSUPPORTED; }
  const uint32_t kel = in16 ? 64u : 32u;          // K elements per 128-byte row
  const uint32_t ocol = out16 ? 64u : 32u;        // output columns per 128-byte staging row
  alignas(64) CUtensorMap tA, tB, tC, tX;
  int rc;
  if ((rc = make_tmap_4d(&tA, d.A, d.a_mn ? TmapBox{{kel, kel, 1, 1}} : TmapBox{{kel, 128, 1, 1}}, 0))) return rc;
  if ((rc = make_tmap_4d(&tB, d.B, d.b_mn ? TmapBox{{kel, kel, 1, 1}} : TmapBox{{kel, uint32_t(d.block_n), 1, 1}}, 0))) return rc;
  if (!split) {
    if ((rc = make_tmap_4d(&tC, d.C, TmapBox{{ocol, 128, 1, 1}}, 0))) return rc;
  } else {
    tC = tA;
  }
  if (d.flags & (EPI_ADD_AUX | EPI_MASK_AUX)) {
    if ((rc = make_tmap_4d(&tX, d.Aux, TmapBox{{ocol, 128, 1, 1}}, 0))) return rc;
  } else {
    tX = tA;
  }
  const int total_kb = (d.K + int(kel) - 1) / int(kel);
  const int splits = split ? std::max(1, std::min(d.split_k, total_kb)) : 1;
  GemmParams p;
  p.M = d.M; p.N = d.N; p.K = d.K; p.nb2 = d.nb2;
  p.a_b2 = d.a_b2; p.a_b3 = d.a_b3; p.b_b2 = d.b_b2; p.b_b3 = d.b_b3; p.c_b2 = d.c_b2; p.c_b3 = d.c_b3;
  p.flags = d.flags; p.alpha = d.alpha; p.bias = d.bias; p.atomic_out = d.atomic_out; p.atomic_ld = int(d.atomic_ld);
  p.drop = d.drop;
  p.colsum_out = d.colsum_out;
  p.rows_dev = d.rows_dev;
  p.bits = d.bits;
  p.rnd = g_round_on_load;
  p.rnd_b = g_round_on_load && !d.b_tf32;
  if (d.flags & (EPI_RELU_BITS | EPI_MASK_BITS)) {
    if (!d.bits || d.N % 32 || out16 || split || d.nb2 != 1 || d.nb3 != 1 || (d.flags & (EPI_DROPOUT | EPI_ADD_AUX | EPI_MASK_AUX)) ||
        ((d.flags & EPI_RELU_BITS) && !(d.flags & EPI_RELU))) {
      arb_set_error("gemm: the ReLU bit mask needs an unbatched fp32 output with N % 32 == 0, no dropout and no aux tile");
      return ARB_E_INVALID_ARG;
    }
    const int core = d.flags & ~EPI_COLSUM;
    if (core != (EPI_BIAS | EPI_RELU | EPI_RELU_BITS) && core != EPI_MASK_BITS && !((core == (EPI_RELU | EPI_RELU_BITS)) && d.bias)) {
      arb_set_error("gemm: the ReLU bit mask serves bias + ReLU (forward) and the plain mask (backward) only");
      return ARB_E_INVALID_ARG;
    }
  }
  if (d.rows_dev && (d.nb2 != 1 || d.nb3 != 1)) { arb_set_error("gemm: a device-side row count serves unbatched launches only"); return ARB_E_INVALID_ARG; }
  if ((d.flags & EPI_COLSUM) && (!d.colsum_out || split)) { arb_set_error("gemm_tf32: EPI_COLSUM needs colsum_out and a non-split launch"); return ARB_E_INVALID_ARG; }
  if ((d.flags & EPI_DROPOUT) && d.drop.thresh == 0) p.flags &= ~EPI_DROPOUT;
  // (checked here, before the kernel is picked: the persistent kernel would otherwise take what the one-tile one refuses)
  if ((p.flags & EPI_DROPOUT) && (d.a_mn || d.b_mn)) { arb_set_error("gemm: the dropout epilogue needs K-major operands"); return ARB_E_UNSUPPORTED; }
  if (p.flags & EPI_DROPOUT) {
    if ((p.flags & EPI_ATOMIC) || d.drop_n < 0 || d.drop_n > d.N) {
      arb_set_error("gemm: the dropout epilogue needs a plain output and 0 <= drop_n <= N"); return ARB_E_INVALID_ARG;
    }
    p.atomic_ld = d.drop_n ? d.drop_n : d.N;
  }
  p.kb_per_split = (total_kb + splits - 1) / splits;
  const int eff_splits = split ? (total_kb + p.kb_per_split - 1) / std::max(1, p.kb_per_split) : 1;
  dim3 grid((d.N + d.block_n - 1) / d.block_n, (d.M + BLOCK_M - 1) / BLOCK_M, split ? std::max(1, eff_splits) : d.nb2 * d.nb3);
  int (*launch)(const GemmDesc&, const CUtensorMap&, const CUtensorMap&, const CUtensorMap&, const CUtensorMap&,
                const GemmParams&, dim3, cudaStream_t) = nullptr;
#define ARB_GEMM_CASE(BN, AM, BM) \
  if (d.block_n == BN && d.a_mn == AM && d.b_mn == BM) launch = launch_t<BN, AM, BM>;
  ARB_GEMM_CASE(32, 0, 0) ARB_GEMM_CASE(32, 0, 1) ARB_GEMM_CASE(32, 1, 0) ARB_GEMM_CASE(32, 1, 1)
  ARB_GEMM_CASE(64, 0, 0) ARB_GEMM_CASE(64, 0, 1) ARB_GEMM_CASE(64, 1, 0) ARB_GEMM_CASE(64, 1, 1)
  ARB_GEMM_CASE(128, 0, 0) ARB_GEMM_CASE(128, 0, 1) ARB_GEMM_CASE(128, 1, 0) ARB_GEMM_CASE(128, 1, 1)
#undef ARB_GEMM_CASE
  if (!launch) { arb_set_error("gemm_tf32: unsupported configuration"); return ARB_E_UNSUPPORTED; }
  // split-K partial tiles and the per-tile bias-gradient column sums go to slots that are summed in order afterwards
  DetParts dp;
  if (p.flags & EPI_COLSUM) dp.add(p.colsum_out, (long long)grid.z * grid.y, 1, d.N, d.N);
  if (split) dp.add(p.atomic_out, grid.z, d.M, d.N, d.atomic_ld);
  if ((rc = dp.begin(st))) return rc;
  if (split) p.atomic_ld = d.N;       // slot row pitch
  if ((rc = launch(d, tA, tB, tC, tX, p, grid, st))) return rc;
  return dp.finish(st);
}

}  // namespace arb

// ------------------------------------------------------------------------------------------------ C ABI (unit-test / building-block entry)
// C[b][M,N] = epilogue(alpha * A[b] op B[b]) on plain row-major fp32 matrices.
//   a_mn = 0: A is [M,K] row-major;  a_mn = 1: A is stored transposed, [K,M] row-major.
//   b_mn = 0: B is [N,K] row-major (an nn.Linear weight);  b_mn = 1: B is [K,N] row-major.
//   batch > 1: operands are `batch` consecutive matrices (stride = rows*cols), unless the stride argument is 0.
extern "C" void arb_set_tf32_round_on_load(int32_t enable) { arb::set_tf32_round_on_load(enable); }
extern "C" void arb_set_gemm_persistent(int32_t on) { arb::set_gemm_persistent(on); }

extern "C" int32_t arb_gemm_tf32(const float* A, const float* B, float* C, const float* aux, const float* bias,
                                 int32_t M, int32_t N, int32_t K, int32_t a_mn, int32_t b_mn, int32_t batch,
                                 int64_t a_bstride, int64_t b_bstride, int64_t c_bstride, int32_t block_n,
                                 int32_t flags, float alpha, int32_t split_k, void* stream) {
  using namespace arb;
  if (!A || !B || !C) { arb_set_error("arb_gemm_tf32: null pointer"); return ARB_E_INVALID_ARG; }
  GemmDesc d;
  d.M = M; d.N = N; d.K = K; d.a_mn = a_mn; d.b_mn = b_mn; d.block_n = block_n; d.flags = flags; d.alpha = alpha;
  d.bias = bias; d.nb2 = batch; d.nb3 = 1; d.split_k = split_k;
  d.a_b2 = a_bstride != 0; d.b_b2 = b_bstride != 0; d.c_b2 = c_bstride != 0;
  auto mat = [](const float* p, int64_t inner, int64_t rows, int64_t nb, int64_t bstride) {
    TRef t; t.ptr = p; t.dim[0] = inner; t.dim[1] = rows; t.dim[2] = bstride ? nb : 1; t.dim[3] = 1;
    t.stride[0] = 1; t.stride[1] = inner; t.stride[2] = bstride; t.stride[3] = 0; return t;
  };
  d.A = a_mn ? mat(A, M, K, batch, a_bstride) : mat(A, K, M, batch, a_bstride);
  d.B = b_mn ? mat(B, N, K, batch, b_bstride) : mat(B, K, N, batch, b_bstride);
  d.C = mat(C, N, M, batch, c_bstride);
  if (aux) d.Aux = mat(aux, N, M, batch, c_bstride);
  if (flags & EPI_ATOMIC) { d.atomic_out = C; d.atomic_ld = N; }
  return launch_gemm_tf32(d, static_cast<cudaStream_t>(stream));
}

// The same building block with bf16 operands (tensor-core m16n8k16, fp32 accumulation): A, B are bfloat16 matrices in the
// layouts described above; C (and aux, if given) is bfloat16 when out_bf16 != 0, else fp32.  With EPI_ATOMIC
// (split-K) C must be fp32 and is accumulated into.
extern "C" int32_t arb_gemm_bf16(const void* A, const void* B, void* C, const void* aux, const float* bias, int32_t M,
                                 int32_t N, int32_t K, int32_t a_mn, int32_t b_mn, int32_t block_n, int32_t flags,
                                 float alpha, int32_t split_k, int32_t out_bf16, float* colsum_out, void* stream) {
  using namespace arb;
  if (!A || !B || !C) { arb_set_error("arb_gemm_bf16: null pointer"); return ARB_E_INVALID_ARG; }
  GemmDesc d;
  d.M = M; d.N = N; d.K = K; d.a_mn = a_mn; d.b_mn = b_mn; d.block_n = block_n; d.flags = flags; d.alpha = alpha;
  d.bias = bias; d.split_k = split_k; d.colsum_out = colsum_out;
  auto mat = [](const void* p, int64_t inner, int64_t rows, int is16) {
    TRef t; t.ptr = p; t.dim[0] = inner; t.dim[1] = rows; t.stride[0] = 1; t.stride[1] = inner; t.bf16 = is16; return t;
  };
  d.A = a_mn ? mat(A, M, K, 1) : mat(A, K, M, 1);
  d.B = b_mn ? mat(B, N, K, 1) : mat(B, K, N, 1);
  d.C = mat(C, N, M, out_bf16 != 0);
  if (aux) d.Aux = mat(aux, N, M, out_bf16 != 0);
  if (flags & EPI_ATOMIC) { d.atomic_out = static_cast<float*>(C); d.atomic_ld = N; }
  return launch_gemm_tf32(d, static_cast<cudaStream_t>(stream));
}

// The whole descriptor, copied field for field: the tests launch exactly what the scorer's helpers build.
extern "C" int32_t arb_gemm_launch(const arb_gemm_desc* in, void* stream) {
  using namespace arb;
  if (!in) { arb_set_error("arb_gemm_launch: null descriptor"); return ARB_E_INVALID_ARG; }
  auto view = [](const arb_gemm_view& v) {
    TRef t; t.ptr = v.ptr; t.bf16 = v.bf16;
    for (int i = 0; i < 4; ++i) { t.dim[i] = v.dim[i]; t.stride[i] = v.stride[i]; }
    return t;
  };
  GemmDesc d;
  d.M = in->M; d.N = in->N; d.K = in->K;
  d.a_mn = in->a_mn; d.b_mn = in->b_mn; d.b_tf32 = in->b_tf32; d.dgrad = in->dgrad;
  d.A = view(in->A); d.B = view(in->B); d.C = view(in->C); d.Aux = view(in->aux);
  d.nb2 = in->nb2; d.nb3 = in->nb3;
  d.a_b2 = in->a_b2; d.a_b3 = in->a_b3; d.b_b2 = in->b_b2; d.b_b3 = in->b_b3; d.c_b2 = in->c_b2; d.c_b3 = in->c_b3;
  d.block_n = in->block_n; d.split_k = in->split_k; d.flags = in->flags; d.alpha = in->alpha;
  d.bias = in->bias; d.atomic_out = in->atomic_out; d.atomic_ld = in->atomic_ld;
  d.drop = DropSite{in->drop_seed, in->drop_thresh, in->drop_scale, in->drop_key, in->drop_call_seed};
  d.colsum_out = in->colsum_out; d.bits = in->bits; d.rows_dev = in->rows_dev;
  return launch_gemm_tf32(d, static_cast<cudaStream_t>(stream));
}
