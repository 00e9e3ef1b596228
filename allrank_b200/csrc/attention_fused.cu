// Fused self-attention core for slates of up to 256 items (head widths 4 ... 32 and 64):
//   ctx = softmax(mask(Q K^T / sqrt(dk))) V
// in ONE kernel, the [S,S] score / probability tile living only in registers.
//
// Reference: attention() allrank/models/transformer.py:137-156 (+ the head split / concat of
// MultiHeadedAttention.forward :193-202, which here are just TMA coordinates).
//
// Nothing of size S^2 touches HBM or shared memory: per (slate, head) the kernel reads 3*S*dk*4 bytes and writes
// S*dk*4 (+ 8*S of softmax statistics for the backward pass) -- versus ~5*S^2*4 bytes for the unfused sequence.
// See attn_fwd_kernel for the organisation.
#include <algorithm>
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "attention_frag.cuh"
#include "attention_fused.h"
#include "block_utils.cuh"
#include "common.h"
#include "sm90_ptx.cuh"

namespace arb {

constexpr int FWD_WARPS = 8;                          // compute warps: one 16-query strip at a time each
constexpr int FWD_THREADS = 32 * (FWD_WARPS + 1);     // + one load warp

template <int DK>
struct FwdSmem {
  static constexpr int NKB = (DK + 31) / 32;           // 32-column slabs of the head (one 128-byte row each)
  static constexpr int STAGE_BYTES = NKB * 16 * 128;   // one warp's output strip: [slab][16 rows][128 B]
  // [operand pool: pool_units rows of 128 B] [output staging: one strip per compute warp] [key bits: 2 slots x 8 words]
  // [mbarriers: full[2], ready[2], empty[2]]
  __host__ __device__ static int stage_off(int pool_units) { return pool_units * 128; }
  __host__ __device__ static int bits_off(int pool_units) { return stage_off(pool_units) + FWD_WARPS * STAGE_BYTES; }
  __host__ __device__ static int bars_off(int pool_units) { return bits_off(pool_units) + 64; }
  __host__ __device__ static int total(int pool_units) { return bars_off(pool_units) + 64 + 1024; }
};

// One CTA per SM walks the (slate, head) items blockIdx.x, blockIdx.x + gridDim.x, ... (head-fastest, as the
// backward).  The last warp loads: an item's Q rows and its K, V rows below round_up(extent, 16) go by TMA in 16-row
// boxes into an operand pool that holds two items (even items of the CTA from its bottom, odd ones from its top).  The
// next item's loads go out as soon as the previous user of its pool slot is done, and -- when the two items do not fit
// side by side -- the current one too.  Once an item has landed, the load warp rounds it to tf32 in place, sets its key
// bits and marks it ready (mbarrier ready[slot]).
//
// The work unit is one 16-query strip over every key below the extent, run by one compute warp.  The strips of the
// CTA's items form one sequence dealt round-robin to the eight compute warps, so a warp that has no strip left in an
// item goes on with the next item's strips as soon as that item is ready; a pool slot is free again once every compute
// warp has arrived on empty[slot].  A warp runs its strip on the tensor cores (mma.sync m16n8k8 tf32):
//   pass A  S = Q K^T, one 8-key block at a time, keeping only the masked row maximum;
//   pass B  the same blocks again: P = exp2((S - max) / sqrt(dk) * log2 e) (key mask, dropout), rounded to tf32 and
//           fed straight from the accumulator registers into O += P V (key order sigma8: no shuffles).
// It then stages O * (1 / rowsum) and TMA-stores it as a 16-row box.
// Packed rows (pack_off != nullptr): the activations hold only the first round_up(extent, 16) rows of every slate,
// slate b starting at row pack_off[b] of one long [rows, h, dk] tensor (TMA coordinates (.., row, head, 0)); exactly
// those rows are loaded and stored, and an empty slate is skipped.  Dense layout: every query row below
// round_up(S, 16) is computed (padded items get the reference's scores) and stored up to S.
template <int DK, bool DROP, bool OUT16 = false>
__global__ void __launch_bounds__(FWD_THREADS, 1) attn_fwd_kernel(
    const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmO, const uint8_t* __restrict__ mask,
    float* __restrict__ stat_max, float* __restrict__ stat_sum, int S, int n_heads, float scale_log2e, DropSite drop,
    const int* __restrict__ extent, const int* __restrict__ pack_off, int n_items, int rnd, int pool_units) {
  using L = FwdSmem<DK>;
  constexpr int NKB = L::NKB;
  constexpr int KSB = DK / 8 / NKB;          // k8 steps per slab
  static_assert(!OUT16 || DK <= 32, "bf16 context: one 64-byte row per query");
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t sbase = (ptx::smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* smem = smem_dyn + (sbase - ptx::smem_u32(smem_dyn));
  uint8_t* stage = smem + L::stage_off(pool_units);
  const uint32_t stage_s = sbase + L::stage_off(pool_units);
  uint32_t* key_bits = reinterpret_cast<uint32_t*>(smem + L::bits_off(pool_units));   // [slot][8]: bit j of word w = key 32w + j is real
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::bars_off(pool_units));
  uint64_t* ready = full + 2;
  uint64_t* empty = full + 4;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const bool packed = pack_off != nullptr;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ); ptx::prefetch_tmap(&tmK); ptx::prefetch_tmap(&tmV); ptx::prefetch_tmap(&tmO);
    for (int s = 0; s < 2; ++s) {
      ptx::mbar_init(full + s, 1);
      ptx::mbar_init(ready + s, 32);
      ptx::mbar_init(empty + s, FWD_WARPS);
    }
    ptx::fence_barrier_init();
  }
  arb_pdl_wait();
  __syncthreads();

  // Keys at or beyond the slate's extent are all masked (probability exactly 0): the products, the softmax and the
  // K / V loads stop at round_up(extent, 16).  At least one key block is always processed, so an all-padded slate in
  // the dense layout still produces the reference's NaN rows.
  struct Item {
    int b, head, kext, krows, qrows, row_base, bc;
    __device__ int units() const { return NKB * (qrows + 2 * krows); }   // 128-byte pool rows: Q, K, V slabs
  };
  auto item_info = [&](int item) {
    Item it{};
    it.b = item / n_heads;
    it.head = item - it.b * n_heads;
    int e = extent ? __ldg(extent + it.b) : S;
    if (packed && e <= 0) return it;            // packed rows: an empty slate holds no rows (qrows = 0: skipped)
    e = max(1, min(S, e));
    it.kext = e;
    it.krows = (e + 15) & ~15;
    it.qrows = packed ? it.krows : ((S + 15) & ~15);
    it.row_base = packed ? __ldg(pack_off + it.b) : 0;
    it.bc = packed ? 0 : it.b;
    return it;
  };
  auto next_item = [&](int item) {
    while (item < n_items && item_info(item).qrows == 0) item += gridDim.x;
    return item;
  };
  // pool offset (bytes) of an item's rows: slot 0 from the bottom, slot 1 from the top; Q slabs, then K, then V
  auto region_off = [&](int slot, int units) { return slot ? (pool_units - units) * 128 : 0; };

  if (warp == FWD_WARPS) {
    // ===== load warp
    auto issue_loads = [&](const Item& it, int slot) {
      uint8_t* region = smem + region_off(slot, it.units());
      ptx::fence_proxy_async_smem();
      if (lane == 0) ptx::mbar_expect_tx(full + slot, uint32_t(it.units()) * 128u);
      __syncwarp();
      const int nq = it.qrows >> 4, nk = it.krows >> 4, nb = nq + 2 * nk;   // 16-row boxes per slab
      for (int j = lane; j < NKB * nb; j += 32) {
        const int kb = j / nb, i = j - kb * nb;
        if (i < nq) {
          ptx::tma_load_4d(region + (kb * it.qrows + 16 * i) * 128, &tmQ, full + slot, 32 * kb, it.row_base + 16 * i, it.head, it.bc);
        } else {
          const int v = i >= nq + nk, r = 16 * (i - nq - v * nk);
          ptx::tma_load_4d(region + (NKB * (it.qrows + v * it.krows) + kb * it.krows + r) * 128, v ? &tmV : &tmK,
                           full + slot, 32 * kb, it.row_base + r, it.head, it.bc);
        }
      }
    };
    // once the item has landed: round it to tf32 in place (nearest even, as the products would on each use), set its
    // key bits, mark it ready (every lane arrives after its own stores)
    auto prepare = [&](const Item& it, int slot, uint32_t parity) {
      uint8_t mk[8];
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const int key = 32 * w + lane;
        mk[w] = key < S ? mask[size_t(it.b) * S + key] : uint8_t(1);
      }
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const uint32_t bw = __ballot_sync(FULL, mk[w] == 0);
        if (lane == 0) key_bits[8 * slot + w] = bw;
      }
      ptx::mbar_wait(full + slot, parity);
      if (rnd) {
        uint4* p = reinterpret_cast<uint4*>(smem + region_off(slot, it.units()));
        const int n = it.units() * 8;
#pragma unroll 4
        for (int i = lane; i < n; i += 32) {
          uint4 v = p[i];
          v.x = ptx::cvt_tf32(__uint_as_float(v.x)); v.y = ptx::cvt_tf32(__uint_as_float(v.y));
          v.z = ptx::cvt_tf32(__uint_as_float(v.z)); v.w = ptx::cvt_tf32(__uint_as_float(v.w));
          p[i] = v;
        }
      }
      ptx::mbar_arrive(ready + slot);
    };
    int item = next_item(blockIdx.x);
    if (item >= n_items) return;
    Item cur = item_info(item);
    issue_loads(cur, 0);
    for (int k = 0;; ++k) {
      const int slot = k & 1;
      prepare(cur, slot, (k >> 1) & 1);
      const int nitem = next_item(item + gridDim.x);
      if (nitem >= n_items) break;
      const Item nxt = item_info(nitem);
      // the next item's slot must be free (its previous user, item k - 1, done), and item k done as well when the two
      // items do not fit side by side
      if (k >= 1) ptx::mbar_wait(empty + (slot ^ 1), ((k - 1) >> 1) & 1);
      if (cur.units() + nxt.units() > pool_units) ptx::mbar_wait(empty + slot, (k >> 1) & 1);
      issue_loads(nxt, slot ^ 1);
      cur = nxt;
      item = nitem;
    }
    return;
  }

  // ===== compute warps
  if constexpr (DROP) drop.seed = drop_seed(drop);
  auto strip = [&](const Item& it, uint32_t region, const uint32_t* bits, int s) {
    const int r0 = 16 * s, qA = r0 + g, qB = qA + 8;
    const uint32_t q_s = region, k_s = q_s + NKB * it.qrows * 128, v_s = k_s + NKB * it.krows * 128;
    const uint32_t slab_k = it.krows * 128;
    uint32_t qa[NKB][KSB][4];
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb) ld_a_head<KSB>(q_s + kb * it.qrows * 128, r0, lane, qa[kb]);
    // raw scores of keys 8j + t, 8j + t + 4 for rows qA, qB
    auto scores = [&](int j, float (&s4)[4]) {
      s4[0] = s4[1] = s4[2] = s4[3] = 0.f;
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb) {
        uint32_t kf[KSB][2];
        ld_b_head<KSB>(k_s + kb * slab_k, 8 * j, lane, kf);
#pragma unroll
        for (int ks = 0; ks < KSB; ++ks) ptx::mma_tf32(s4, qa[kb][ks], kf[ks]);
      }
    };
    const int nj = (it.kext + 7) >> 3;
    // ---- pass A: masked row maxima
    float mxA = -CUDART_INF_F, mxB = -CUDART_INF_F;
#pragma unroll 2
    for (int j = 0; j < nj; ++j) {
      float s4[4];
      scores(j, s4);
      const uint32_t kw = bits[j >> 2] >> ((8 * j & 31) + t);     // bit 0: key 8j + t, bit 4: key 8j + t + 4
      if (kw & 1u) { mxA = fmaxf(mxA, s4[0]); mxB = fmaxf(mxB, s4[2]); }
      if (kw & 16u) { mxA = fmaxf(mxA, s4[1]); mxB = fmaxf(mxB, s4[3]); }
    }
    mxA = fmaxf(mxA, __shfl_xor_sync(FULL, mxA, 1)); mxA = fmaxf(mxA, __shfl_xor_sync(FULL, mxA, 2));
    mxB = fmaxf(mxB, __shfl_xor_sync(FULL, mxB, 1)); mxB = fmaxf(mxB, __shfl_xor_sync(FULL, mxB, 2));
    // ---- pass B: probabilities and O = P V
    const float mxsA = mxA * scale_log2e, mxsB = mxB * scale_log2e;
    const unsigned long long dbase = (unsigned long long)(it.b * n_heads + it.head) * S;
    const bool odd = (t & 1) != 0;
    float sumA = 0.f, sumB = 0.f;
    float o[NKB][KSB][4];
#pragma unroll
    for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
      for (int nt = 0; nt < KSB; ++nt) o[kb][nt][0] = o[kb][nt][1] = o[kb][nt][2] = o[kb][nt][3] = 0.f;
#pragma unroll 2
    for (int j = 0; j < nj; ++j) {
      float s4[4];
      scores(j, s4);
      const uint32_t kw = bits[j >> 2] >> ((8 * j & 31) + t);
      // exp((s - max)/sqrt(dk)) as exp2; padded keys contribute exactly 0.  An all-padded slate gives
      // (-inf) - (-inf) = NaN like the reference (quirk Q2).
      float p[4];
      p[0] = (kw & 1u) ? ex2_approx(fmaf(s4[0], scale_log2e, -mxsA)) : 0.0f;
      p[1] = (kw & 16u) ? ex2_approx(fmaf(s4[1], scale_log2e, -mxsA)) : 0.0f;
      p[2] = (kw & 1u) ? ex2_approx(fmaf(s4[2], scale_log2e, -mxsB)) : 0.0f;
      p[3] = (kw & 16u) ? ex2_approx(fmaf(s4[3], scale_log2e, -mxsB)) : 0.0f;
      // Row sums (softmax normalises BEFORE dropout, transformer.py:153-155), added in the association of a plain
      // fragment layout: quad lane u adds p[8j + 2u] + p[8j + 2u + 1] to its sum.  Here lane t holds keys t, t + 4;
      // exchanging one value with lane t ^ 1 gives lanes 0, 2, 1, 3 the pairs of u = 0, 1, 2, 3.
      const float xA = __shfl_xor_sync(FULL, odd ? p[0] : p[1], 1);
      const float xB = __shfl_xor_sync(FULL, odd ? p[2] : p[3], 1);
      sumA += odd ? xA + p[1] : p[0] + xA;
      sumB += odd ? xB + p[3] : p[2] + xB;
      if constexpr (DROP) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const unsigned long long idx = (dbase + (i < 2 ? qA : qB)) * (unsigned long long)S + (8 * j + t + 4 * (i & 1));
          p[i] = drop_keep(idx, drop.seed, drop.thresh) ? p[i] * drop.scale : 0.0f;
        }
      }
      // the accumulators {rows g, g+8} x {keys t, t+4} are the A fragment over k-slots {t, t+4}
      const uint32_t pa[4] = {__float_as_uint(round_tf32(p[0])), __float_as_uint(round_tf32(p[2])),
                              __float_as_uint(round_tf32(p[1])), __float_as_uint(round_tf32(p[3]))};
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb) {
        uint32_t v0[KSB], v1[KSB];
        ld_b_out<KSB>(v_s + kb * slab_k, 8 * j + t, g, v0);
        ld_b_out<KSB>(v_s + kb * slab_k, 8 * j + t + 4, g, v1);
#pragma unroll
        for (int nt = 0; nt < KSB; ++nt) {
          const uint32_t vb[2] = {v0[nt], v1[nt]};
          ptx::mma_tf32(o[kb][nt], pa, vb);
        }
      }
    }
    // quad lanes 0, 2 hold the pairs of u = 0, 1 and lanes 1, 3 those of u = 2, 3: (s0 + s1) + (s2 + s3)
    sumA += __shfl_xor_sync(FULL, sumA, 2); sumA += __shfl_xor_sync(FULL, sumA, 1);
    sumB += __shfl_xor_sync(FULL, sumB, 2); sumB += __shfl_xor_sync(FULL, sumB, 1);
    if (t == 0) {
      const size_t so = (size_t(it.b) * n_heads + it.head) * S;
      if (qA < S) { stat_max[so + qA] = mxA; stat_sum[so + qA] = sumA; }
      if (qB < S) { stat_max[so + qB] = mxB; stat_sum[so + qB] = sumB; }
    }
    // ---- stage O / rowsum (the warp's previous strip must have been read out) and TMA-store it
    if (lane == 0) ptx::tma_store_wait_read();
    __syncwarp();
    const uint32_t st_w = stage_s + warp * L::STAGE_BYTES;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = g + 8 * h;
      const float inv = 1.0f / (h ? sumB : sumA);
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb) {
        float v[2][KSB];      // v[0]: head columns of output column 2t, v[1]: of 2t + 1 (n-tile order)
#pragma unroll
        for (int nt = 0; nt < KSB; ++nt) { v[0][nt] = o[kb][nt][2 * h] * inv; v[1][nt] = o[kb][nt][2 * h + 1] * inv; }
        if constexpr (OUT16) {
          // bf16 mode: the context only feeds the output projection -- dense bfloat16 rows of 32 columns (64 bytes),
          // unswizzled tensor map
          if constexpr (KSB == 4) {
            sts64(st_w + r * 64 + 8 * t, make_uint2(ptx::pack_bf16(v[0][0], v[0][1]), ptx::pack_bf16(v[0][2], v[0][3])));
            sts64(st_w + r * 64 + 32 + 8 * t, make_uint2(ptx::pack_bf16(v[1][0], v[1][1]), ptx::pack_bf16(v[1][2], v[1][3])));
          } else {
            sts64(st_w + r * 64 + 8 * t, make_uint2(ptx::pack_bf16(v[0][0], v[0][1]), ptx::pack_bf16(v[1][0], v[1][1])));
          }
        } else {
          const uint32_t part = st_w + kb * 2048;
          if constexpr (KSB == 4) {
            sts128(part + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[0][2]), __float_as_uint(v[0][3])));
            sts128(part + ptx::sw128(r, 64 + 16 * t), make_uint4(__float_as_uint(v[1][0]), __float_as_uint(v[1][1]), __float_as_uint(v[1][2]), __float_as_uint(v[1][3])));
          } else {
            sts128(part + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[1][0]), __float_as_uint(v[1][1])));
          }
        }
      }
    }
    ptx::fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      constexpr int OSLABS = OUT16 ? 1 : NKB;
      for (int sl = 0; sl < OSLABS; ++sl)
        ptx::tma_store_4d(&tmO, stage + warp * L::STAGE_BYTES + sl * 2048, 32 * sl, it.row_base + r0, it.head, it.bc);
      ptx::tma_store_commit();
    }
  };

  int k = 0, dealt = 0;     // dealt: strips of the CTA's earlier items
  for (int item = next_item(blockIdx.x); item < n_items; item = next_item(item + gridDim.x), ++k) {
    const Item it = item_info(item);
    const int slot = k & 1, ns = it.qrows >> 4;
    ptx::mbar_wait(ready + slot, (k >> 1) & 1);
    const uint32_t region = sbase + region_off(slot, it.units());
    for (int s = (warp - dealt) & (FWD_WARPS - 1); s < ns; s += FWD_WARPS) strip(it, region, key_bits + 8 * slot, s);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(empty + slot);
    dealt += ns;
  }
  if (lane == 0) ptx::tma_store_wait_all();
}

// Both settings run attn_fwd_kernel; the switch is kept for the C ABI (arb_set_attention_fwd_two_pass).
void set_attn_fwd_two_pass(int) {}

template <int DK>
static int launch_fwd_t(const AttnFwdArgs& a, cudaStream_t st) {
  using L = FwdSmem<DK>;
  alignas(64) CUtensorMap tQ, tK, tV, tO;
  int rc;
  const TmapBox box{{32, 16, 1, 1}};
  if ((rc = make_tmap_4d(&tQ, a.q, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tK, a.k, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tV, a.v, box, 0))) return rc;
  const bool out16 = a.o.bf16 != 0;
  // the bfloat16 head view's head stride (2 w bytes) must be a multiple of 16 bytes for TMA
  if (out16 && (DK > 32 || a.dk % 8)) { arb_set_error("attn_fwd: a bf16 context needs head width 8, 16, 24 or 32"); return ARB_E_UNSUPPORTED; }
  const bool packed = a.pack_off != nullptr;
  if (packed && !a.extent) { arb_set_error("attn_fwd: packed rows need the slate extents"); return ARB_E_UNSUPPORTED; }
  if ((rc = make_tmap_4d(&tO, a.o, box, out16 ? 1 : 0))) return rc;
  const bool drop = a.drop.thresh != 0;
  void (*kern)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, const uint8_t*, float*, float*, int, int, float,
               DropSite, const int*, const int*, int, int, int);
  if constexpr (DK <= 32) {
    if (out16) kern = drop ? attn_fwd_kernel<DK, true, true> : attn_fwd_kernel<DK, false, true>;
    else kern = drop ? attn_fwd_kernel<DK, true> : attn_fwd_kernel<DK, false>;
  } else {
    kern = drop ? attn_fwd_kernel<DK, true> : attn_fwd_kernel<DK, false>;
  }
  // the operand pool holds two items of the largest shape when the 227 KB of shared memory allow it, else one
  const int item_units = L::NKB * 3 * ((a.S + 15) & ~15);
  const int pool_units = std::min(2 * item_units, ((227 * 1024 - L::total(0)) / 128) & ~15);
  if (pool_units < item_units) { arb_set_error("attn_fwd: slate too large for the shared-memory operand pool"); return ARB_E_UNSUPPORTED; }
  // one CTA per SM walking the (slate, head) items head-fastest
  const int n_items = a.h * a.B;
  dim3 grid(std::max(1, std::min(n_items, sm_count())));
  ProfScope ps(ARB_PROF_GEMM, (a.extent ? arb_attn_frac() : 1.0) * 4.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
               (packed ? arb_row_frac() : 1.0) * 4.0 * double(a.B) * a.h * a.S * ((out16 ? 3.5 : 4.0) * a.dk + 2.0),
               "attn_fwd_kernel");
  return launch(kern, grid, dim3(FWD_THREADS), size_t(L::total(pool_units)), st, /*pdl=*/true, tQ, tK, tV, tO, a.mask,
                a.stat_max, a.stat_sum, a.S, a.h, a.scale * 1.4426950408889634f, a.drop, a.extent, a.pack_off, n_items,
                tf32_round_on_load(), pool_units);
}

// attn_fwd_kernel: S <= 256 at head widths 4 ... 32 in steps of 4 and at 64; attention_long.cu: S <= 4096 at 4 ... 256 in
// steps of 4 (every width above 32 but 64 at S <= 256 runs there).  Widths below 16 run on DK 16 and widths 20 ... 28
// on DK 32, as in attention_long.cu: the tensor maps have the real width, so TMA loads zero-fill the columns past it
// and TMA stores clip there.
bool attn_fused_supported(int S, int dk) {
  return S >= 1 && S <= 4096 && dk >= 4 && dk <= 256 && dk % 4 == 0;
}

int launch_attn_fwd(const AttnFwdArgs& a, cudaStream_t st) {
  if (!attn_fused_supported(a.S, a.dk)) { arb_set_error("fused attention: unsupported shape"); return ARB_E_UNSUPPORTED; }
  if (a.S > 256 || (a.dk > 32 && a.dk != 64)) return launch_attn_long_fwd(a, st);
  if (a.dk <= 16) return launch_fwd_t<16>(a, st);
  if (a.dk <= 32) return launch_fwd_t<32>(a, st);
  return launch_fwd_t<64>(a, st);
}

}  // namespace arb
