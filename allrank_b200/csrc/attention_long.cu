// Fused self-attention for slates of 257 ... 4096 items at head width 16 or 32, forward and backward, without the
// S x S matrix.  attention_fused.cu / attention_fused_bwd.cu serve S <= 256 by holding a whole (slate, head) in shared
// memory; that stops fitting beyond 256 rows, so here a work item is one 128-row tile of a (slate, head) and the other
// side of its products streams through a ring of shared-memory stages:
//   attn_long_fwd_kernel   tile of 128 queries;  streams K (pass A), then K and V (pass B)          -> ctx, row stats
//   attn_long_dkdv_kernel  tile of 128 keys;     streams Q, dO and the queries' {nm, delta}         -> dK, dV
//   attn_long_dq_kernel    tile of 128 queries;  streams K, V                                      -> dQ
// Each 16-row strip of a tile is one compute warp's and runs the short kernels' per-strip arithmetic in the same key /
// query order (two-pass softmax, no rescaling), so a slate that the short kernels serve gets the same bits here: the
// context, row statistics and dQ / dK / dV.  Only the QKV bias gradient is summed in another order.
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

constexpr int LONG_WARPS = 8;                         // compute warps: one 16-row strip of the tile each
constexpr int LONG_THREADS = 32 * (LONG_WARPS + 1);   // + one load warp
constexpr int LONG_BLK = 128;                         // rows of a tile and of a streamed block
constexpr int LONG_NST = 4;                           // stages of the ring
constexpr int LONG_OP = LONG_BLK * 128;               // one operand of a buffer: 128 rows of 128 bytes
constexpr int LONG_BUF = 2 * LONG_OP + 1024;          // two operands + aux (key bits, or float2 {nm, delta} per query)
constexpr int LONG_OUT = 2 * 2048;                    // per compute warp: two 16-row output boxes

struct LongSmem {
  // [tile buffer] [ring: LONG_NST buffers] [output boxes] [mbarriers: full[NST] empty[NST] res_full res_empty]
  static constexpr int ring = LONG_BUF;
  static constexpr int out = ring + LONG_NST * LONG_BUF;
  static constexpr int bars = out + LONG_WARPS * LONG_OUT;
  static constexpr int total = bars + 8 * (2 * LONG_NST + 2) + 1024;
};
static_assert(LongSmem::total <= 227 * 1024, "attention_long: shared memory");

enum { LONG_FWD = 0, LONG_DKDV = 1, LONG_DQ = 2 };
enum { AUX_NONE = 0, AUX_BITS = 1, AUX_STATS = 2 };

// One CTA per SM walks the items blockIdx.x, blockIdx.x + gridDim.x, ...; item ((b * h) + head) * tiles + tile.
// The last warp loads.  Per item it TMA-loads the tile's rows (forward: Q; dK / dV: K, V; dQ: Q, dO) into the tile
// buffer (res_full; free again once every compute warp has taken its fragments: res_empty), then the streamed blocks
// into the ring, in 16-row boxes up to the extent, each stage completing on full[stage] and freed by one arrival per
// compute warp on empty[stage].  With the rows it writes a buffer's aux: the real-key bits of its keys, or the
// per-query {nm = -max c - log2 sum, delta} of its queries (c = log2(e) / sqrt(dk)).  Operands are rounded to tf32
// (cvt.rn) after every fragment load, which gives the values the short kernels round in place; with rounding off the
// tensor core truncates.
//
// Extents: keys at or beyond a slate's extent are masked (probability exactly 0) and not streamed, so the work is
// proportional to S * extent.  The forward computes every query row below round_up(S, 16) (padded items get the
// reference's scores).  The backward's extent also bounds the queries (their d ctx rows are zero): its strips at or
// beyond round_up(extent, 16) stream nothing and store exact zeros.
template <int MODE, int DK, bool DROP>
__device__ __forceinline__ void attn_long_body(
    const CUtensorMap* tmR0, const CUtensorMap* tmR1, const CUtensorMap* tmS0, const CUtensorMap* tmS1,
    const CUtensorMap* tmO0, const CUtensorMap* tmO1, const uint8_t* __restrict__ mask, float* __restrict__ stat_max,
    float* __restrict__ stat_sum, const float* __restrict__ delta, int S, int n_heads, float scale, DropSite drop,
    float* __restrict__ dbias, int d_model, const int* __restrict__ extent, int n_items, int rnd) {
  constexpr int KS = DK / 8;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t sbase = (ptx::smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* smem = smem_dyn + (sbase - ptx::smem_u32(smem_dyn));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + LongSmem::bars);
  uint64_t* empty = full + LONG_NST;
  uint64_t* res_full = empty + LONG_NST;
  uint64_t* res_empty = res_full + 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float c_log2e = scale * 1.4426950408889634f;
  const int tiles = (S + LONG_BLK - 1) / LONG_BLK;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(tmR0); ptx::prefetch_tmap(tmR1); ptx::prefetch_tmap(tmS0); ptx::prefetch_tmap(tmS1);
    for (int s = 0; s < LONG_NST; ++s) {
      ptx::mbar_init(full + s, 33);         // the expect_tx arrival + every load lane after its aux stores
      ptx::mbar_init(empty + s, LONG_WARPS);
    }
    ptx::mbar_init(res_full, 33);
    ptx::mbar_init(res_empty, LONG_WARPS);
    ptx::fence_barrier_init();
  }
  arb_pdl_wait();
  __syncthreads();

  struct Item { int b, head, tile, e, ns, live, rows16, nblk; };
  auto item_info = [&](int item) {
    Item it;
    it.tile = item % tiles;
    const int bh = item / tiles;
    it.b = bh / n_heads;
    it.head = bh - it.b * n_heads;
    it.e = max(1, min(S, extent ? __ldg(extent + it.b) : S));
    it.rows16 = (it.e + 15) & ~15;
    it.ns = min(LONG_WARPS, (S + 15) / 16 - LONG_WARPS * it.tile);       // strips of the tile below round_up(S, 16)
    it.live = MODE == LONG_FWD ? it.ns : max(0, min(it.ns, it.rows16 / 16 - LONG_WARPS * it.tile));
    it.nblk = it.live > 0 ? (it.rows16 + LONG_BLK - 1) / LONG_BLK : 0;  // streamed blocks (keys, or queries for dK / dV)
    return it;
  };
  constexpr int NPASS = MODE == LONG_FWD ? 2 : 1;

  if (warp == LONG_WARPS) {
    // ===== load warp
    // rows row0 ... row0 + rows - 1 of `ops` operands into buffer `buf` (operand o at buf + o * LONG_OP), its aux, and
    // the arrivals on `bar`
    auto fill = [&](uint8_t* buf, uint64_t* bar, const Item& it, int row0, int rows, int ops, const CUtensorMap* m0,
                    const CUtensorMap* m1, int aux) {
      ptx::fence_proxy_async_smem();
      if (lane == 0) ptx::mbar_expect_tx(bar, uint32_t(rows * ops * 128));
      __syncwarp();
      const int nb = rows >> 4;
      for (int j = lane; j < ops * nb; j += 32) {
        const int o = j / nb, i = j - o * nb;
        ptx::tma_load_4d(buf + o * LONG_OP + i * 2048, o ? m1 : m0, bar, 0, row0 + 16 * i, it.head, it.b);
      }
      uint8_t* ax = buf + 2 * LONG_OP;
      if (aux == AUX_BITS) {          // bit j of word w: key row0 + 32 w + j is real
#pragma unroll
        for (int w = 0; w < LONG_BLK / 32; ++w) {
          const int key = row0 + 32 * w + lane;
          const uint32_t bw = __ballot_sync(FULL, key < S && mask[size_t(it.b) * S + key] == 0);
          if (lane == 0) reinterpret_cast<uint32_t*>(ax)[w] = bw;
        }
      } else if (aux == AUX_STATS) {  // queries the slate does not have: nm = -inf (probability 0)
#pragma unroll
        for (int w = 0; w < LONG_BLK / 32; ++w) {
          const int qi = row0 + 32 * w + lane;
          float2 st = make_float2(-CUDART_INF_F, 0.f);
          if (qi < S) {
            const size_t so = (size_t(it.b) * n_heads + it.head) * S + qi;
            st = make_float2(-(stat_max[so] * c_log2e) - log2f(stat_sum[so]), delta[so]);
          }
          reinterpret_cast<float2*>(ax)[32 * w + lane] = st;
        }
      }
      ptx::mbar_arrive(bar);
    };
    constexpr int RES_OPS = MODE == LONG_FWD ? 1 : 2;
    constexpr int RES_AUX = MODE == LONG_FWD ? AUX_NONE : (MODE == LONG_DKDV ? AUX_BITS : AUX_STATS);
    constexpr int STR_AUX = MODE == LONG_DKDV ? AUX_STATS : AUX_BITS;
    int cnt = 0, k = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++k) {
      const Item it = item_info(item);
      if (k >= 1) ptx::mbar_wait(res_empty, (k - 1) & 1);
      fill(smem, res_full, it, LONG_BLK * it.tile, 16 * it.live, RES_OPS, tmR0, tmR1, RES_AUX);
      for (int pass = 0; pass < NPASS; ++pass) {
        for (int blk = 0; blk < it.nblk; ++blk, ++cnt) {
          const int st = cnt % LONG_NST;
          if (cnt >= LONG_NST) ptx::mbar_wait(empty + st, ((cnt / LONG_NST) - 1) & 1);
          fill(smem + LongSmem::ring + st * LONG_BUF, full + st, it, LONG_BLK * blk,
               min(LONG_BLK, it.rows16 - LONG_BLK * blk), (MODE == LONG_FWD && pass == 0) ? 1 : 2, tmS0, tmS1, STR_AUX);
        }
      }
    }
    return;
  }

  // ===== compute warps
  if constexpr (DROP) drop.seed = drop_seed(drop);
  auto rt = [&](uint32_t& x) { if (rnd) x = ptx::cvt_tf32(__uint_as_float(x)); };
  const uint32_t res_s = sbase, box_s = sbase + LongSmem::out + warp * LONG_OUT;
  uint8_t* box = smem + LongSmem::out + warp * LONG_OUT;
  int cnt = 0, k = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++k) {
    const Item it = item_info(item);
    const bool has = warp < it.ns, live = warp < it.live;
    const int strip = LONG_WARPS * it.tile + warp, r0 = 16 * warp;      // r0: the strip's rows in the tile buffer
    const unsigned long long dbase = (unsigned long long)(it.b * n_heads + it.head) * S;
    // the streamed blocks of this item: fn(block, buffer address) on the warps that have a live strip; every warp
    // frees every stage
    auto consume = [&](auto&& fn) {
      for (int blk = 0; blk < it.nblk; ++blk, ++cnt) {
        const int st = cnt % LONG_NST;
        ptx::mbar_wait(full + st, (cnt / LONG_NST) & 1);
        if (live) fn(blk, sbase + LongSmem::ring + st * LONG_BUF);
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(empty + st);
      }
    };
    auto release_tile = [&]() {
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(res_empty);
    };
    // a finished 16-row strip (rows g, g + 8 of acc, x mul) into the 128B-swizzled output box at `b`
    auto stage_strip = [&](uint32_t b, const float (&acc)[KS][4], float mul) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = g + 8 * h;
        float v[2][KS];      // v[0]: head columns of output column 2t, v[1]: of 2t + 1 (n-tile order)
#pragma unroll
        for (int nt = 0; nt < KS; ++nt) { v[0][nt] = acc[nt][2 * h] * mul; v[1][nt] = acc[nt][2 * h + 1] * mul; }
        if constexpr (KS == 4) {
          sts128(b + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[0][2]), __float_as_uint(v[0][3])));
          sts128(b + ptx::sw128(r, 64 + 16 * t), make_uint4(__float_as_uint(v[1][0]), __float_as_uint(v[1][1]), __float_as_uint(v[1][2]), __float_as_uint(v[1][3])));
        } else {
          sts128(b + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[1][0]), __float_as_uint(v[1][1])));
        }
      }
    };
    // QKV bias gradient: the staged strip's column sums (rows in order) added to this warp's own slot -- one slot per
    // (CTA, warp), its items in a fixed order; DetParts sums the slots in order
    auto bias_add = [&](int bx, int col0) {
      if (dbias == nullptr || lane >= DK) return;
      float s = 0.f;
#pragma unroll
      for (int r = 0; r < 16; ++r) s += *reinterpret_cast<const float*>(box + bx * 2048 + ptx::sw128(r, 4 * lane));
      dbias[(size_t(blockIdx.x) * LONG_WARPS + warp) * 3 * d_model + col0 + it.head * DK + lane] += s;
    };
    auto store_wait = [&]() {   // this warp's previous strip must have been read out of its boxes
      if (lane == 0) ptx::tma_store_wait_read();
      __syncwarp();
    };
    auto store = [&](int nbox) {
      ptx::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        ptx::tma_store_4d(tmO0, box, 0, 16 * strip, it.head, it.b);
        if (nbox > 1) ptx::tma_store_4d(tmO1, box + 2048, 0, 16 * strip, it.head, it.b);
        ptx::tma_store_commit();
      }
    };
    ptx::mbar_wait(res_full, k & 1);

    if constexpr (MODE == LONG_FWD) {
      // ===== 16 queries: pass A masked row maxima, pass B probabilities and O = P V (attn_fwd_kernel's strip)
      const int qA = 16 * strip + g, qB = qA + 8;
      uint32_t qa[KS][4];
      if (live) {
        ld_a_head<KS>(res_s, r0, lane, qa);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) { rt(qa[ks][0]); rt(qa[ks][1]); rt(qa[ks][2]); rt(qa[ks][3]); }
      }
      release_tile();
      // raw scores of keys 8j + t, 8j + t + 4 of the block at k_s for rows qA, qB
      auto scores = [&](uint32_t k_s, int j, float (&s4)[4]) {
        s4[0] = s4[1] = s4[2] = s4[3] = 0.f;
        uint32_t kf[KS][2];
        ld_b_head<KS>(k_s, 8 * j, lane, kf);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) { rt(kf[ks][0]); rt(kf[ks][1]); ptx::mma_tf32(s4, qa[ks], kf[ks]); }
      };
      const int nj_all = (it.e + 7) >> 3;
      float mxA = -CUDART_INF_F, mxB = -CUDART_INF_F;
      consume([&](int blk, uint32_t buf) {
        const uint32_t* bits = reinterpret_cast<const uint32_t*>(smem + (buf - sbase) + 2 * LONG_OP);
        const int nj = min(LONG_BLK / 8, nj_all - LONG_BLK / 8 * blk);
#pragma unroll 2
        for (int j = 0; j < nj; ++j) {
          float s4[4];
          scores(buf, j, s4);
          const uint32_t kw = bits[j >> 2] >> ((8 * j & 31) + t);
          if (kw & 1u) { mxA = fmaxf(mxA, s4[0]); mxB = fmaxf(mxB, s4[2]); }
          if (kw & 16u) { mxA = fmaxf(mxA, s4[1]); mxB = fmaxf(mxB, s4[3]); }
        }
      });
      mxA = fmaxf(mxA, __shfl_xor_sync(FULL, mxA, 1)); mxA = fmaxf(mxA, __shfl_xor_sync(FULL, mxA, 2));
      mxB = fmaxf(mxB, __shfl_xor_sync(FULL, mxB, 1)); mxB = fmaxf(mxB, __shfl_xor_sync(FULL, mxB, 2));
      const float mxsA = mxA * c_log2e, mxsB = mxB * c_log2e;
      const bool odd = (t & 1) != 0;
      float sumA = 0.f, sumB = 0.f;
      float o[KS][4];
#pragma unroll
      for (int nt = 0; nt < KS; ++nt) o[nt][0] = o[nt][1] = o[nt][2] = o[nt][3] = 0.f;
      consume([&](int blk, uint32_t buf) {
        const uint32_t* bits = reinterpret_cast<const uint32_t*>(smem + (buf - sbase) + 2 * LONG_OP);
        const uint32_t v_s = buf + LONG_OP;
        const int nj = min(LONG_BLK / 8, nj_all - LONG_BLK / 8 * blk);
#pragma unroll 2
        for (int j = 0; j < nj; ++j) {
          float s4[4];
          scores(buf, j, s4);
          const uint32_t kw = bits[j >> 2] >> ((8 * j & 31) + t);
          // an all-padded slate gives (-inf) - (-inf) = NaN like the reference
          float p[4];
          p[0] = (kw & 1u) ? ex2_approx(fmaf(s4[0], c_log2e, -mxsA)) : 0.0f;
          p[1] = (kw & 16u) ? ex2_approx(fmaf(s4[1], c_log2e, -mxsA)) : 0.0f;
          p[2] = (kw & 1u) ? ex2_approx(fmaf(s4[2], c_log2e, -mxsB)) : 0.0f;
          p[3] = (kw & 16u) ? ex2_approx(fmaf(s4[3], c_log2e, -mxsB)) : 0.0f;
          // row sums before dropout, in attn_fwd_kernel's association
          const float xA = __shfl_xor_sync(FULL, odd ? p[0] : p[1], 1);
          const float xB = __shfl_xor_sync(FULL, odd ? p[2] : p[3], 1);
          sumA += odd ? xA + p[1] : p[0] + xA;
          sumB += odd ? xB + p[3] : p[2] + xB;
          if constexpr (DROP) {
            const int key0 = LONG_BLK * blk + 8 * j + t;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const unsigned long long idx = (dbase + (i < 2 ? qA : qB)) * (unsigned long long)S + (key0 + 4 * (i & 1));
              p[i] = drop_keep(idx, drop.seed, drop.thresh) ? p[i] * drop.scale : 0.0f;
            }
          }
          const uint32_t pa[4] = {__float_as_uint(round_tf32(p[0])), __float_as_uint(round_tf32(p[2])),
                                  __float_as_uint(round_tf32(p[1])), __float_as_uint(round_tf32(p[3]))};
          uint32_t v0[KS], v1[KS];
          ld_b_out<KS>(v_s, 8 * j + t, g, v0);
          ld_b_out<KS>(v_s, 8 * j + t + 4, g, v1);
#pragma unroll
          for (int nt = 0; nt < KS; ++nt) {
            rt(v0[nt]); rt(v1[nt]);
            const uint32_t vb[2] = {v0[nt], v1[nt]};
            ptx::mma_tf32(o[nt], pa, vb);
          }
        }
      });
      if (has) {
        sumA += __shfl_xor_sync(FULL, sumA, 2); sumA += __shfl_xor_sync(FULL, sumA, 1);
        sumB += __shfl_xor_sync(FULL, sumB, 2); sumB += __shfl_xor_sync(FULL, sumB, 1);
        if (t == 0) {
          const size_t so = (size_t(it.b) * n_heads + it.head) * S;
          if (qA < S) { stat_max[so + qA] = mxA; stat_sum[so + qA] = sumA; }
          if (qB < S) { stat_max[so + qB] = mxB; stat_sum[so + qB] = sumB; }
        }
        store_wait();
        // O / rowsum, per row (one reciprocal each, as attn_fwd_kernel)
        float oA[KS][4];
        const float invA = 1.0f / sumA, invB = 1.0f / sumB;
#pragma unroll
        for (int nt = 0; nt < KS; ++nt) {
          oA[nt][0] = o[nt][0] * invA; oA[nt][1] = o[nt][1] * invA;
          oA[nt][2] = o[nt][2] * invB; oA[nt][3] = o[nt][3] * invB;
        }
        stage_strip(box_s, oA, 1.0f);
        store(1);
      }
    } else if constexpr (MODE == LONG_DKDV) {
      // ===== 16 keys kA = 16 strip + g, kB = kA + 8: dV, dK over the streamed queries (attn_bwd_kernel's key strip)
      const int kA = 16 * strip + g, kB = kA + 8;
      uint32_t ka[KS][4], va[KS][4];
      bool liveA = false, liveB = false;
      if (live) {
        const uint32_t kw = reinterpret_cast<const uint32_t*>(smem + 2 * LONG_OP)[warp >> 1];
        liveA = (kw >> ((r0 + g) & 31)) & 1u;
        liveB = (kw >> ((r0 + g + 8) & 31)) & 1u;
        ld_a_head<KS>(res_s, r0, lane, ka);
        ld_a_head<KS>(res_s + LONG_OP, r0, lane, va);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
          for (int i = 0; i < 4; ++i) { rt(ka[ks][i]); rt(va[ks][i]); }
      }
      release_tile();
      float dv[KS][4], dk[KS][4];
#pragma unroll
      for (int nt = 0; nt < KS; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) dv[nt][i] = dk[nt][i] = 0.f;
      const int nq8 = (it.e + 7) & ~7;     // queries at or beyond the extent have zero d ctx rows
      consume([&](int blk, uint32_t buf) {
        const uint32_t q_s = buf, do_s = buf + LONG_OP, st_s = buf + 2 * LONG_OP;
        const int qbase = LONG_BLK * blk, nq = min(LONG_BLK, nq8 - qbase);
        // S^T, dP^T of the 8-query block q0 (of the buffer)
        auto products = [&](int q0, float (&s)[4], float (&dp)[4]) {
#pragma unroll
          for (int i = 0; i < 4; ++i) s[i] = dp[i] = 0.f;
          uint32_t qb[KS][2], ob[KS][2];
          ld_b_head<KS>(q_s, q0, lane, qb);
          ld_b_head<KS>(do_s, q0, lane, ob);
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            rt(qb[ks][0]); rt(qb[ks][1]); rt(ob[ks][0]); rt(ob[ks][1]);
            ptx::mma_tf32(s, ka[ks], qb[ks]);
            ptx::mma_tf32(dp, va[ks], ob[ks]);
          }
        };
        // P^T, dS^T of the block and its dV, dK products
        auto accumulate = [&](int q0, const float (&s)[4], const float (&dp)[4]) {
          const uint2 st0 = lds64(st_s + 8 * (q0 + t)), st1 = lds64(st_s + 8 * (q0 + t + 4));
          float pu[4], ds[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int q = qbase + q0 + t + 4 * (i & 1);
            const float nm = __uint_as_float((i & 1) ? st1.x : st0.x), dl = __uint_as_float((i & 1) ? st1.y : st0.y);
            const float p = (i < 2 ? liveA : liveB) ? ex2_approx(fmaf(s[i], c_log2e, nm)) : 0.0f;
            float p_used = p, dpv = dp[i];
            if constexpr (DROP) {
              const unsigned long long idx = (dbase + q) * (unsigned long long)S + (i < 2 ? kA : kB);
              const float m = drop_keep(idx, drop.seed, drop.thresh) ? drop.scale : 0.0f;
              p_used = p * m;
              dpv *= m;
            }
            pu[i] = round_tf32(p_used);
            ds[i] = round_tf32(p * (dpv - dl));
          }
          const uint32_t pa[4] = {__float_as_uint(pu[0]), __float_as_uint(pu[2]), __float_as_uint(pu[1]), __float_as_uint(pu[3])};
          const uint32_t dsa[4] = {__float_as_uint(ds[0]), __float_as_uint(ds[2]), __float_as_uint(ds[1]), __float_as_uint(ds[3])};
          uint32_t o0[KS], o1[KS], q0v[KS], q1v[KS];
          ld_b_out<KS>(do_s, q0 + t, g, o0); ld_b_out<KS>(do_s, q0 + t + 4, g, o1);
          ld_b_out<KS>(q_s, q0 + t, g, q0v); ld_b_out<KS>(q_s, q0 + t + 4, g, q1v);
#pragma unroll
          for (int nt = 0; nt < KS; ++nt) {
            rt(o0[nt]); rt(o1[nt]); rt(q0v[nt]); rt(q1v[nt]);
            const uint32_t ob[2] = {o0[nt], o1[nt]}, qb[2] = {q0v[nt], q1v[nt]};
            ptx::mma_tf32(dv[nt], pa, ob);
            ptx::mma_tf32(dk[nt], dsa, qb);
          }
        };
        // two blocks in flight
        int q0 = 0;
        for (; q0 + 16 <= nq; q0 += 16) {
          float s0[4], dp0[4], s1[4], dp1[4];
          products(q0, s0, dp0);
          products(q0 + 8, s1, dp1);
          accumulate(q0, s0, dp0);
          accumulate(q0 + 8, s1, dp1);
        }
        if (q0 < nq) {
          float s0[4], dp0[4];
          products(q0, s0, dp0);
          accumulate(q0, s0, dp0);
        }
      });
      if (has) {
        store_wait();
        stage_strip(box_s, dv, 1.0f);
        stage_strip(box_s + 2048, dk, scale);
        __syncwarp();
        if (live) { bias_add(0, 2 * d_model); bias_add(1, d_model); }
        store(2);
      }
    } else {
      // ===== 16 queries qA = 16 strip + g, qB = qA + 8: dQ over the streamed keys (attn_bwd_kernel's query strip)
      const int qA = 16 * strip + g, qB = qA + 8;
      uint32_t qa[KS][4], oa[KS][4];
      float2 stA = make_float2(0.f, 0.f), stB = stA;
      if (live) {
        const float2* qst = reinterpret_cast<const float2*>(smem + 2 * LONG_OP);
        stA = qst[r0 + g];
        stB = qst[r0 + g + 8];
        ld_a_head<KS>(res_s, r0, lane, qa);
        ld_a_head<KS>(res_s + LONG_OP, r0, lane, oa);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
          for (int i = 0; i < 4; ++i) { rt(qa[ks][i]); rt(oa[ks][i]); }
      }
      release_tile();
      float dq[KS][4];
#pragma unroll
      for (int nt = 0; nt < KS; ++nt) dq[nt][0] = dq[nt][1] = dq[nt][2] = dq[nt][3] = 0.f;
      const int nk8 = (it.e + 7) & ~7;     // keys at or beyond the extent are masked
      consume([&](int blk, uint32_t buf) {
        const uint32_t k_s = buf, v_s = buf + LONG_OP, kb_s = buf + 2 * LONG_OP;
        const int kbase = LONG_BLK * blk, nk = min(LONG_BLK, nk8 - kbase);
        // S, dP of the 8-key block k0 (of the buffer)
        auto products = [&](int k0, float (&s)[4], float (&dp)[4]) {
#pragma unroll
          for (int i = 0; i < 4; ++i) s[i] = dp[i] = 0.f;
          uint32_t kb[KS][2], vb[KS][2];
          ld_b_head<KS>(k_s, k0, lane, kb);
          ld_b_head<KS>(v_s, k0, lane, vb);
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            rt(kb[ks][0]); rt(kb[ks][1]); rt(vb[ks][0]); rt(vb[ks][1]);
            ptx::mma_tf32(s, qa[ks], kb[ks]);
            ptx::mma_tf32(dp, oa[ks], vb[ks]);
          }
        };
        // dS of the block and its dQ products
        auto accumulate = [&](int k0, const float (&s)[4], const float (&dp)[4]) {
          const uint32_t kw = lds32(kb_s + 4 * (k0 >> 5)) >> ((k0 & 31) + t);
          float ds[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int key = kbase + k0 + t + 4 * (i & 1);
            const float2 st = i < 2 ? stA : stB;
            const float p = ((kw >> (4 * (i & 1))) & 1u) ? ex2_approx(fmaf(s[i], c_log2e, st.x)) : 0.0f;
            float dpv = dp[i];
            if constexpr (DROP) {
              const unsigned long long idx = (dbase + (i < 2 ? qA : qB)) * (unsigned long long)S + key;
              dpv *= drop_keep(idx, drop.seed, drop.thresh) ? drop.scale : 0.0f;
            }
            ds[i] = round_tf32(p * (dpv - st.y));
          }
          const uint32_t dsa[4] = {__float_as_uint(ds[0]), __float_as_uint(ds[2]), __float_as_uint(ds[1]), __float_as_uint(ds[3])};
          uint32_t k0v[KS], k1v[KS];
          ld_b_out<KS>(k_s, k0 + t, g, k0v); ld_b_out<KS>(k_s, k0 + t + 4, g, k1v);
#pragma unroll
          for (int nt = 0; nt < KS; ++nt) {
            rt(k0v[nt]); rt(k1v[nt]);
            const uint32_t kb[2] = {k0v[nt], k1v[nt]};
            ptx::mma_tf32(dq[nt], dsa, kb);
          }
        };
        int k0 = 0;
        for (; k0 + 16 <= nk; k0 += 16) {
          float s0[4], dp0[4], s1[4], dp1[4];
          products(k0, s0, dp0);
          products(k0 + 8, s1, dp1);
          accumulate(k0, s0, dp0);
          accumulate(k0 + 8, s1, dp1);
        }
        if (k0 < nk) {
          float s0[4], dp0[4];
          products(k0, s0, dp0);
          accumulate(k0, s0, dp0);
        }
      });
      if (has) {
        store_wait();
        stage_strip(box_s, dq, scale);
        __syncwarp();
        if (live) bias_add(0, 0);
        store(1);
      }
    }
  }
  if (lane == 0) ptx::tma_store_wait_all();
}

#define ARB_LONG_KERNEL(name, MODE)                                                                                   \
  template <int DK, bool DROP>                                                                                        \
  __global__ void __launch_bounds__(LONG_THREADS, 1) name(                                                            \
      const __grid_constant__ CUtensorMap tmR0, const __grid_constant__ CUtensorMap tmR1,                             \
      const __grid_constant__ CUtensorMap tmS0, const __grid_constant__ CUtensorMap tmS1,                             \
      const __grid_constant__ CUtensorMap tmO0, const __grid_constant__ CUtensorMap tmO1, const uint8_t* mask,         \
      float* stat_max, float* stat_sum, const float* delta, int S, int n_heads, float scale, DropSite drop,           \
      float* dbias, int d_model, const int* extent, int n_items, int rnd) {                                           \
    attn_long_body<MODE, DK, DROP>(&tmR0, &tmR1, &tmS0, &tmS1, &tmO0, &tmO1, mask, stat_max, stat_sum, delta, S,      \
                                   n_heads, scale, drop, dbias, d_model, extent, n_items, rnd);                       \
  }
ARB_LONG_KERNEL(attn_long_fwd_kernel, LONG_FWD)
ARB_LONG_KERNEL(attn_long_dkdv_kernel, LONG_DKDV)
ARB_LONG_KERNEL(attn_long_dq_kernel, LONG_DQ)
#undef ARB_LONG_KERNEL

using LongKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap,
                            const uint8_t*, float*, float*, const float*, int, int, float, DropSite, float*, int,
                            const int*, int, int);

static int long_items(int B, int h, int S) { return B * h * ((S + LONG_BLK - 1) / LONG_BLK); }

// Bytes the kernels request from L2 / HBM per (slate, head): the tile side once, the streamed side once per tile
// (the ProfScope accounting; the streamed rows mostly hit L2)
static double long_bytes(int S, int dk, int tile_ops, int stream_ops, int out_ops) {
  const double tiles = (S + LONG_BLK - 1) / LONG_BLK;
  return 4.0 * S * dk * (tile_ops + out_ops + tiles * stream_ops);
}

template <int DK>
static int launch_long_fwd_t(const AttnFwdArgs& a, cudaStream_t st) {
  alignas(64) CUtensorMap tQ, tK, tV, tO;
  int rc;
  const TmapBox box{{32, 16, 1, 1}};
  if ((rc = make_tmap_4d(&tQ, a.q, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tK, a.k, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tV, a.v, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tO, a.o, box, 0))) return rc;
  const LongKernel kern = a.drop.thresh != 0 ? attn_long_fwd_kernel<DK, true> : attn_long_fwd_kernel<DK, false>;
  const int n_items = long_items(a.B, a.h, a.S);
  dim3 grid(std::max(1, std::min(n_items, sm_count())));
  ProfScope ps(ARB_PROF_GEMM, (a.extent ? arb_attn_frac() : 1.0) * 4.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
               double(a.B) * a.h * (long_bytes(a.S, a.dk, 1, 3, 1) + 8.0 * a.S), "attn_long_fwd_kernel");
  return launch(kern, grid, dim3(LONG_THREADS), size_t(LongSmem::total), st, /*pdl=*/true, tQ, tQ, tK, tV, tO, tO,
                a.mask, a.stat_max, a.stat_sum, static_cast<const float*>(nullptr), a.S, a.h, a.scale, a.drop,
                static_cast<float*>(nullptr), 0, a.extent, n_items, tf32_round_on_load());
}

int launch_attn_long_fwd(const AttnFwdArgs& a, cudaStream_t st) {
  if (a.o.bf16) { arb_set_error("attn_fwd: a bf16 context needs slate_length <= 256"); return ARB_E_UNSUPPORTED; }
  if (a.pack_off) { arb_set_error("attn_fwd: packed rows need slate_length <= 256"); return ARB_E_UNSUPPORTED; }
  return a.dk == 16 ? launch_long_fwd_t<16>(a, st) : launch_long_fwd_t<32>(a, st);
}

template <int DK>
static int launch_long_bwd_t(const AttnBwdArgs& a, cudaStream_t st) {
  alignas(64) CUtensorMap tQ, tK, tV, tDO, tDQ, tDK, tDV;
  int rc;
  const TmapBox box{{32, 16, 1, 1}};
  if ((rc = make_tmap_4d(&tQ, a.q, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tK, a.k, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tV, a.v, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tDO, a.d_o, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tDQ, a.dq, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tDK, a.dk_, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tDV, a.dv, box, 0))) return rc;
  const bool drop = a.drop.thresh != 0;
  const LongKernel kdkdv = drop ? attn_long_dkdv_kernel<DK, true> : attn_long_dkdv_kernel<DK, false>;
  const LongKernel kdq = drop ? attn_long_dq_kernel<DK, true> : attn_long_dq_kernel<DK, false>;
  const int n_items = long_items(a.B, a.h, a.S);
  const int n_ctas = std::max(1, std::min(n_items, sm_count()));
  // the QKV bias gradient: one slot per (CTA, compute warp), summed in order afterwards
  float* dbias = a.dbias_qkv;
  DetParts dp;
  dp.add(dbias, (long long)n_ctas * LONG_WARPS, 1, 3LL * a.d_model, 3LL * a.d_model);
  if ((rc = dp.begin(st))) return rc;
  float* smax = const_cast<float*>(a.stat_max);
  float* ssum = const_cast<float*>(a.stat_sum);
  const double frac = a.extent ? arb_attn_frac() : 1.0;
  {
    ProfScope ps(ARB_PROF_GEMM, frac * 8.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
                 double(a.B) * a.h * (long_bytes(a.S, a.dk, 2, 2, 2) + 8.0 * a.S), "attn_long_dkdv_kernel");
    if ((rc = launch(kdkdv, dim3(n_ctas), dim3(LONG_THREADS), size_t(LongSmem::total), st, /*pdl=*/true, tK, tV, tQ,
                     tDO, tDV, tDK, a.mask, smax, ssum, a.delta, a.S, a.h, a.scale, a.drop, dbias, a.d_model, a.extent,
                     n_items, tf32_round_on_load())))
      return rc;
  }
  {
    ProfScope ps(ARB_PROF_GEMM, frac * 6.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
                 double(a.B) * a.h * (long_bytes(a.S, a.dk, 2, 2, 1) + 12.0 * a.S), "attn_long_dq_kernel");
    if ((rc = launch(kdq, dim3(n_ctas), dim3(LONG_THREADS), size_t(LongSmem::total), st, /*pdl=*/true, tQ, tDO, tK,
                     tV, tDQ, tDQ, a.mask, smax, ssum, a.delta, a.S, a.h, a.scale, a.drop, dbias, a.d_model, a.extent,
                     n_items, tf32_round_on_load())))
      return rc;
  }
  return dp.finish(st);
}

int launch_attn_long_bwd(const AttnBwdArgs& a, cudaStream_t st) {
  return a.dk == 16 ? launch_long_bwd_t<16>(a, st) : launch_long_bwd_t<32>(a, st);
}

}  // namespace arb
