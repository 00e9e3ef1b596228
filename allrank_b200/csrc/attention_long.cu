// Fused self-attention at head widths 4 ... 32 for slates of 257 ... 4096 items, and at head widths 36 ... 256 for slates
// of 1 ... 4096 items (w % 4 == 0), forward and backward, without the S x S matrix.  attention_fused.cu /
// attention_fused_bwd.cu serve S <= 256 at width <= 32 (the forward also 64) by holding a whole (slate, head) in shared
// memory; that stops fitting beyond 256 rows or 32 columns, so here a work item is one 128-row tile (DK 192, 256: 64
// rows) of a (slate, head) and the other side of its products streams through a ring of shared-memory stages:
//   attn_long_fwd_kernel   tile of queries;  streams K (pass A), then K and V (pass B)              -> ctx, row stats
//   attn_long_dkdv_kernel  tile of keys;     streams Q, dO and the queries' {nm, delta}             -> dK, dV
//   attn_long_dq_kernel    tile of queries;  streams K, V                                          -> dQ
// Each 16-row strip of a tile is one compute warp's and runs the short kernels' per-strip arithmetic in the same key /
// query order (two-pass softmax, no rescaling), so a slate that the short kernels serve gets the same bits here: the
// context, row statistics and dQ / dK / dV.  Only the QKV bias gradient is summed in another order.  At DK 192 and 256
// a strip is two warps': both compute its full score rows with the same instructions (so the same P / dS bits), and
// each multiplies them into its own half of the output columns.
#include <algorithm>
#include <cstdint>
#include <type_traits>
#include <cuda.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "attention_frag.cuh"
#include "attention_fused.h"
#include "block_utils.cuh"
#include "common.h"
#include "sm90_ptx.cuh"

namespace arb {

constexpr int LONG_WARPS = 8;                         // compute warps: one 16-row strip of the tile each (DK 192, 256:
                                                      // warps i and i + 4 share strip i)
constexpr int LONG_THREADS = 32 * (LONG_WARPS + 1);   // + one load warp
constexpr int LONG_BLK = 128;                         // rows of a tile (DK 192, 256: LongSmem::BLK = 64)

// An operand row of DK columns is NKB slabs of 128 bytes (32 fp32 columns; TMA zero-fills the columns past the head
// width), each slab of a buffer 128B-swizzled in its own 16-row boxes.  A buffer holds two operands, slab after slab,
// and an aux region (key bits, or float2 {nm, delta} per query).
//   DK <= 32: 128-row streamed blocks in four stages; the fragments of the tile's rows stay in registers, the tile is
//             free again once they are loaded, and each compute warp stages its strips in two boxes of its own.
//   DK 64, 96, 128 (wide): 64-row streamed blocks in four / two stages (DK 128: 32-row blocks in two stages, since a
//             tile of 2 x 4 slabs takes 129 KB); the tile stays resident for the whole item: the dK / dV and dQ strips
//             re-read its fragments for every k-step (they would not fit in registers beside the accumulators), and
//             each warp stages its finished strip over its own 16 rows of the tile.
//   DK 192, 256 (paired): 64-row tiles (48 / 64 KB per operand), 32- / 16-row streamed blocks in two stages; the two
//             warps of a strip own NKB / 2 output slabs each (the accumulators of DK 96 / 128) and stage into their
//             own slabs of the strip's tile rows, after both are done reading those rows.
template <int DK>
struct LongSmem {
  static constexpr bool WIDE = DK > 32;
  static constexpr bool PAIR = DK > 128;              // two warps per strip, each with half the output columns
  static constexpr int BLK = PAIR ? 64 : LONG_BLK;    // rows of a tile
  static constexpr int STRIPS = BLK / 16;             // strips of a tile
  static constexpr int NKB = (DK + 31) / 32;          // 128-byte slabs per operand row
  static constexpr int NKO = PAIR ? NKB / 2 : NKB;    // output slabs per warp
  static constexpr int KSB = DK / 8 / NKB;            // k8 steps per slab
  static constexpr int SBLK = DK > 192 ? 16 : DK > 96 ? 32 : WIDE ? 64 : 128;   // rows of a streamed block
  static constexpr int SAUX = SBLK < 32 ? 32 : SBLK;  // rows of a streamed block's aux (whole 32-bit key words)
  static constexpr int NST = DK <= 64 ? 4 : 2;        // stages of the ring
  static constexpr int TSLAB = BLK * 128;             // one slab of a tile operand
  static constexpr int SSLAB = SBLK * 128;            // one slab of a streamed operand
  static constexpr int TOP = NKB * TSLAB, SOP = NKB * SSLAB;
  static constexpr int TBUF = 2 * TOP + 1024, SBUF = 2 * SOP + 1024;
  static constexpr int OUT = WIDE ? 0 : 2 * 2048;     // per compute warp: two 16-row output boxes (wide: none)
  // [tile buffer] [ring: NST buffers] [output boxes] [mbarriers: full[NST] empty[NST] res_full res_empty]
  static constexpr int ring = TBUF;
  static constexpr int out = ring + NST * SBUF;
  static constexpr int bars = out + LONG_WARPS * OUT;
  static constexpr int total = bars + 8 * (2 * NST + 2) + 1024;
  static_assert(total <= 227 * 1024, "attention_long: shared memory");
  static_assert(DK % 32 == 0 || DK == 16, "attention_long: DK is 16 or a multiple of 32");
};

enum { LONG_FWD = 0, LONG_DKDV = 1, LONG_DQ = 2 };
enum { AUX_NONE = 0, AUX_BITS = 1, AUX_STATS = 2 };

// One CTA per SM walks the items blockIdx.x, blockIdx.x + gridDim.x, ...; item ((b * h) + head) * tiles + tile.
// The last warp loads.  Per item it TMA-loads the tile's rows (forward: Q; dK / dV: K, V; dQ: Q, dO) into the tile
// buffer (res_full; free again once every compute warp is done with it: res_empty), then the streamed blocks into the
// ring, in 16-row boxes up to the extent, each stage completing on full[stage] and freed by one arrival per compute
// warp on empty[stage].  With the rows it writes a buffer's aux: the real-key bits of its keys, or the per-query
// {nm = -max c - log2 sum, delta} of its queries (c = log2(e) / sqrt(w)).  Operands are rounded to tf32 (cvt.rn) after
// every fragment load, which gives the values the short kernels round in place; with rounding off the tensor core
// truncates.  Products run slab by slab and k-step by k-step, i.e. over the head columns in order, as the short
// kernels do.
//
// Head widths w that are not a slab multiple run on the next DK up: the tensor maps have w columns, so TMA loads give
// exact zeros in columns w ... DK - 1 (they add exact zeros to every product) and TMA stores clip at w.
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
  using L = LongSmem<DK>;
  constexpr int NKB = L::NKB, NKO = L::NKO, KSB = L::KSB, SBLK = L::SBLK, NST = L::NST, BLK = L::BLK;
  constexpr int STRIPS = L::STRIPS;
  constexpr bool WIDE = L::WIDE, PAIR = L::PAIR;
  // the tile's fragments stay in registers for the whole item (the forward's Q up to DK 96: at 128 Q's 64 registers
  // and O's 64 would spill)
  constexpr bool KEEP = !WIDE || (MODE == LONG_FWD && DK <= 96);
  constexpr int DKDV_NB = DK > 64 ? 1 : 2;      // 8-query blocks in flight in dK / dV
  constexpr int DQ_NB = DK > 192 ? 1 : 2;       // 8-key blocks in flight in dQ
  // DK 128: dK and dV are two passes over the streamed queries (dK, then dV), one 64-register accumulator each
  constexpr bool SPLIT = MODE == LONG_DKDV && DK > 96;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t sbase = (ptx::smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* smem = smem_dyn + (sbase - ptx::smem_u32(smem_dyn));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::bars);
  uint64_t* empty = full + NST;
  uint64_t* res_full = empty + NST;
  uint64_t* res_empty = res_full + 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float c_log2e = scale * 1.4426950408889634f;
  const int tiles = (S + BLK - 1) / BLK;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(tmR0); ptx::prefetch_tmap(tmR1); ptx::prefetch_tmap(tmS0); ptx::prefetch_tmap(tmS1);
    for (int s = 0; s < NST; ++s) {
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
    it.ns = min(STRIPS, (S + 15) / 16 - STRIPS * it.tile);               // strips of the tile below round_up(S, 16)
    it.live = MODE == LONG_FWD ? it.ns : max(0, min(it.ns, it.rows16 / 16 - STRIPS * it.tile));
    it.nblk = it.live > 0 ? (it.rows16 + SBLK - 1) / SBLK : 0;          // streamed blocks (keys, or queries for dK / dV)
    return it;
  };
  constexpr int NPASS = (MODE == LONG_FWD || SPLIT) ? 2 : 1;

  if (warp == LONG_WARPS) {
    // ===== load warp
    // rows row0 ... row0 + rows - 1 of `ops` operands into buffer `buf` (operand o, slab kb at buf + (o NKB + kb) slab),
    // its aux (for `cap` rows), and the arrivals on `bar`
    auto fill = [&](uint8_t* buf, uint64_t* bar, const Item& it, int row0, int rows, int ops, int slab, int cap,
                    const CUtensorMap* m0, const CUtensorMap* m1, int aux) {
      ptx::fence_proxy_async_smem();
      if (lane == 0) ptx::mbar_expect_tx(bar, uint32_t(rows * ops * NKB * 128));
      __syncwarp();
      const int nb = rows >> 4;
      for (int j = lane; j < ops * NKB * nb; j += 32) {
        const int o = j / (NKB * nb), r = j - o * (NKB * nb), kb = r / nb, i = r - kb * nb;
        ptx::tma_load_4d(buf + (o * NKB + kb) * slab + i * 2048, o ? m1 : m0, bar, 32 * kb, row0 + 16 * i, it.head, it.b);
      }
      uint8_t* ax = buf + 2 * NKB * slab;
      if (aux == AUX_BITS) {          // bit j of word w: key row0 + 32 w + j is real
#pragma unroll 4
        for (int w = 0; w < cap / 32; ++w) {
          const int key = row0 + 32 * w + lane;
          const uint32_t bw = __ballot_sync(FULL, key < S && mask[size_t(it.b) * S + key] == 0);
          if (lane == 0) reinterpret_cast<uint32_t*>(ax)[w] = bw;
        }
      } else if (aux == AUX_STATS) {  // queries the slate does not have: nm = -inf (probability 0)
#pragma unroll 4
        for (int w = 0; w < cap / 32; ++w) {
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
      fill(smem, res_full, it, BLK * it.tile, 16 * it.live, RES_OPS, L::TSLAB, BLK, tmR0, tmR1, RES_AUX);
      for (int pass = 0; pass < NPASS; ++pass) {
        for (int blk = 0; blk < it.nblk; ++blk, ++cnt) {
          const int st = cnt % NST;
          if (cnt >= NST) ptx::mbar_wait(empty + st, ((cnt / NST) - 1) & 1);
          fill(smem + L::ring + st * L::SBUF, full + st, it, SBLK * blk, min(SBLK, it.rows16 - SBLK * blk),
               (MODE == LONG_FWD && pass == 0) ? 1 : 2, L::SSLAB, L::SAUX, tmS0, tmS1, STR_AUX);
        }
      }
    }
    return;
  }

  // ===== compute warps
  if constexpr (DROP) drop.seed = drop_seed(drop);
  auto rt = [&](uint32_t& x) { if (rnd) x = ptx::cvt_tf32(__uint_as_float(x)); };
  const int sw = PAIR ? warp % STRIPS : warp;                          // the warp's strip of the tile
  const int kb0 = PAIR ? (warp / STRIPS) * NKO : 0;                    // the warp's first output slab
  const int r0 = 16 * sw;                                              // the warp's strip rows in the tile buffer
  // paired: both warps of the strip are done reading its tile rows, which either may now overwrite in its own slabs
  auto pair_sync = [&]() {
    if constexpr (PAIR) ptx::named_bar_sync(1 + sw, 64);
  };
  const uint32_t res_s = sbase;
  // output boxes: operand o, slab kb at ob_s + o * OB_OP + kb * L::TSLAB (wide: the warp's own tile rows)
  constexpr int OB_OP = WIDE ? L::TOP : 2048;
  const uint32_t ob_s = WIDE ? res_s + r0 * 128 : sbase + L::out + warp * L::OUT;
  uint8_t* ob = smem + (ob_s - sbase);
  // A fragment of k-step ks of slab kb of tile operand o, rows r0 ... r0 + 15 (wide dK / dV and dQ: from shared memory)
  uint32_t ta[KEEP ? NKB : 1][KSB][4], tb[KEEP && MODE != LONG_FWD ? NKB : 1][KSB][4];
  auto tfrag = [&](int o, int kb, int ks, uint32_t (&a)[4]) {
    if constexpr (KEEP) {
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = o ? tb[kb][ks][i] : ta[kb][ks][i];
    } else {
      ld_a_step(res_s + o * L::TOP + kb * L::TSLAB, r0, lane, ks, a);
#pragma unroll
      for (int i = 0; i < 4; ++i) rt(a[i]);
    }
  };
  auto load_tile_frags = [&](int ops) {
    if constexpr (KEEP) {
#pragma unroll
      for (int kb = 0; kb < NKB; ++kb) {
        ld_a_head<KSB>(res_s + kb * L::TSLAB, r0, lane, ta[kb]);
        if (ops > 1) ld_a_head<KSB>(res_s + L::TOP + kb * L::TSLAB, r0, lane, tb[kb]);
#pragma unroll
        for (int ks = 0; ks < KSB; ++ks)
#pragma unroll
          for (int i = 0; i < 4; ++i) { rt(ta[kb][ks][i]); if (ops > 1) rt(tb[kb][ks][i]); }
      }
    }
  };
  int cnt = 0, k = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++k) {
    const Item it = item_info(item);
    const bool has = sw < it.ns, live = sw < it.live;
    const int strip = STRIPS * it.tile + sw;
    const unsigned long long dbase = (unsigned long long)(it.b * n_heads + it.head) * S;
    // the streamed blocks of this item: fn(block, buffer address) on the warps that have a live strip; every warp
    // frees every stage
    auto consume = [&](auto&& fn) {
      for (int blk = 0; blk < it.nblk; ++blk, ++cnt) {
        const int st = cnt % NST;
        ptx::mbar_wait(full + st, (cnt / NST) & 1);
        if (live) fn(blk, sbase + L::ring + st * L::SBUF);
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(empty + st);
      }
    };
    auto release_tile = [&]() {
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(res_empty);
    };
    // a finished 16-row strip (rows g, g + 8 of acc, x mul) into the 128B-swizzled output box of operand o (the warp's
    // NKO slabs from kb0)
    auto stage_strip = [&](int o, const float (&acc)[NKO][KSB][4], float mul) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = g + 8 * h;
#pragma unroll
        for (int kb = 0; kb < NKO; ++kb) {
          const uint32_t b = ob_s + o * OB_OP + (kb0 + kb) * L::TSLAB;
          float v[2][KSB];      // v[0]: head columns of output column 2t, v[1]: of 2t + 1 (n-tile order)
#pragma unroll
          for (int nt = 0; nt < KSB; ++nt) { v[0][nt] = acc[kb][nt][2 * h] * mul; v[1][nt] = acc[kb][nt][2 * h + 1] * mul; }
          if constexpr (KSB == 4) {
            sts128(b + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[0][2]), __float_as_uint(v[0][3])));
            sts128(b + ptx::sw128(r, 64 + 16 * t), make_uint4(__float_as_uint(v[1][0]), __float_as_uint(v[1][1]), __float_as_uint(v[1][2]), __float_as_uint(v[1][3])));
          } else {
            sts128(b + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[1][0]), __float_as_uint(v[1][1])));
          }
        }
      }
    };
    // QKV bias gradient: the staged strip's column sums (rows in order) of the head's w real columns, added to this
    // warp's own slot -- one slot per (CTA, warp), its items in a fixed order; DetParts sums the slots in order (paired:
    // each warp sums only its own slabs' columns)
    auto bias_add = [&](int o, int col0) {
      if (dbias == nullptr) return;
      const int w = d_model / n_heads;
#pragma unroll
      for (int kb = 0; kb < NKO; ++kb) {
        const int c = 32 * (kb0 + kb) + lane;
        if (c >= w) break;
        const uint8_t* b = ob + o * OB_OP + (kb0 + kb) * L::TSLAB;
        float s = 0.f;
#pragma unroll
        for (int r = 0; r < 16; ++r) s += *reinterpret_cast<const float*>(b + ptx::sw128(r, 4 * lane));
        dbias[(size_t(blockIdx.x) * LONG_WARPS + warp) * 3 * d_model + col0 + it.head * w + c] += s;
      }
    };
    auto store_wait = [&]() {   // this warp's previous strip must have been read out of its boxes
      if (lane == 0) ptx::tma_store_wait_read();
      __syncwarp();
    };
    auto store = [&](int nbox) {
      ptx::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) {
        for (int o = 0; o < nbox; ++o)
#pragma unroll
          for (int kb = 0; kb < NKO; ++kb) {
            // paired: a slab wholly beyond the head width (e.g. columns 160 ... 191 at width 132) has nothing to store
            if (PAIR && 32 * (kb0 + kb) >= d_model / n_heads) break;
            ptx::tma_store_4d(o ? tmO1 : tmO0, ob + o * OB_OP + (kb0 + kb) * L::TSLAB, 32 * (kb0 + kb), 16 * strip,
                              it.head, it.b);
          }
        ptx::tma_store_commit();
      }
    };
    // the narrow kernels free the tile as soon as its fragments are in registers; the wide ones once the strip's
    // output has been read out of the tile rows
    auto finish_tile = [&]() {
      if constexpr (WIDE) {
        store_wait();
        release_tile();
      }
    };
    ptx::mbar_wait(res_full, k & 1);

    if constexpr (MODE == LONG_FWD) {
      // ===== 16 queries: pass A masked row maxima, pass B probabilities and O = P V (attn_fwd_kernel's strip)
      const int qA = 16 * strip + g, qB = qA + 8;
      if (live) load_tile_frags(1);
      if constexpr (!WIDE) release_tile();
      // raw scores of keys 8j + t, 8j + t + 4 of the block at k_s for rows qA, qB
      auto scores = [&](uint32_t k_s, int j, float (&s4)[4]) {
        s4[0] = s4[1] = s4[2] = s4[3] = 0.f;
#pragma unroll
        for (int kb = 0; kb < NKB; ++kb) {
          uint32_t kf[KSB][2];
          ld_b_head<KSB>(k_s + kb * L::SSLAB, 8 * j, lane, kf);
#pragma unroll
          for (int ks = 0; ks < KSB; ++ks) {
            uint32_t qa[4];
            tfrag(0, kb, ks, qa);
            rt(kf[ks][0]); rt(kf[ks][1]);
            ptx::mma_tf32(s4, qa, kf[ks]);
          }
        }
      };
      const int nj_all = (it.e + 7) >> 3;
      float mxA = -CUDART_INF_F, mxB = -CUDART_INF_F;
      consume([&](int blk, uint32_t buf) {
        const uint32_t* bits = reinterpret_cast<const uint32_t*>(smem + (buf - sbase) + 2 * L::SOP);
        const int nj = min(SBLK / 8, nj_all - SBLK / 8 * blk);
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
      float o[NKO][KSB][4];
#pragma unroll
      for (int kb = 0; kb < NKO; ++kb)
#pragma unroll
        for (int nt = 0; nt < KSB; ++nt) o[kb][nt][0] = o[kb][nt][1] = o[kb][nt][2] = o[kb][nt][3] = 0.f;
      consume([&](int blk, uint32_t buf) {
        const uint32_t* bits = reinterpret_cast<const uint32_t*>(smem + (buf - sbase) + 2 * L::SOP);
        const uint32_t v_s = buf + L::SOP;
        const int nj = min(SBLK / 8, nj_all - SBLK / 8 * blk);
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
            const int key0 = SBLK * blk + 8 * j + t;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const unsigned long long idx = (dbase + (i < 2 ? qA : qB)) * (unsigned long long)S + (key0 + 4 * (i & 1));
              p[i] = drop_keep(idx, drop.seed, drop.thresh) ? p[i] * drop.scale : 0.0f;
            }
          }
          const uint32_t pa[4] = {__float_as_uint(round_tf32(p[0])), __float_as_uint(round_tf32(p[2])),
                                  __float_as_uint(round_tf32(p[1])), __float_as_uint(round_tf32(p[3]))};
#pragma unroll
          for (int kb = 0; kb < NKO; ++kb) {
            uint32_t v0[KSB], v1[KSB];
            ld_b_out<KSB>(v_s + (kb0 + kb) * L::SSLAB, 8 * j + t, g, v0);
            ld_b_out<KSB>(v_s + (kb0 + kb) * L::SSLAB, 8 * j + t + 4, g, v1);
#pragma unroll
            for (int nt = 0; nt < KSB; ++nt) {
              rt(v0[nt]); rt(v1[nt]);
              const uint32_t vb[2] = {v0[nt], v1[nt]};
              ptx::mma_tf32(o[kb][nt], pa, vb);
            }
          }
        }
      });
      if (has) {
        sumA += __shfl_xor_sync(FULL, sumA, 2); sumA += __shfl_xor_sync(FULL, sumA, 1);
        sumB += __shfl_xor_sync(FULL, sumB, 2); sumB += __shfl_xor_sync(FULL, sumB, 1);
        if (t == 0 && kb0 == 0) {     // (paired: both warps have the same statistics)
          const size_t so = (size_t(it.b) * n_heads + it.head) * S;
          if (qA < S) { stat_max[so + qA] = mxA; stat_sum[so + qA] = sumA; }
          if (qB < S) { stat_max[so + qB] = mxB; stat_sum[so + qB] = sumB; }
        }
        store_wait();
        // O / rowsum, per row (one reciprocal each, as attn_fwd_kernel)
        const float invA = 1.0f / sumA, invB = 1.0f / sumB;
#pragma unroll
        for (int kb = 0; kb < NKO; ++kb)
#pragma unroll
          for (int nt = 0; nt < KSB; ++nt) {
            o[kb][nt][0] *= invA; o[kb][nt][1] *= invA;
            o[kb][nt][2] *= invB; o[kb][nt][3] *= invB;
          }
        pair_sync();
        stage_strip(0, o, 1.0f);
        store(1);
      }
      finish_tile();
    } else if constexpr (MODE == LONG_DKDV) {
      // ===== 16 keys kA = 16 strip + g, kB = kA + 8: dV, dK over the streamed queries (attn_bwd_kernel's key strip)
      const int kA = 16 * strip + g, kB = kA + 8;
      bool liveA = false, liveB = false;
      if (live) {
        const uint32_t kw = reinterpret_cast<const uint32_t*>(smem + 2 * L::TOP)[sw >> 1];
        liveA = (kw >> ((r0 + g) & 31)) & 1u;
        liveB = (kw >> ((r0 + g + 8) & 31)) & 1u;
        load_tile_frags(2);
      }
      if constexpr (!WIDE) release_tile();
      const int nq8 = (it.e + 7) & ~7;     // queries at or beyond the extent have zero d ctx rows
      // one pass over the streamed queries that adds their dV products to dv (with_dv) and / or their dK products to dk
      // (with_dk), in the same query order either way; a dV-only pass needs neither dP nor the tile's V.  The flags are
      // constants at every call, so each call compiles to its own loop.
      auto dkdv_pass = [&](bool with_dv, bool with_dk, float (&dv)[NKO][KSB][4], float (&dk)[NKO][KSB][4]) {
#pragma unroll
        for (int kb = 0; kb < NKO; ++kb)
#pragma unroll
          for (int nt = 0; nt < KSB; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              if (with_dv) dv[kb][nt][i] = 0.f;
              if (with_dk) dk[kb][nt][i] = 0.f;
            }
        consume([&](int blk, uint32_t buf) {
          const uint32_t q_s = buf, do_s = buf + L::SOP, st_s = buf + 2 * L::SOP;
          const int qbase = SBLK * blk, nq = min(SBLK, nq8 - qbase);
          // S^T, dP^T of the NB 8-query blocks q0, q0 + 8 (of the buffer)
          auto products = [&](auto nbc, int q0, float (&s)[2][4], float (&dp)[2][4]) {
            constexpr int NB = decltype(nbc)::value;
#pragma unroll
            for (int n = 0; n < NB; ++n)
#pragma unroll
              for (int i = 0; i < 4; ++i) s[n][i] = dp[n][i] = 0.f;
#pragma unroll
            for (int kb = 0; kb < NKB; ++kb) {
              uint32_t qb[NB][KSB][2], ob2[NB][KSB][2];
#pragma unroll
              for (int n = 0; n < NB; ++n) {
                ld_b_head<KSB>(q_s + kb * L::SSLAB, q0 + 8 * n, lane, qb[n]);
                if (with_dk) ld_b_head<KSB>(do_s + kb * L::SSLAB, q0 + 8 * n, lane, ob2[n]);
              }
#pragma unroll
              for (int ks = 0; ks < KSB; ++ks) {
                uint32_t ka[4], va[4];
                tfrag(0, kb, ks, ka);
                if (with_dk) tfrag(1, kb, ks, va);
#pragma unroll
                for (int n = 0; n < NB; ++n) {
                  rt(qb[n][ks][0]); rt(qb[n][ks][1]);
                  if (with_dk) { rt(ob2[n][ks][0]); rt(ob2[n][ks][1]); }
                  ptx::mma_tf32(s[n], ka, qb[n][ks]);
                  if (with_dk) ptx::mma_tf32(dp[n], va, ob2[n][ks]);
                }
              }
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
#pragma unroll
            for (int kb = 0; kb < NKO; ++kb) {
              const uint32_t do_b = do_s + (kb0 + kb) * L::SSLAB, q_b = q_s + (kb0 + kb) * L::SSLAB;
              uint32_t o0[KSB], o1[KSB], q0v[KSB], q1v[KSB];
              if (with_dv) { ld_b_out<KSB>(do_b, q0 + t, g, o0); ld_b_out<KSB>(do_b, q0 + t + 4, g, o1); }
              if (with_dk) { ld_b_out<KSB>(q_b, q0 + t, g, q0v); ld_b_out<KSB>(q_b, q0 + t + 4, g, q1v); }
#pragma unroll
              for (int nt = 0; nt < KSB; ++nt) {
                if (with_dv) {
                  rt(o0[nt]); rt(o1[nt]);
                  const uint32_t obv[2] = {o0[nt], o1[nt]};
                  ptx::mma_tf32(dv[kb][nt], pa, obv);
                }
                if (with_dk) {
                  rt(q0v[nt]); rt(q1v[nt]);
                  const uint32_t qbv[2] = {q0v[nt], q1v[nt]};
                  ptx::mma_tf32(dk[kb][nt], dsa, qbv);
                }
              }
            }
          };
          // two blocks in flight (DK 96, 128: one, or the accumulators spill)
          int q0 = 0;
          for (; q0 + 8 * DKDV_NB <= nq; q0 += 8 * DKDV_NB) {
            float s[2][4], dp[2][4];
            products(std::integral_constant<int, DKDV_NB>{}, q0, s, dp);
#pragma unroll
            for (int n = 0; n < DKDV_NB; ++n) accumulate(q0 + 8 * n, s[n], dp[n]);
          }
          if (q0 < nq) {
            float s[2][4], dp[2][4];
            products(std::integral_constant<int, 1>{}, q0, s, dp);
            accumulate(q0, s[0], dp[0]);
          }
        });
      };
      if constexpr (SPLIT) {
        // dK first, staged over the warp's own V rows (the dV pass reads only K), then dV over its K rows
        float acc[NKO][KSB][4];
        dkdv_pass(false, true, acc, acc);
        if (has) {
          store_wait();
          pair_sync();
          stage_strip(1, acc, scale);
        }
        dkdv_pass(true, false, acc, acc);
        if (has) {
          pair_sync();
          stage_strip(0, acc, 1.0f);
        }
      } else {
        float dv[NKO][KSB][4], dk[NKO][KSB][4];
        dkdv_pass(true, true, dv, dk);
        if (has) {
          store_wait();
          stage_strip(0, dv, 1.0f);
          stage_strip(1, dk, scale);
        }
      }
      if (has) {
        __syncwarp();
        if (live) { bias_add(0, 2 * d_model); bias_add(1, d_model); }
        store(2);
      }
      finish_tile();
    } else {
      // ===== 16 queries qA = 16 strip + g, qB = qA + 8: dQ over the streamed keys (attn_bwd_kernel's query strip)
      const int qA = 16 * strip + g, qB = qA + 8;
      float2 stA = make_float2(0.f, 0.f), stB = stA;
      if (live) {
        const float2* qst = reinterpret_cast<const float2*>(smem + 2 * L::TOP);
        stA = qst[r0 + g];
        stB = qst[r0 + g + 8];
        load_tile_frags(2);
      }
      if constexpr (!WIDE) release_tile();
      float dq[NKO][KSB][4];
#pragma unroll
      for (int kb = 0; kb < NKO; ++kb)
#pragma unroll
        for (int nt = 0; nt < KSB; ++nt) dq[kb][nt][0] = dq[kb][nt][1] = dq[kb][nt][2] = dq[kb][nt][3] = 0.f;
      const int nk8 = (it.e + 7) & ~7;     // keys at or beyond the extent are masked
      consume([&](int blk, uint32_t buf) {
        const uint32_t k_s = buf, v_s = buf + L::SOP, kb_s = buf + 2 * L::SOP;
        const int kbase = SBLK * blk, nk = min(SBLK, nk8 - kbase);
        // S, dP of the NB 8-key blocks k0, k0 + 8 (of the buffer)
        auto products = [&](auto nbc, int k0, float (&s)[2][4], float (&dp)[2][4]) {
          constexpr int NB = decltype(nbc)::value;
#pragma unroll
          for (int n = 0; n < NB; ++n)
#pragma unroll
            for (int i = 0; i < 4; ++i) s[n][i] = dp[n][i] = 0.f;
#pragma unroll
          for (int kb = 0; kb < NKB; ++kb) {
            uint32_t kbf[NB][KSB][2], vbf[NB][KSB][2];
#pragma unroll
            for (int n = 0; n < NB; ++n) {
              ld_b_head<KSB>(k_s + kb * L::SSLAB, k0 + 8 * n, lane, kbf[n]);
              ld_b_head<KSB>(v_s + kb * L::SSLAB, k0 + 8 * n, lane, vbf[n]);
            }
#pragma unroll
            for (int ks = 0; ks < KSB; ++ks) {
              uint32_t qa[4], oa[4];
              tfrag(0, kb, ks, qa);
              tfrag(1, kb, ks, oa);
#pragma unroll
              for (int n = 0; n < NB; ++n) {
                rt(kbf[n][ks][0]); rt(kbf[n][ks][1]); rt(vbf[n][ks][0]); rt(vbf[n][ks][1]);
                ptx::mma_tf32(s[n], qa, kbf[n][ks]);
                ptx::mma_tf32(dp[n], oa, vbf[n][ks]);
              }
            }
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
#pragma unroll
          for (int kb = 0; kb < NKO; ++kb) {
            const uint32_t k_b = k_s + (kb0 + kb) * L::SSLAB;
            uint32_t k0v[KSB], k1v[KSB];
            ld_b_out<KSB>(k_b, k0 + t, g, k0v); ld_b_out<KSB>(k_b, k0 + t + 4, g, k1v);
#pragma unroll
            for (int nt = 0; nt < KSB; ++nt) {
              rt(k0v[nt]); rt(k1v[nt]);
              const uint32_t kbv[2] = {k0v[nt], k1v[nt]};
              ptx::mma_tf32(dq[kb][nt], dsa, kbv);
            }
          }
        };
        // two blocks in flight (DK 256: one, or the fragments spill)
        int k0 = 0;
        for (; k0 + 8 * DQ_NB <= nk; k0 += 8 * DQ_NB) {
          float s[2][4], dp[2][4];
          products(std::integral_constant<int, DQ_NB>{}, k0, s, dp);
#pragma unroll
          for (int n = 0; n < DQ_NB; ++n) accumulate(k0 + 8 * n, s[n], dp[n]);
        }
        if (k0 < nk) {
          float s[2][4], dp[2][4];
          products(std::integral_constant<int, 1>{}, k0, s, dp);
          accumulate(k0, s[0], dp[0]);
        }
      });
      if (has) {
        store_wait();
        pair_sync();
        stage_strip(0, dq, scale);
        __syncwarp();
        if (live) bias_add(0, 0);
        store(1);
      }
      finish_tile();
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

static int long_items(int B, int h, int S, int blk) { return B * h * ((S + blk - 1) / blk); }

// Bytes the kernels request from L2 / HBM per (slate, head): the tile side once, the streamed side once per tile of
// blk rows (the ProfScope accounting; the streamed rows mostly hit L2)
static double long_bytes(int S, int dk, int blk, int tile_ops, int stream_ops, int out_ops) {
  const double tiles = (S + blk - 1) / blk;
  return 4.0 * S * dk * (tile_ops + out_ops + tiles * stream_ops);
}

// the instantiation that serves head width dk: 16 (4 ... 16), 32 (20 ... 32), or the next slab multiple (64, 96, 128),
// then 192 and 256
static int long_dk(int dk) {
  return dk <= 16 ? 16 : dk <= 32 ? 32 : dk <= 64 ? 64 : dk <= 96 ? 96 : dk <= 128 ? 128 : dk <= 192 ? 192 : 256;
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
  constexpr int blk = LongSmem<DK>::BLK;
  const int n_items = long_items(a.B, a.h, a.S, blk);
  dim3 grid(std::max(1, std::min(n_items, sm_count())));
  ProfScope ps(ARB_PROF_GEMM, (a.extent ? arb_attn_frac() : 1.0) * 4.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
               double(a.B) * a.h * (long_bytes(a.S, a.dk, blk, 1, 3, 1) + 8.0 * a.S), "attn_long_fwd_kernel");
  // d_model = h * dk: the paired kernels store no slab that lies wholly beyond the head width
  return launch(kern, grid, dim3(LONG_THREADS), size_t(LongSmem<DK>::total), st, /*pdl=*/true, tQ, tQ, tK, tV, tO, tO,
                a.mask, a.stat_max, a.stat_sum, static_cast<const float*>(nullptr), a.S, a.h, a.scale, a.drop,
                static_cast<float*>(nullptr), a.h * a.dk, a.extent, n_items, tf32_round_on_load());
}

int launch_attn_long_fwd(const AttnFwdArgs& a, cudaStream_t st) {
  if (a.o.bf16) { arb_set_error("attn_fwd: a bf16 context needs slate_length <= 256 and head width 8, 16, 24 or 32"); return ARB_E_UNSUPPORTED; }
  if (a.pack_off) { arb_set_error("attn_fwd: packed rows need slate_length <= 256 and head width <= 32 or 64"); return ARB_E_UNSUPPORTED; }
  switch (long_dk(a.dk)) {
    case 16: return launch_long_fwd_t<16>(a, st);
    case 32: return launch_long_fwd_t<32>(a, st);
    case 64: return launch_long_fwd_t<64>(a, st);
    case 96: return launch_long_fwd_t<96>(a, st);
    case 128: return launch_long_fwd_t<128>(a, st);
    case 192: return launch_long_fwd_t<192>(a, st);
    default: return launch_long_fwd_t<256>(a, st);
  }
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
  constexpr size_t smem = size_t(LongSmem<DK>::total);
  constexpr int blk = LongSmem<DK>::BLK;
  const int n_items = long_items(a.B, a.h, a.S, blk);
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
                 double(a.B) * a.h * (long_bytes(a.S, a.dk, blk, 2, 2, 2) + 8.0 * a.S), "attn_long_dkdv_kernel");
    if ((rc = launch(kdkdv, dim3(n_ctas), dim3(LONG_THREADS), smem, st, /*pdl=*/true, tK, tV, tQ,
                     tDO, tDV, tDK, a.mask, smax, ssum, a.delta, a.S, a.h, a.scale, a.drop, dbias, a.d_model, a.extent,
                     n_items, tf32_round_on_load())))
      return rc;
  }
  {
    ProfScope ps(ARB_PROF_GEMM, frac * 6.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
                 double(a.B) * a.h * (long_bytes(a.S, a.dk, blk, 2, 2, 1) + 12.0 * a.S), "attn_long_dq_kernel");
    if ((rc = launch(kdq, dim3(n_ctas), dim3(LONG_THREADS), smem, st, /*pdl=*/true, tQ, tDO, tK,
                     tV, tDQ, tDQ, a.mask, smax, ssum, a.delta, a.S, a.h, a.scale, a.drop, dbias, a.d_model, a.extent,
                     n_items, tf32_round_on_load())))
      return rc;
  }
  return dp.finish(st);
}

int launch_attn_long_bwd(const AttnBwdArgs& a, cudaStream_t st) {
  switch (long_dk(a.dk)) {
    case 16: return launch_long_bwd_t<16>(a, st);
    case 32: return launch_long_bwd_t<32>(a, st);
    case 64: return launch_long_bwd_t<64>(a, st);
    case 96: return launch_long_bwd_t<96>(a, st);
    case 128: return launch_long_bwd_t<128>(a, st);
    case 192: return launch_long_bwd_t<192>(a, st);
    default: return launch_long_bwd_t<256>(a, st);
  }
}

}  // namespace arb
