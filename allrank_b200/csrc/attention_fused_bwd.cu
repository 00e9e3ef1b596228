// Fused self-attention backward for slates of up to 256 items and head widths 4 ... 32 (on DK 16 or 32; other shapes:
// attention_long.cu).
//
// Reference: autograd of attention() allrank/models/transformer.py:137-156.  Given d ctx it produces dQ, dK, dV
// without ever materialising the S x S probabilities in HBM: they are recomputed from Q, K and the row statistics
// (max, sum) the fused forward kernel saved.  See attn_bwd_kernel for the organisation.
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>
#include <math_constants.h>

#include "attention_frag.cuh"
#include "attention_fused.h"
#include "block_utils.cuh"
#include "common.h"
#include "defaults.h"
#include "sm90_ptx.cuh"

namespace arb {

constexpr int BWD_WARPS = 8;                          // compute warps: one 16-row strip at a time each
constexpr int BWD_THREADS = 32 * (BWD_WARPS + 2);     // + one load warp, one store warp

// delta[b,h,q] = sum_e dO[b,q,h,e] * O[b,q,h,e]: one warp per row of the [B*S, d_model] activations, 128-bit loads,
// segmented shuffle reduction over the dk/4 lanes that share a head (dk in {4, 8, 16, 32, 64, 128}: 1, 2, 4, 8, 16 or
// 32 lanes per head); other widths (12 ... 28, 36 ... 124) reduce one head at a time over the whole warp.  Widths above
// 128: attn_delta_wide_kernel.
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
  if (dk & (dk - 1)) {
    // a width that is not a power of two (12 ... 28, 36 ... 124, dense rows): one head at a time, lane l takes its
    // columns 4l ... 4l + 3 (dk / 4 <= 31 lanes), reduced over the whole warp
    for (int head = 0; head < h; ++head) {
      const int c = head * dk + lane * 4;
      const bool on = lane < lanes_per_head;
#pragma unroll
      for (int q = 0; q < DELTA_RPW; ++q) {
        float acc = 0.f;
        if (on && item[q] >= 0) {
          const long long row = row0 + q;
          const float4 x = *reinterpret_cast<const float4*>(d_o + row * pitch + c);
          float4 y;
          if (o_bf16) {     // bf16 mode (width 24): the saved context is bfloat16
            const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(o) + row * pitch + c);
            y = make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                            __uint_as_float(u.y & 0xffff0000u));
          } else {
            y = *reinterpret_cast<const float4*>(o + row * pitch + c);
          }
          acc = x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
        }
        for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(FULL, acc, off);
        if (item[q] >= 0 && lane == 0) {
          const int b = int(item[q] / S), qi = int(item[q] - (long long)b * S);
          delta[((long long)b * h + head) * S + qi] = acc;
        }
      }
    }
    return;
  }
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

// delta at head widths 132 ... 256 (dense fp32 rows): one head at a time, lane l takes the head's 4-column groups l and
// l + 32 (columns 4l ... 4l + 3 and 128 + 4l ... 128 + 4l + 3, those below dk), summed in that order, then reduced
// over the whole warp.  Rows as attn_delta_kernel's.
__global__ void __launch_bounds__(256) attn_delta_wide_kernel(const float* __restrict__ d_o, const float* __restrict__ o,
                                                              long long pitch, int S, int h, int dk,
                                                              float* __restrict__ delta, const int* __restrict__ rows_dev,
                                                              const int* __restrict__ rowmap, long long rows_cap) {
  arb_pdl_wait();
  const int lane = threadIdx.x & 31;
  const long long row0 = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * DELTA_RPW;
  const long long rows = rows_dev ? min(rows_cap, (long long)__ldg(rows_dev)) : rows_cap;
  if (row0 >= rows) return;
  long long item[DELTA_RPW];
#pragma unroll
  for (int q = 0; q < DELTA_RPW; ++q) item[q] = (row0 + q < rows) ? (rowmap ? (long long)rowmap[row0 + q] : row0 + q) : -1;
  for (int head = 0; head < h; ++head) {
#pragma unroll
    for (int q = 0; q < DELTA_RPW; ++q) {
      float acc = 0.f;
      if (item[q] >= 0) {
        const long long row = row0 + q;
#pragma unroll
        for (int grp = 0; grp < 2; ++grp) {
          const int col = 128 * grp + 4 * lane;
          if (col < dk) {
            const float4 x = *reinterpret_cast<const float4*>(d_o + row * pitch + head * dk + col);
            const float4 y = *reinterpret_cast<const float4*>(o + row * pitch + head * dk + col);
            acc += x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
          }
        }
      }
      for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(FULL, acc, off);
      if (item[q] >= 0 && lane == 0) {
        const int b = int(item[q] / S), qi = int(item[q] - (long long)b * S);
        delta[((long long)b * h + head) * S + qi] = acc;
      }
    }
  }
}

constexpr int BOX_BYTES = 16 * 128;       // one 16-row box of 128-byte rows
constexpr int ITEM_ROW_BYTES = 4 * 128;   // Q, K, V, dO of one item row
constexpr int POOL_ROWS_MAX = 352;        // item rows of the operand pool: two items of MSLR-shaped slates fit
constexpr int RING = 12;                  // staging slots, one finished unit each: dV | dK of a key strip, or dQ
constexpr int RING_BYTES = 2 * BOX_BYTES;
constexpr int STORE_LAG = 4;              // store groups the store warp leaves reading before it frees their slots

struct BwdSmem {
  // [operand pool: pool_rows x (Q | K | V | dO) rows] [staging ring: RING x two 16-row boxes] [zero box]
  // [float2 stats: 2 slots x 256] [key bits: 2 slots x 8 words] [mbarriers: full[2] ready[2] empty[2] staged[RING]
  // freed[RING]] [QKV bias gradient: 3 * d_model floats]
  __host__ __device__ static int stage_off(int pool_rows) { return pool_rows * ITEM_ROW_BYTES; }
  __host__ __device__ static int zero_off(int pool_rows) { return stage_off(pool_rows) + RING * RING_BYTES; }
  __host__ __device__ static int stats_off(int pool_rows) { return zero_off(pool_rows) + BOX_BYTES; }
  __host__ __device__ static int bits_off(int pool_rows) { return stats_off(pool_rows) + 2 * 256 * 8; }
  __host__ __device__ static int bars_off(int pool_rows) { return bits_off(pool_rows) + 64; }
  __host__ __device__ static int bias_off(int pool_rows) { return bars_off(pool_rows) + 8 * (6 + 2 * RING); }
  __host__ __device__ static int total(int pool_rows, int d_model) { return bias_off(pool_rows) + 12 * d_model + 1024; }
};

// One CTA walks the (slate, head) items blockIdx.x, blockIdx.x + gridDim.x, ... (one CTA per item, or -- persistent --
// one per SM), with three warp roles.
//
// The load warp (warp BWD_WARPS) TMA-loads an item's Q, K, V, dO rows below round_up(extent, 16) in 16-row boxes into
// an operand pool that holds two items: even items of the CTA from its bottom, odd ones from its top.  The next item's
// loads go out as soon as the previous user of its pool slot is done, and -- when the two items do not fit side by
// side -- the current one too.  For each item it writes the slot's key bits and per-query {nm, delta}, stores the zero
// boxes past the extent (dense layout), waits for the loads (full[slot]), rounds the operands to tf32 in place and
// marks the slot ready (ready[slot]).
//
// The compute warps (0 ... BWD_WARPS - 1) run work units.  The units of an item are, per 128-row tile, its key strips
// (dK, dV) and then its query strips (dQ) of 16 rows below round_up(extent, 16).  The units of all of the CTA's items
// form one sequence dealt round-robin to the compute warps, so a warp with no unit left in an item arrives on
// empty[slot] and goes on with the next item's units as soon as that item is ready.  A unit runs on the tensor cores
// (mma.sync m16n8k8 tf32) with its products in registers, two 8-row blocks in flight:
//   key strip (16 keys):      S^T = K Q^T, dP^T = V dO^T over 8-query blocks, P^T = exp2(S^T c + nm_q) (key mask,
//                             dropout), dS^T = P^T * (dP^T - delta_q), dV += P^T dO, dK += dS^T Q
//   query strip (16 queries): S = Q K^T, dP = dO V^T over 8-key blocks, dS as above, dQ += dS K
// with nm_q = -max_q c - log2 l_q from the forward's row statistics and c = log2(e) / sqrt(dk).  The warp stages its
// finished unit in slot (sequence number % RING) of the staging ring and hands it to the store warp (staged[]).
//
// The store warp (warp BWD_WARPS + 1) takes the units in sequence order: it adds the staged rows to its running column
// sums for the QKV bias gradient (lane c: column c of dV, dK and dQ; each output's rows of a tile in order, added to
// the CTA's accumulator tile by tile), TMA-stores the unit as 16-row boxes and frees the slot (freed[]) once the store
// has read it.  It never waits on the operand pool, so staging cannot deadlock against loading.
template <int DK, bool DROP, bool OUT16 = false>
__global__ void __launch_bounds__(BWD_THREADS, 1) attn_bwd_kernel(
    const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmDO,
    const __grid_constant__ CUtensorMap tmDQ, const __grid_constant__ CUtensorMap tmDK,
    const __grid_constant__ CUtensorMap tmDV, const uint8_t* __restrict__ mask, const float* __restrict__ stat_max,
    const float* __restrict__ stat_sum, const float* __restrict__ delta, int S, int n_heads, float scale, DropSite drop,
    float* __restrict__ dbias_qkv, int d_model, const int* __restrict__ extent, const int* __restrict__ pack_off,
    int n_items, int rnd, int pool_rows) {
  constexpr int KS = DK / 8;
  extern __shared__ __align__(1024) uint8_t smem_dyn[];
  const uint32_t sbase = (ptx::smem_u32(smem_dyn) + 1023u) & ~1023u;
  uint8_t* smem = smem_dyn + (sbase - ptx::smem_u32(smem_dyn));
  const uint32_t stats_s = sbase + BwdSmem::stats_off(pool_rows), bits_s = sbase + BwdSmem::bits_off(pool_rows);
  float2* qstats = reinterpret_cast<float2*>(smem + BwdSmem::stats_off(pool_rows));    // [slot][256]
  uint32_t* key_bits = reinterpret_cast<uint32_t*>(smem + BwdSmem::bits_off(pool_rows));   // [slot][8]
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + BwdSmem::bars_off(pool_rows));
  uint64_t* ready = full + 2;
  uint64_t* empty = full + 4;
  uint64_t* staged = full + 6;
  uint64_t* freed = staged + RING;
  uint8_t* zero_box = smem + BwdSmem::zero_off(pool_rows);
  float* bias_acc = reinterpret_cast<float*>(smem + BwdSmem::bias_off(pool_rows));
  uint8_t* stage = smem + BwdSmem::stage_off(pool_rows);
  const uint32_t stage_s = sbase + BwdSmem::stage_off(pool_rows);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const float c_log2e = scale * 1.4426950408889634f;
  const bool packed = pack_off != nullptr;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ); ptx::prefetch_tmap(&tmK); ptx::prefetch_tmap(&tmV); ptx::prefetch_tmap(&tmDO);
    for (int s = 0; s < 2; ++s) {
      ptx::mbar_init(full + s, 1);
      ptx::mbar_init(ready + s, 32);
      ptx::mbar_init(empty + s, BWD_WARPS);
    }
    for (int r = 0; r < RING; ++r) {
      ptx::mbar_init(staged + r, 1);
      ptx::mbar_init(freed + r, 1);
    }
    ptx::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < BOX_BYTES / 16; i += BWD_THREADS) reinterpret_cast<uint4*>(zero_box)[i] = make_uint4(0u, 0u, 0u, 0u);
  if (dbias_qkv != nullptr)
    for (int i = threadIdx.x; i < 3 * d_model; i += BWD_THREADS) bias_acc[i] = 0.f;
  ptx::fence_proxy_async_smem();
  arb_pdl_wait();
  __syncthreads();

  // Rows at or beyond a slate's extent are masked keys (probability exactly 0) whose d ctx rows are exactly zero:
  // neither their key strips nor their query strips contribute anything, and their dQ / dK / dV rows are zero.  Only
  // the strips below round_up(extent, 16) are processed; in the dense layout the rows beyond are written as zeros.
  // Packed rows (see attn_fwd_kernel): slate b holds its first ext16 = round_up(extent, 16) rows at row pack_off[b] of
  // one long tensor -- exactly the rows loaded and stored here.  Its queries at or beyond S get probability zero
  // through their statistics (-inf).
  struct Item { int b, head, e, rows, q_lim, q_live, row_base, bc; };
  auto item_info = [&](int item) {
    Item it{};
    it.b = item / n_heads;
    it.head = item - it.b * n_heads;
    int e = extent ? __ldg(extent + it.b) : S;
    if (packed && e <= 0) return it;            // packed rows: an empty slate holds no rows (rows = 0: skipped)
    e = max(1, min(S, e));
    it.e = e;
    it.rows = (e + 15) & ~15;
    it.q_lim = packed ? min(S, it.rows) : S;    // queries at or beyond it do not exist in this slate
    // queries at or beyond q_live contribute nothing (the dense layout's padding has zero d ctx rows; packed rows: the
    // slate has no such queries)
    it.q_live = packed ? it.q_lim : (extent ? e : S);
    it.row_base = packed ? __ldg(pack_off + it.b) : 0;
    it.bc = packed ? 0 : it.b;
    return it;
  };
  auto next_item = [&](int item) {
    while (item < n_items && item_info(item).rows == 0) item += gridDim.x;
    return item;
  };
  // pool offset of an item's rows: slot 0 from the bottom, slot 1 from the top
  auto region_off = [&](int slot, int rows) { return slot ? (pool_rows - rows) * ITEM_ROW_BYTES : 0; };

  if (warp == BWD_WARPS) {
    // ===== load warp
    // an item's Q, K, V, dO rows in 16-row boxes (operand o at region + o * rows * 128), completing on full[slot]
    auto issue_loads = [&](const Item& it, int slot) {
      const int nb = it.rows >> 4;
      uint8_t* region = smem + region_off(slot, it.rows);
      ptx::fence_proxy_async_smem();
      if (lane == 0) ptx::mbar_expect_tx(full + slot, uint32_t(it.rows) * ITEM_ROW_BYTES);
      __syncwarp();
      for (int j = lane; j < 4 * nb; j += 32) {
        const int o = j / nb, i = j - o * nb;
        const CUtensorMap* m = o == 0 ? &tmQ : (o == 1 ? &tmK : (o == 2 ? &tmV : &tmDO));
        ptx::tma_load_4d(region + (o * it.rows + 16 * i) * 128, m, full + slot, 0, it.row_base + 16 * i, it.head, it.bc);
      }
    };
    // the slot's key bits and per-query statistics (nm = -max*c - log2(sum); -inf for queries the slate does not
    // have), the dense layout's zero rows; once the item has landed, its operands rounded to tf32 in place (nearest
    // even, as the products would on each use); then the slot is ready (every lane arrives after its own stores)
    auto prepare = [&](const Item& it, int slot, uint32_t parity) {
      bool live[8];
      float mx[8], sm[8], dl[8];
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const int qi = 32 * w + lane;
        live[w] = qi < S && mask[size_t(it.b) * S + qi] == 0;
        mx[w] = 0.f; sm[w] = 1.f; dl[w] = 0.f;
        if (qi < it.q_lim) {
          const size_t so = (size_t(it.b) * n_heads + it.head) * S + qi;
          mx[w] = stat_max[so];
          sm[w] = stat_sum[so];
          dl[w] = delta[so];
        }
      }
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const int qi = 32 * w + lane;
        float2 st = make_float2(-CUDART_INF_F, 0.f);
        if (qi < it.q_lim) st = make_float2(-(mx[w] * c_log2e) - log2f(sm[w]), dl[w]);
        qstats[256 * slot + qi] = st;
        const uint32_t bw = __ballot_sync(FULL, live[w]);
        if (lane == 0) key_bits[8 * slot + w] = bw;
      }
      if (!packed && it.rows < S) {
        // dense layout: rows at or beyond round_up(extent, 16) are zero -- one zero box, TMA-stored over every such
        // 16-row box of dQ, dK and dV (TMA clips at S)
        const int z0 = it.rows >> 4, nz = (S + 15) / 16 - z0;
        for (int j = lane; j < 3 * nz; j += 32) {
          const int o = j / nz, i = z0 + j - o * nz;
          ptx::tma_store_4d(o == 0 ? &tmDQ : (o == 1 ? &tmDK : &tmDV), zero_box, 0, 16 * i, it.head, it.b);
        }
        ptx::tma_store_commit();
      }
      ptx::mbar_wait(full + slot, parity);
      if (rnd) {
        uint4* p = reinterpret_cast<uint4*>(smem + region_off(slot, it.rows));
        const int n = it.rows * (ITEM_ROW_BYTES / 16);
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
    if (item < n_items) {
      Item cur = item_info(item);
      issue_loads(cur, 0);
      for (int k = 0;; ++k) {
        const int slot = k & 1;
        prepare(cur, slot, (k >> 1) & 1);
        const int nitem = next_item(item + gridDim.x);
        if (nitem >= n_items) break;
        const Item nxt = item_info(nitem);
        // the next item's slot must be free (its previous user, item k - 1, done), and item k done as well when the
        // two items do not fit side by side
        if (k >= 1) ptx::mbar_wait(empty + (slot ^ 1), ((k - 1) >> 1) & 1);
        if (cur.rows + nxt.rows > pool_rows) ptx::mbar_wait(empty + slot, (k >> 1) & 1);
        issue_loads(nxt, slot ^ 1);
        cur = nxt;
        item = nitem;
      }
    }
    ptx::tma_store_wait_all();
    return;
  }

  if (warp == BWD_WARPS + 1) {
    // ===== store warp
    // running column sum over a staged 16-row box, rows in order
    auto colsum = [&](const uint8_t* box, float s) {
      float v[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        if constexpr (OUT16) v[r] = __uint_as_float(uint32_t(*reinterpret_cast<const uint16_t*>(box + r * 64 + lane * 2)) << 16);
        else v[r] = *reinterpret_cast<const float*>(box + ptx::sw128(r, 4 * lane));
      }
#pragma unroll
      for (int r = 0; r < 16; ++r) s += v[r];
      return s;
    };
    // lane c sums column c of the head's w real columns (w < DK: the staged columns past w are zeros, never stored)
    const int w = d_model / n_heads;
    const bool sums = dbias_qkv != nullptr && lane < w;
    int seq = 0;
    for (int item = next_item(blockIdx.x); item < n_items; item = next_item(item + gridDim.x)) {
      const Item it = item_info(item);
      const int n = it.rows >> 4;
      for (int tile = 0; 8 * tile < n; ++tile) {
        const int ns = min(8, n - 8 * tile);
        // bias gradient of the QKV projection: per output column, the tile's rows (dQ / dK / dV values as stored) in
        // order, then added to the CTA's accumulator tile by tile
        float sv = 0.f, sk = 0.f, sq = 0.f;
        for (int l = 0; l < 2 * ns; ++l, ++seq) {
          const int rs = seq % RING;
          ptx::mbar_wait(staged + rs, (seq / RING) & 1);
          const uint8_t* box = stage + rs * RING_BYTES;
          const bool key = l < ns;
          if (sums) {
            if (key) { sv = colsum(box, sv); sk = colsum(box + BOX_BYTES, sk); }
            else sq = colsum(box, sq);
          }
          __syncwarp();
          if (lane == 0) {
            const int r = it.row_base + 16 * (8 * tile + (key ? l : l - ns));
            if (key) {
              ptx::tma_store_4d(&tmDV, box, 0, r, it.head, it.bc);
              ptx::tma_store_4d(&tmDK, box + BOX_BYTES, 0, r, it.head, it.bc);
            } else {
              ptx::tma_store_4d(&tmDQ, box, 0, r, it.head, it.bc);
            }
            ptx::tma_store_commit();
            if (seq >= STORE_LAG) {
              ptx::tma_store_wait_read<STORE_LAG>();
              ptx::mbar_arrive(freed + (seq - STORE_LAG) % RING);
            }
          }
        }
        if (sums) {
          bias_acc[2 * d_model + it.head * w + lane] += sv;
          bias_acc[d_model + it.head * w + lane] += sk;
          bias_acc[it.head * w + lane] += sq;
        }
      }
    }
    if (dbias_qkv != nullptr) {
      // this CTA's slot of the bias gradient (its items in a fixed order; the slots are summed in order by DetParts)
      __syncwarp();
      for (int i = lane; i < 3 * d_model; i += 32) dbias_qkv[size_t(blockIdx.x) * 3 * d_model + i] = bias_acc[i];
    }
    if (lane == 0) ptx::tma_store_wait_all();
    return;
  }

  // ===== compute warps
  if constexpr (DROP) drop.seed = drop_seed(drop);
  // a finished strip of one output (rows g, g + 8 of its accumulator, x mul) into the 16-row staging box at `box`
  auto stage_strip = [&](uint32_t box, const float (&acc)[KS][4], float mul) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = g + 8 * h;
      float v[2][KS];      // v[0]: head columns of output column 2t, v[1]: of 2t + 1 (n-tile order)
#pragma unroll
      for (int nt = 0; nt < KS; ++nt) { v[0][nt] = acc[nt][2 * h] * mul; v[1][nt] = acc[nt][2 * h + 1] * mul; }
      if constexpr (OUT16) {
        // bf16 mode: dQ / dK / dV only feed the QKV weight- and input-gradient products: dense bfloat16 rows of 32
        // columns (64 bytes), unswizzled tensor maps
        if constexpr (KS == 4) {
          sts64(box + r * 64 + 8 * t, make_uint2(ptx::pack_bf16(v[0][0], v[0][1]), ptx::pack_bf16(v[0][2], v[0][3])));
          sts64(box + r * 64 + 32 + 8 * t, make_uint2(ptx::pack_bf16(v[1][0], v[1][1]), ptx::pack_bf16(v[1][2], v[1][3])));
        } else {
          sts64(box + r * 64 + 8 * t, make_uint2(ptx::pack_bf16(v[0][0], v[0][1]), ptx::pack_bf16(v[1][0], v[1][1])));
        }
      } else {
        if constexpr (KS == 4) {
          sts128(box + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[0][2]), __float_as_uint(v[0][3])));
          sts128(box + ptx::sw128(r, 64 + 16 * t), make_uint4(__float_as_uint(v[1][0]), __float_as_uint(v[1][1]), __float_as_uint(v[1][2]), __float_as_uint(v[1][3])));
        } else {
          sts128(box + ptx::sw128(r, 16 * t), make_uint4(__float_as_uint(v[0][0]), __float_as_uint(v[0][1]), __float_as_uint(v[1][0]), __float_as_uint(v[1][1])));
        }
      }
    }
  };
  // the staging slot of unit `seq` of the CTA's sequence, once the store warp has freed it
  auto staging_slot = [&](int seq) {
    ptx::mbar_wait(freed + seq % RING, ((seq / RING) & 1) ^ 1);
    return stage_s + (seq % RING) * RING_BYTES;
  };
  // hand the staged unit to the store warp (every lane's stores visible to the TMA engine first)
  auto hand_over = [&](int seq) {
    ptx::fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(staged + seq % RING);
  };

  int k = 0, dealt = 0;     // dealt: units of the CTA's earlier items
  for (int item = next_item(blockIdx.x); item < n_items; item = next_item(item + gridDim.x), ++k) {
    const Item cur = item_info(item);
    const int slot = k & 1, n = cur.rows >> 4;
    ptx::mbar_wait(ready + slot, (k >> 1) & 1);
    const uint32_t q_s = sbase + region_off(slot, cur.rows), k_s = q_s + cur.rows * 128, v_s = k_s + cur.rows * 128,
                   do_s = v_s + cur.rows * 128;
    const uint32_t st_s = stats_s + slot * 256 * 8, kb_s = bits_s + slot * 32;
    const float2* qst = qstats + 256 * slot;
    const unsigned long long dbase = (unsigned long long)(cur.b * n_heads + cur.head) * S;
    // units of a 128-row tile: its ns key strips, then its ns query strips
    for (int u = (warp - dealt) & (BWD_WARPS - 1); u < 2 * n; u += BWD_WARPS) {
      const int tile = u >> 4, l = u & 15, ns = min(8, n - 8 * tile), seq = dealt + u;
      if (l < ns) {
        // ===== key strip: dV, dK of keys kA = 16 strip + g, kB = kA + 8
        const int strip = 8 * tile + l, kA = 16 * strip + g, kB = kA + 8;
        const uint32_t kw = lds32(kb_s + 4 * (strip >> 1));
        const bool liveA = (kw >> (kA & 31)) & 1u, liveB = (kw >> (kB & 31)) & 1u;
        uint32_t ka[KS][4], va[KS][4];
        ld_a_head<KS>(k_s, 16 * strip, lane, ka);
        ld_a_head<KS>(v_s, 16 * strip, lane, va);
        float dv[KS][4], dk[KS][4];
#pragma unroll
        for (int nt = 0; nt < KS; ++nt)
#pragma unroll
          for (int i = 0; i < 4; ++i) dv[nt][i] = dk[nt][i] = 0.f;
        // S^T, dP^T of the 8-query block q0
        auto products = [&](int q0, float (&s)[4], float (&dp)[4]) {
#pragma unroll
          for (int i = 0; i < 4; ++i) s[i] = dp[i] = 0.f;
          uint32_t qb[KS][2], ob[KS][2];
          ld_b_head<KS>(q_s, q0, lane, qb);
          ld_b_head<KS>(do_s, q0, lane, ob);
#pragma unroll
          for (int ks = 0; ks < KS; ++ks) {
            ptx::mma_tf32(s, ka[ks], qb[ks]);
            ptx::mma_tf32(dp, va[ks], ob[ks]);
          }
        };
        // P^T, dS^T of the block and its dV, dK products
        auto accumulate = [&](int q0, const float (&s)[4], const float (&dp)[4]) {
          // accumulator columns 2t, 2t + 1 are queries q0 + t, q0 + t + 4: their {nm, delta}
          const uint2 st0 = lds64(st_s + 8 * (q0 + t)), st1 = lds64(st_s + 8 * (q0 + t + 4));
          float pu[4], ds[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int q = q0 + t + 4 * (i & 1);
            const float nm = __uint_as_float((i & 1) ? st1.x : st0.x), dl = __uint_as_float((i & 1) ? st1.y : st0.y);
            const float p = (i < 2 ? liveA : liveB) ? ex2_approx(fmaf(s[i], c_log2e, nm)) : 0.0f;
            float p_used = p, dpv = dp[i];
            if constexpr (DROP) {        // regenerate the forward's dropout mask on the probabilities
              const unsigned long long idx = (dbase + q) * (unsigned long long)S + (i < 2 ? kA : kB);
              const float m = drop_keep(idx, drop.seed, drop.thresh) ? drop.scale : 0.0f;
              p_used = p * m;
              dpv *= m;
            }
            pu[i] = round_tf32(p_used);
            ds[i] = round_tf32(p * (dpv - dl));
          }
          // the accumulators {rows g, g+8} x {queries t, t+4} are the A fragments over k-slots {t, t+4}
          const uint32_t pa[4] = {__float_as_uint(pu[0]), __float_as_uint(pu[2]), __float_as_uint(pu[1]), __float_as_uint(pu[3])};
          const uint32_t dsa[4] = {__float_as_uint(ds[0]), __float_as_uint(ds[2]), __float_as_uint(ds[1]), __float_as_uint(ds[3])};
          uint32_t o0[KS], o1[KS], q0v[KS], q1v[KS];
          ld_b_out<KS>(do_s, q0 + t, g, o0); ld_b_out<KS>(do_s, q0 + t + 4, g, o1);
          ld_b_out<KS>(q_s, q0 + t, g, q0v); ld_b_out<KS>(q_s, q0 + t + 4, g, q1v);
#pragma unroll
          for (int nt = 0; nt < KS; ++nt) {
            const uint32_t ob[2] = {o0[nt], o1[nt]}, qb[2] = {q0v[nt], q1v[nt]};
            ptx::mma_tf32(dv[nt], pa, ob);
            ptx::mma_tf32(dk[nt], dsa, qb);
          }
        };
        // two blocks in flight: block j + 1's S^T, dP^T go out before block j's exponentials and products
        const int nq8 = (cur.q_live + 7) & ~7;
        int q0 = 0;
        for (; q0 + 16 <= nq8; q0 += 16) {
          float s0[4], dp0[4], s1[4], dp1[4];
          products(q0, s0, dp0);
          products(q0 + 8, s1, dp1);
          accumulate(q0, s0, dp0);
          accumulate(q0 + 8, s1, dp1);
        }
        if (q0 < nq8) {
          float s0[4], dp0[4];
          products(q0, s0, dp0);
          accumulate(q0, s0, dp0);
        }
        const uint32_t box = staging_slot(seq);
        stage_strip(box, dv, 1.0f);
        stage_strip(box + BOX_BYTES, dk, scale);
        hand_over(seq);
      } else {
        // ===== query strip: dQ of queries qA = 16 strip + g, qB = qA + 8
        const int strip = 8 * tile + l - ns, qA = 16 * strip + g, qB = qA + 8;
        float dq[KS][4];
#pragma unroll
        for (int nt = 0; nt < KS; ++nt) dq[nt][0] = dq[nt][1] = dq[nt][2] = dq[nt][3] = 0.f;
        if (16 * strip < cur.q_live) {
          const float2 stA = qst[qA], stB = qst[qB];
          uint32_t qa[KS][4], oa[KS][4];
          ld_a_head<KS>(q_s, 16 * strip, lane, qa);
          ld_a_head<KS>(do_s, 16 * strip, lane, oa);
          // S, dP of the 8-key block k0
          auto products = [&](int k0, float (&s)[4], float (&dp)[4]) {
#pragma unroll
            for (int i = 0; i < 4; ++i) s[i] = dp[i] = 0.f;
            uint32_t kb[KS][2], vb[KS][2];
            ld_b_head<KS>(k_s, k0, lane, kb);
            ld_b_head<KS>(v_s, k0, lane, vb);
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) {
              ptx::mma_tf32(s, qa[ks], kb[ks]);
              ptx::mma_tf32(dp, oa[ks], vb[ks]);
            }
          };
          // dS of the block and its dQ products
          auto accumulate = [&](int k0, const float (&s)[4], const float (&dp)[4]) {
            // accumulator columns 2t, 2t + 1 are keys k0 + t, k0 + t + 4
            const uint32_t kw = lds32(kb_s + 4 * (k0 >> 5)) >> ((k0 & 31) + t);
            float ds[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int key = k0 + t + 4 * (i & 1);
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
              const uint32_t kb[2] = {k0v[nt], k1v[nt]};
              ptx::mma_tf32(dq[nt], dsa, kb);
            }
          };
          const int nk8 = (cur.e + 7) & ~7;          // keys at or beyond the extent are masked
          int k0 = 0;
          for (; k0 + 16 <= nk8; k0 += 16) {
            float s0[4], dp0[4], s1[4], dp1[4];
            products(k0, s0, dp0);
            products(k0 + 8, s1, dp1);
            accumulate(k0, s0, dp0);
            accumulate(k0 + 8, s1, dp1);
          }
          if (k0 < nk8) {
            float s0[4], dp0[4];
            products(k0, s0, dp0);
            accumulate(k0, s0, dp0);
          }
        }
        const uint32_t box = staging_slot(seq);
        stage_strip(box, dq, scale);
        hand_over(seq);
      }
    }
    // this warp is done with the item's operands, statistics and key bits
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(empty + slot);
    dealt += 2 * n;
  }
}

static int g_attn_bwd_persistent = ARB_DEFAULT_ATTN_BWD_PERSISTENT;
void set_attn_bwd_persistent(int on) { g_attn_bwd_persistent = on; }

// delta = rowsum(dO * O) per (slate, head, query), for either backward
static int launch_delta(const AttnBwdArgs& a, cudaStream_t st) {
  const bool packed = a.pack_off != nullptr;
  const double rf = packed ? arb_row_frac() : 1.0;
  ProfScope ps(ARB_PROF_SCORER_SIMT, rf * double(a.B) * a.S * (8.0 * a.h * a.dk + 4.0 * a.h), st, 0.0, "attn_delta_kernel");
  const long long rows = packed ? (long long)a.q.dim[1] : (long long)a.B * a.S;   // packed: the buffers' row count
  if (a.dk > 128) {
    if (a.o_bf16) { arb_set_error("attn_delta: a bf16 context needs head width <= 128"); return ARB_E_UNSUPPORTED; }
    return launch(attn_delta_wide_kernel, dim3(unsigned((rows + 8 * DELTA_RPW - 1) / (8 * DELTA_RPW))), dim3(256), 0,
                  st, /*pdl=*/true, a.do_ptr, static_cast<const float*>(a.o_ptr), (long long)a.o_pitch, a.S, a.h, a.dk,
                  a.delta, a.rows_dev, a.rowmap, rows);
  }
  return launch(attn_delta_kernel, dim3(unsigned((rows + 8 * DELTA_RPW - 1) / (8 * DELTA_RPW))), dim3(256), 0, st,
                /*pdl=*/true, a.do_ptr, static_cast<const float*>(a.o_ptr), (long long)a.o_pitch, a.B, a.S, a.h,
                a.dk, a.delta, a.o_bf16, a.rows_dev, a.rowmap, rows);
}

template <int DK>
static int launch_bwd_t(const AttnBwdArgs& a, cudaStream_t st) {
  alignas(64) CUtensorMap tQ, tK, tV, tDO, tDQ, tDK, tDV;
  int rc;
  const TmapBox box{{32, 16, 1, 1}};
  if ((rc = make_tmap_4d(&tQ, a.q, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tK, a.k, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tV, a.v, box, 0))) return rc;
  if ((rc = make_tmap_4d(&tDO, a.d_o, box, 0))) return rc;
  const bool out16 = a.dq.bf16 != 0;
  if ((a.dk_.bf16 != 0) != out16 || (a.dv.bf16 != 0) != out16) { arb_set_error("attn_bwd: dQ, dK, dV must share an element type"); return ARB_E_INVALID_ARG; }
  const bool packed = a.pack_off != nullptr;
  if (packed && !(a.extent && a.rows_dev && a.rowmap)) { arb_set_error("attn_bwd: packed rows need the extents, the row count and the row map"); return ARB_E_INVALID_ARG; }
  if ((rc = make_tmap_4d(&tDQ, a.dq, box, out16 ? 1 : 0))) return rc;
  if ((rc = make_tmap_4d(&tDK, a.dk_, box, out16 ? 1 : 0))) return rc;
  if ((rc = make_tmap_4d(&tDV, a.dv, box, out16 ? 1 : 0))) return rc;
  const double rf = packed ? arb_row_frac() : 1.0;
  if ((rc = launch_delta(a, st))) return rc;
  const bool drop = a.drop.thresh != 0;
  auto kern = out16 ? (drop ? attn_bwd_kernel<DK, true, true> : attn_bwd_kernel<DK, false, true>)
                    : (drop ? attn_bwd_kernel<DK, true> : attn_bwd_kernel<DK, false>);
  // the operand pool takes what the 227 KB of shared memory leave, up to POOL_ROWS_MAX; it must hold one whole slate
  const int d_bias = a.dbias_qkv ? a.d_model : 0;
  const int pool_rows = std::min(POOL_ROWS_MAX, ((227 * 1024 - BwdSmem::total(0, d_bias)) / ITEM_ROW_BYTES) & ~15);
  if (pool_rows < ((a.S + 15) & ~15)) { arb_set_error("attn_bwd: d_model too large for the shared-memory operand pool"); return ARB_E_UNSUPPORTED; }
  const int smem = BwdSmem::total(pool_rows, d_bias);
  // one CTA per (slate, head), or -- persistent (default) -- one per SM walking the items head-fastest and loading
  // the next item while it computes the current one
  const int n_items = a.h * a.B;
  const int n_ctas = g_attn_bwd_persistent ? std::min(n_items, sm_count()) : n_items;
  dim3 grid(n_ctas);
  // the QKV bias gradient: one slot per CTA, summed in CTA order afterwards
  float* dbias = a.dbias_qkv;
  DetParts dp;
  dp.add(dbias, n_ctas, 1, 3LL * a.d_model, 3LL * a.d_model);
  if ((rc = dp.begin(st))) return rc;
  {
    ProfScope ps(ARB_PROF_GEMM, (a.extent ? arb_attn_frac() : 1.0) * 10.0 * double(a.S) * a.S * a.dk * a.h * a.B, st,
                 rf * 4.0 * double(a.B) * a.h * a.S * (7.0 * a.dk + 3.0), "attn_bwd_kernel");
    if ((rc = launch(kern, grid, dim3(BWD_THREADS), size_t(smem), st, /*pdl=*/true, tQ, tK, tV, tDO, tDQ, tDK, tDV,
                     a.mask, a.stat_max, a.stat_sum, a.delta, a.S, a.h, a.scale, a.drop, dbias, a.d_model, a.extent,
                     a.pack_off, n_items, tf32_round_on_load(), pool_rows)))
      return rc;
  }
  return dp.finish(st);
}


// head widths 4 ... 256 in steps of 4: S <= 256 at widths up to 32 here (below 16 on DK 16, 20 ... 28 on DK 32, with
// tensor maps of the real width), the rest in attention_long.cu
bool attn_fused_bwd_supported(int S, int dk) {
  return S >= 1 && S <= 4096 && dk >= 4 && dk <= 256 && dk % 4 == 0;
}

int launch_attn_bwd(const AttnBwdArgs& a, cudaStream_t st) {
  if (!attn_fused_bwd_supported(a.S, a.dk)) { arb_set_error("fused attention backward: unsupported shape"); return ARB_E_UNSUPPORTED; }
  // the long kernels: slates beyond 256 items, and every width above 32 (whose statistics the short forward writes in
  // the same [B, h, S] format at width 64)
  if (a.S > 256 || a.dk > 32) {
    if (a.o_bf16 || a.dq.bf16 || a.dk_.bf16 || a.dv.bf16 || a.pack_off) {
      arb_set_error("fused attention backward: bf16 operands and packed rows need slate_length <= 256 and head width <= 32");
      return ARB_E_UNSUPPORTED;
    }
    int rc = launch_delta(a, st);
    return rc ? rc : launch_attn_long_bwd(a, st);
  }
  // the same DK as attention_long.cu's long_dk, so a slate gets the same bits from either
  return a.dk <= 16 ? launch_bwd_t<16>(a, st) : launch_bwd_t<32>(a, st);
}

}  // namespace arb
