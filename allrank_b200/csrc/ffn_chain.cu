// The encoder's feed-forward linears chained on chip, one kernel per direction:
//
//   Y = epi2( sum_j epi1( X A_j^T ) B_j^T )      j = 64-unit chunks of the hidden layer, in increasing order
//
//   forward         X = LN(x) [rows, d]   A = W1 [d_ff, d]    B = W2 [d, d_ff]
//                   epi1: + b1, ReLU, ReLU bit words, H -> hidden buffer;  epi2: + b2 + residual
//   input gradient  X = dY [rows, d]      A = W2^T [d_ff, d]  B = W1^T [d, d_ff]
//                   epi1: mask by the forward's bit words, dH -> hidden buffer, b1 gradient column sums;  epi2: none
//
// The two products the scorer used to launch separately (gemm_tf32.cu, persistent kernel) read the hidden layer back
// from HBM right after writing it; here each 64-unit chunk of it stays in shared memory between the products, which
// saves one [rows, d_ff] fp32 read per direction and layer.  H / dH are still written: the weight gradients read them.
//
// Results are bit-identical to the two GEMMs (DESIGN.md 4.13): the same wgmma m64 x k8 tf32 instructions in ascending
// k order into one accumulator per product (the second one across chunks, in chunk order), A operands loaded and
// rounded in registers by the GEMM's own ptx::load_a_tf32, the chunk staged unrounded in the 128-byte-swizzled
// K-major layout the second GEMM read from its ring, and the epilogue operations in epi_chunk_f32's order.
//
// Structure: one CTA per SM walks the 128-row tiles (bounded by the device-side live row count); warp 8 is the TMA
// producer (its warpgroup gives its registers to the others), warps 0-3 and 4-7 are two warpgroups owning rows 0-63
// and 64-127 of the tile and all d output columns.
// A warpgroup's epi1 chunk is then exactly the A operand of its own second product, and each warp re-reads only the 16
// rows it wrote itself.  Shared memory: the X tile, the two warpgroups' chunk staging and a ring of 8 KB weight units
// (64 weight rows x 32 k).  The warpgroups hand nothing to each other except the b1 gradient's column sums.
#include <algorithm>
#include <cstdio>
#include <cuda.h>
#include <cuda_runtime.h>

#include "common.h"
#include "gemm_tf32.h"
#include "sm90_ptx.cuh"

namespace arb {

namespace {

constexpr int CH_ROWS = 128;                  // rows per tile
constexpr int CH_UNITS = 64;                  // hidden units per chunk
constexpr int UNIT_BYTES = 64 * 128;          // ring unit: 64 weight rows x 32 fp32 (one 128-byte swizzle row each)
constexpr int X_SLAB_BYTES = CH_ROWS * 128;   // X tile: one [128 rows][32 k] slab per k-block
constexpr int H_SLAB_BYTES = 64 * 128;        // chunk staging: [64 rows][32 units] per warpgroup and 32-unit half
constexpr int CH_THREADS = 384;               // two consumer warpgroups + the producer warpgroup
constexpr int SMEM_LIMIT = 227 * 1024;        // opt-in shared memory per block on sm_90

// Shared memory, from a 1024-byte aligned base: X tile | chunk staging (2 warpgroups x 2 slabs) | weight ring | tail.
// d = 128: 64 + 32 + 16 x 8 + 1 KB = 225 KB;  d = 256: 128 + 32 + 8 x 8 + 1 KB = 225 KB; + 1 KB alignment slack.
template <int D>
struct ChainLayout {
  static constexpr int KB1 = D / 32;              // k-blocks of the first product (X slabs, W1 units per chunk)
  static constexpr int NBU = (D + 63) / 64;       // ring units per k-block of the second product
  static constexpr int X_BYTES = KB1 * X_SLAB_BYTES;
  static constexpr int H_BYTES = 2 * 2 * H_SLAB_BYTES;
  static constexpr int TAIL_BYTES = 1024;         // barriers (<= 45 x 8 bytes) and the column-sum exchange (512 bytes)
  static constexpr int NU_FIT = (SMEM_LIMIT - 1024 - TAIL_BYTES - X_BYTES - H_BYTES) / UNIT_BYTES;
  static constexpr int NU = NU_FIT < 16 ? NU_FIT : 16;   // ring units
  static constexpr int RING_OFF = X_BYTES + H_BYTES;
  static constexpr int TAIL_OFF = RING_OFF + NU * UNIT_BYTES;
  static constexpr int total() { return TAIL_OFF + TAIL_BYTES + 1024; }
  static_assert(D % 32 == 0 && D >= 32 && D <= 256, "d: a multiple of 32 up to 256");
  static_assert(NU >= 2 * NBU, "the ring holds at least one k-block of the second product");
  static_assert(total() <= SMEM_LIMIT, "shared memory budget");
};

struct ChainParams {
  int M;                 // rows (tensor-map bound)
  int F;                 // hidden units, a multiple of 64
  int rnd;               // round the register A operands to tf32 (nearest); else the tensor core truncates
  int store_h;           // write H / dH
  const float* b1;       // forward: [F]
  const float* b2;       // forward: [D]
  const float* aux;      // forward: residual [M, D] (may alias y)
  float* y;              // [M, D]
  uint32_t* bits;        // [M, F / 32]: written by the forward (nullable), read by the backward
  float* colsum;         // backward: per-tile slots [tiles][F] of the b1 gradient (nullable)
  const int* rows_dev;   // packed rows: device-side live row count (nullable)
};

// acc[:, all D columns] += A (64 x 8, registers) x the k8 step at byte offset 32 ks of the second product's k-block,
// whose weight rows 64 u .. 64 u + 63 are in ring unit desc[u].  d a multiple of 64: m64n64 per unit, as the W2 GEMM's
// 128-column tiles issue it; otherwise m64n32 per 32 rows, as its 64-column tiles do.
template <int D, int U = 0>
__device__ __forceinline__ void second_mma(float (&acc)[D / 8][4], const uint32_t (&a)[4],
                                           const uint64_t (&desc)[(D + 63) / 64], int ks) {
  constexpr int WN = D % 64 == 0 ? 64 : 32;
  if constexpr (U < D / WN) {
    if constexpr (WN == 64) ptx::wgmma_m64n64k8_tf32<8 * U>(acc, a, desc[U] + 2 * ks);
    else ptx::wgmma_m64n32k8_tf32<4 * U>(acc, a, desc[U / 2] + (U & 1) * (32 * 128 / 16) + 2 * ks);
    second_mma<D, U + 1>(acc, a, desc, ks);
  }
}

template <int D, bool BWD>
__global__ void __launch_bounds__(CH_THREADS, 1) ffn_chain_kernel(const __grid_constant__ CUtensorMap tmX,
                                                                 const __grid_constant__ CUtensorMap tmA,
                                                                 const __grid_constant__ CUtensorMap tmB,
                                                                 const __grid_constant__ CUtensorMap tmH,
                                                                 const ChainParams p) {
  using L = ChainLayout<D>;
  constexpr int NU = L::NU, KB1 = L::KB1, NBU = L::NBU, NTY = D / 8;
  extern __shared__ uint8_t smem_dyn[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~uintptr_t(1023));
  uint8_t* xs = smem;
  uint8_t* ring = smem + L::RING_OFF;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::TAIL_OFF);
  uint64_t* empty = full + NU;         // 8 consumer-warp arrivals
  uint64_t* xfull = empty + NU;        // [KB1]: X slab landed
  uint64_t* xfree = xfull + 8;         // every consumer warp has read the X tile for the last time
  uint64_t* csfull = xfree + 1;        // [2]: warpgroup 1's column-sum pairs of a chunk are in csx
  uint64_t* csempty = csfull + 2;      // [2]: warpgroup 0 has read them
  float* csx = reinterpret_cast<float*>(smem + L::TAIL_OFF + 512);   // [2][64]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmX);
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmB);
    if (p.store_h) ptx::prefetch_tmap(&tmH);
    for (int s = 0; s < NU; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
    for (int kb = 0; kb < KB1; ++kb) ptx::mbar_init(&xfull[kb], 1);
    ptx::mbar_init(xfree, 8);
    for (int b = 0; b < 2; ++b) { ptx::mbar_init(&csfull[b], 128); ptx::mbar_init(&csempty[b], 128); }
    ptx::fence_barrier_init();
  }
  arb_pdl_wait();          // everything above overlaps the previous kernel's tail; global memory is touched below
  __syncthreads();
  int n_tiles = (p.M + CH_ROWS - 1) / CH_ROWS;
  if (p.rows_dev) n_tiles = min(n_tiles, (__ldg(p.rows_dev) + CH_ROWS - 1) / CH_ROWS);
  const int n_chunks = p.F / CH_UNITS;

  if (warp >= 8) {
    // ===================== TMA producer (one thread) =====================
    // The register file is split evenly over the SM's four schedulers, each holding three of the twelve warps: the
    // producer warpgroup hands its registers to the consumers, whose accumulators take up to d / 2 + 32 of them.
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    // per tile: the X slabs (once the previous tile's last first product is done with them), then per chunk the KB1
    // units of A (rows 64 j.., k-block kb) and the 2 x NBU units of B (rows 64 u.., hidden units 64 j + 32 kb2 ..)
    if (warp == 8 && lane == 0) {
      uint32_t it = 0;
      auto unit = [&](const CUtensorMap* tm, int c0, int c1) {
        const int s = it % NU;
        const uint32_t round = it / NU;
        if (round > 0) ptx::mbar_wait(&empty[s], (round - 1) & 1);
        ptx::mbar_expect_tx(&full[s], UNIT_BYTES);
        ptx::tma_load_4d(ring + s * UNIT_BYTES, tm, &full[s], c0, c1, 0, 0);
        ++it;
      };
      int local = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++local) {
        const int m0 = t * CH_ROWS;
        if (local > 0) ptx::mbar_wait(xfree, (local - 1) & 1);
        for (int kb = 0; kb < KB1; ++kb) {
          ptx::mbar_expect_tx(&xfull[kb], X_SLAB_BYTES);
          ptx::tma_load_4d(xs + kb * X_SLAB_BYTES, &tmX, &xfull[kb], 32 * kb, m0, 0, 0);
        }
        if (!BWD) {          // the residual tile is read at the end of the tile: have it in L2 by then
          const long long bytes = (long long)(min(p.M, m0 + CH_ROWS) - m0) * D * 4;
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;"
                       ::"l"(p.aux + (long long)m0 * D), "r"(uint32_t(bytes)) : "memory");
        }
        for (int j = 0; j < n_chunks; ++j) {
          for (int kb = 0; kb < KB1; ++kb) unit(&tmA, 32 * kb, CH_UNITS * j);
          for (int kb2 = 0; kb2 < 2; ++kb2)
            for (int u = 0; u < NBU; ++u) unit(&tmB, CH_UNITS * j + 32 * kb2, 64 * u);
        }
      }
    }
  } else {
    // ===================== two consumer warpgroups =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int g = warp >> 2, w = warp & 3, gq = lane >> 2, t4 = lane & 3, gt = threadIdx.x & 127;
    uint8_t* hs = smem + L::X_BYTES + g * 2 * H_SLAB_BYTES;
    const int fw = p.F >> 5;                          // bit words per row
    uint32_t it = 0, cj = 0;
    int local = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++local) {
      const int m0 = t * CH_ROWS;
      const int row0 = m0 + 64 * g + 16 * w + gq;    // accumulator elements [0], [1]: row0; [2], [3]: row0 + 8
      float accY[NTY][4];
#pragma unroll
      for (int n = 0; n < NTY; ++n) accY[n][0] = accY[n][1] = accY[n][2] = accY[n][3] = 0.f;
#pragma unroll 1
      for (int j = 0; j < n_chunks; ++j, ++cj) {
        uint32_t mw[2][2] = {{0u, 0u}, {0u, 0u}};    // backward: mask words [row row0 / row0 + 8][32-unit half]
        if constexpr (BWD) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (row0 + 8 * h < p.M) {
              mw[h][0] = __ldg(p.bits + (long long)(row0 + 8 * h) * fw + 2 * j);
              mw[h][1] = __ldg(p.bits + (long long)(row0 + 8 * h) * fw + 2 * j + 1);
            }
        }
        // ---- first product: accH = X (this warpgroup's 64 rows) x A_j^T, k-blocks ascending
        float accH[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n) accH[n][0] = accH[n][1] = accH[n][2] = accH[n][3] = 0.f;
#pragma unroll 1
        for (int kb = 0; kb < KB1; ++kb, ++it) {
          const int s = it % NU;
          ptx::mbar_wait(&full[s], (it / NU) & 1);
          if (j == 0) ptx::mbar_wait(&xfull[kb], local & 1);
          uint32_t a[4][4];
          ptx::load_a_tf32(a, xs + kb * X_SLAB_BYTES, 64 * g + 16 * w, p.rnd);
          const uint64_t desc = ptx::wgmma_desc_sw128(ring + s * UNIT_BYTES);
          ptx::wgmma_fence_acc(accH);
          ptx::wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) ptx::wgmma_m64n64k8_tf32<0>(accH, a[ks], desc + 2 * ks);
          ptx::wgmma_commit();
          ptx::wgmma_wait0();
          ptx::wgmma_fence_acc(accH);
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(&empty[s]);
        }
        if (j == n_chunks - 1) {
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(xfree);
        }
        // ---- epi1 into the staging slabs: this warp's rows 16 w .. 16 w + 15, unrounded, 128-byte swizzled
        if (p.store_h && lane == 0) ptx::tma_store_wait_read<0>();   // the previous chunk's H store has read them
        if (BWD && p.colsum) ptx::named_bar_sync(1 + g, 128);         // ... and the previous column sums
        __syncwarp();
        uint32_t wb[2][2] = {{0u, 0u}, {0u, 0u}};   // forward: ReLU bit words, as mw
#pragma unroll
        for (int n = 0; n < 8; ++n) {
          const int c = 8 * n + 2 * t4, bp = 8 * (n & 3) + 2 * t4;   // column in the chunk; bit in its word
          float2 bb = make_float2(0.f, 0.f);
          if constexpr (!BWD) bb = __ldg(reinterpret_cast<const float2*>(p.b1 + CH_UNITS * j + c));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float o0 = accH[n][2 * h], o1 = accH[n][2 * h + 1];
            if constexpr (BWD) {
              o0 = (mw[h][n >> 2] >> bp) & 1u ? o0 : 0.f;
              o1 = (mw[h][n >> 2] >> (bp + 1)) & 1u ? o1 : 0.f;
            } else {
              o0 += bb.x; o1 += bb.y;
              o0 = fmaxf(o0, 0.0f); o1 = fmaxf(o1, 0.0f);
              wb[h][n >> 2] |= (o0 > 0.f ? 1u : 0u) << bp | (o1 > 0.f ? 1u : 0u) << (bp + 1);
            }
            *reinterpret_cast<float2*>(hs + (n >> 2) * H_SLAB_BYTES + ptx::sw128(16 * w + gq + 8 * h, 4 * (c & 31))) =
                make_float2(o0, o1);
          }
        }
        if (!BWD && p.bits) {       // the quad's four lanes hold the bits of the same two rows: OR them
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int s = 0; s < 2; ++s) {
              wb[h][s] |= __shfl_xor_sync(0xffffffffu, wb[h][s], 1);
              wb[h][s] |= __shfl_xor_sync(0xffffffffu, wb[h][s], 2);
            }
          const int h = t4 >> 1, s = t4 & 1;
          const uint32_t word = t4 == 0 ? wb[0][0] : t4 == 1 ? wb[0][1] : t4 == 2 ? wb[1][0] : wb[1][1];
          if (row0 + 8 * h < p.M) p.bits[(long long)(row0 + 8 * h) * fw + 2 * j + s] = word;
        }
        if (p.store_h) ptx::fence_proxy_async_smem();    // generic-proxy writes -> the TMA store's reads
        __syncwarp();
        if (p.store_h && lane == 0) {
#pragma unroll
          for (int s = 0; s < 2; ++s)
            ptx::tma_store_4d(&tmH, hs + s * H_SLAB_BYTES + 16 * w * 128, CH_UNITS * j + 32 * s, m0 + 64 * g + 16 * w, 0, 0);
          ptx::tma_store_commit();
        }
        if constexpr (BWD) {
          if (p.colsum) {
            // b1 gradient of this tile, as the EPI_COLSUM epilogue: per column, four 32-row segments summed in row
            // order from 0.f, then (s0 + s1) + (s2 + s3).  This warpgroup forms its pair over its 64 rows; warpgroup 1
            // hands its pair to warpgroup 0, which adds the two and writes the tile's slot.
            ptx::named_bar_sync(1 + g, 128);
            const int cc = gt >> 1, seg = gt & 1, c5 = cc & 31;
            const uint8_t* slab = hs + (cc >> 5) * H_SLAB_BYTES;
            float ts = 0.f;
#pragma unroll 8
            for (int r = 32 * seg; r < 32 * seg + 32; ++r)
              ts += *reinterpret_cast<const float*>(slab + r * 128 + ((((c5 >> 2) ^ (r & 7)) << 4) | ((c5 & 3) << 2)));
            ts += __shfl_xor_sync(0xffffffffu, ts, 1);
            const int b = cj & 1;
            const uint32_t use = cj >> 1;
            if (g == 1) {
              if (use > 0) ptx::mbar_wait(&csempty[b], (use - 1) & 1);
              if (seg == 0) csx[b * 64 + cc] = ts;
              ptx::mbar_arrive(&csfull[b]);
            } else {
              ptx::mbar_wait(&csfull[b], use & 1);
              const float other = csx[b * 64 + cc];
              ptx::mbar_arrive(&csempty[b]);
              if (seg == 0) p.colsum[(long long)t * p.F + CH_UNITS * j + cc] = ts + other;
            }
          }
        }
        // ---- second product: accY += chunk x B_j^T, k-blocks (32 units) ascending
#pragma unroll 1
        for (int kb2 = 0; kb2 < 2; ++kb2, it += NBU) {
          uint32_t a[4][4];
          ptx::load_a_tf32(a, hs + kb2 * H_SLAB_BYTES, 16 * w, p.rnd);
          uint64_t desc[NBU];
#pragma unroll
          for (int u = 0; u < NBU; ++u) {
            const uint32_t iu = it + u;
            ptx::mbar_wait(&full[iu % NU], (iu / NU) & 1);
            desc[u] = ptx::wgmma_desc_sw128(ring + (iu % NU) * UNIT_BYTES);
          }
          ptx::wgmma_fence_acc(accY);
          ptx::wgmma_fence();
#pragma unroll
          for (int ks = 0; ks < 4; ++ks) second_mma<D>(accY, a[ks], desc, ks);
          ptx::wgmma_commit();
          ptx::wgmma_wait0();
          ptx::wgmma_fence_acc(accY);
          __syncwarp();
          if (lane == 0) {
#pragma unroll
            for (int u = 0; u < NBU; ++u) ptx::mbar_arrive(&empty[(it + u) % NU]);
          }
        }
      }
      // ---- epi2: forward + b2 + residual (epi_chunk_f32's order); backward as is.  Straight from the accumulator:
      // a quad's float2 stores cover 32 contiguous bytes of a row.  The residual may alias the output, so its loads
      // are issued a 64-column group at a time ahead of the group's stores (else each would wait for the last store).
#pragma unroll
      for (int n0 = 0; n0 < NTY; n0 += 8) {
        constexpr int G = NTY < 8 ? NTY : 8;
        float2 r[G][2];
        if constexpr (!BWD) {
#pragma unroll
          for (int n = 0; n < G && n0 + n < NTY; ++n)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              r[n][h] = row0 + 8 * h < p.M
                            ? *reinterpret_cast<const float2*>(p.aux + (long long)(row0 + 8 * h) * D + 8 * (n0 + n) + 2 * t4)
                            : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int n = 0; n < G && n0 + n < NTY; ++n) {      // (d = 96, 160, 224: a last group of 32 columns)
          const int c = 8 * (n0 + n) + 2 * t4;
          float2 bb = make_float2(0.f, 0.f);
          if constexpr (!BWD) bb = __ldg(reinterpret_cast<const float2*>(p.b2 + c));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = row0 + 8 * h;
            if (row >= p.M) continue;
            float2 o = make_float2(accY[n0 + n][2 * h], accY[n0 + n][2 * h + 1]);
            if constexpr (!BWD) {
              o.x += bb.x; o.y += bb.y;
              o.x += r[n][h].x; o.y += r[n][h].y;
            }
            *reinterpret_cast<float2*>(p.y + (long long)row * D + c) = o;
          }
        }
      }
    }
    if (p.store_h && lane == 0) ptx::tma_store_wait_all();
  }
  __syncthreads();
}

template <int D, bool BWD>
int launch_chain_t(const CUtensorMap& tX, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tH,
                   const ChainParams& p, int grid, cudaStream_t st) {
  return launch(ffn_chain_kernel<D, BWD>, dim3(grid), dim3(CH_THREADS), ChainLayout<D>::total(), st, /*pdl=*/true, tX,
                tA, tB, tH, p);
}

template <bool BWD>
int launch_chain(int d, const CUtensorMap& tX, const CUtensorMap& tA, const CUtensorMap& tB, const CUtensorMap& tH,
                 const ChainParams& p, int grid, cudaStream_t st) {
  switch (d) {
    case 32: return launch_chain_t<32, BWD>(tX, tA, tB, tH, p, grid, st);
    case 64: return launch_chain_t<64, BWD>(tX, tA, tB, tH, p, grid, st);
    case 96: return launch_chain_t<96, BWD>(tX, tA, tB, tH, p, grid, st);
    case 128: return launch_chain_t<128, BWD>(tX, tA, tB, tH, p, grid, st);
    case 160: return launch_chain_t<160, BWD>(tX, tA, tB, tH, p, grid, st);
    case 192: return launch_chain_t<192, BWD>(tX, tA, tB, tH, p, grid, st);
    case 224: return launch_chain_t<224, BWD>(tX, tA, tB, tH, p, grid, st);
    case 256: return launch_chain_t<256, BWD>(tX, tA, tB, tH, p, grid, st);
    default: arb_set_error("ffn_chain: d must be a multiple of 32 up to 256"); return ARB_E_UNSUPPORTED;
  }
}

TRef matrix(const float* p, int64_t cols, int64_t rows) {
  TRef t; t.ptr = p; t.dim[0] = cols; t.dim[1] = rows; t.stride[0] = 1; t.stride[1] = cols; return t;
}

}  // namespace

bool ffn_chain_supported(int d, int f) { return d % 32 == 0 && d >= 32 && d <= 256 && f > 0 && f % CH_UNITS == 0; }

int launch_ffn_chain(const FfnChain& c, cudaStream_t st) {
  if (!ffn_chain_supported(c.d, c.f)) {
    arb_set_error("ffn_chain: needs d a multiple of 32 up to 256 and d_ff a multiple of 64");
    return ARB_E_UNSUPPORTED;
  }
  if (c.rows < 0 || !c.x || !c.a || !c.b || !c.y || (c.bwd ? !c.bits : (!c.b1 || !c.b2 || !c.aux))) {
    arb_set_error("ffn_chain: bad arguments");
    return ARB_E_INVALID_ARG;
  }
  if (c.rows == 0) return ARB_OK;
  alignas(64) CUtensorMap tX, tA, tB, tH;
  int rc;
  if ((rc = make_tmap_4d(&tX, matrix(c.x, c.d, c.rows), TmapBox{{32, CH_ROWS, 1, 1}}, 0))) return rc;
  if ((rc = make_tmap_4d(&tA, matrix(c.a, c.d, c.f), TmapBox{{32, 64, 1, 1}}, 0))) return rc;
  if ((rc = make_tmap_4d(&tB, matrix(c.b, c.f, c.d), TmapBox{{32, 64, 1, 1}}, 0))) return rc;
  if (c.h) {
    if ((rc = make_tmap_4d(&tH, matrix(c.h, c.f, c.rows), TmapBox{{32, 16, 1, 1}}, 0))) return rc;
  } else {
    tH = tX;
  }
  ChainParams p;
  p.M = c.rows; p.F = c.f; p.rnd = tf32_round_on_load(); p.store_h = c.h != nullptr;
  p.b1 = c.b1; p.b2 = c.b2; p.aux = c.aux; p.y = c.y; p.bits = c.bits; p.colsum = c.bwd ? c.colsum : nullptr;
  p.rows_dev = c.rows_dev;
  const int tiles = (c.rows + CH_ROWS - 1) / CH_ROWS;
  const int grid = std::min(tiles, sm_count());
  DetParts dp;     // the b1 gradient: one slot per tile, summed in order afterwards (as the EPI_COLSUM epilogue's)
  dp.add(p.colsum, tiles, 1, c.f, c.f);
  if ((rc = dp.begin(st))) return rc;
  {
    // accounting: both products' flops; the HBM operands moved: X, the output (and the residual), H / dH, the bits
    const double R = double(c.rows) * (c.rows_dev ? arb_row_frac() : 1.0), d = c.d, f = c.f;
    const double bytes = 4.0 * R * d * (c.bwd ? 2.0 : 3.0) + (c.h ? 4.0 * R * f : 0.0) + (c.bits ? R * f / 8.0 : 0.0);
    char name[56];
    std::snprintf(name, sizeof name, "ffn_chain[%s M%d d%d f%d]", c.bwd ? "bwd" : "fwd", c.rows, c.d, c.f);
    ProfScope ps(ARB_PROF_GEMM, 4.0 * R * d * f, st, bytes, name);
    rc = c.bwd ? launch_chain<true>(c.d, tX, tA, tB, tH, p, grid, st) : launch_chain<false>(c.d, tX, tA, tB, tH, p, grid, st);
  }
  if (rc) return rc;
  return dp.finish(st);
}

}  // namespace arb

// ------------------------------------------------------------------------------------------------ test entry points
// The chained FFN kernels on their own (include/allrank_b200.h), through the scorer's launcher.
extern "C" int32_t arb_ffn_forward(const float* x, const float* w1, const float* b1, const float* w2, const float* b2,
                                   const float* res, int32_t rows, int32_t d, int32_t d_ff, float* y, float* h,
                                   uint32_t* bits, const int32_t* rows_dev, void* stream) {
  arb::FfnChain c;
  c.rows = rows; c.d = d; c.f = d_ff; c.x = x; c.a = w1; c.b = w2; c.b1 = b1; c.b2 = b2; c.aux = res;
  c.y = y; c.h = h; c.bits = bits; c.rows_dev = rows_dev; c.bwd = 0;
  return arb::launch_ffn_chain(c, static_cast<cudaStream_t>(stream));
}

extern "C" int32_t arb_ffn_backward_input(const float* dy, const float* w2t, const float* w1t, const uint32_t* bits,
                                          int32_t rows, int32_t d, int32_t d_ff, float* dx, float* dh,
                                          float* grad_b1, const int32_t* rows_dev, void* stream) {
  arb::FfnChain c;
  c.rows = rows; c.d = d; c.f = d_ff; c.x = dy; c.a = w2t; c.b = w1t; c.bits = const_cast<uint32_t*>(bits);
  c.y = dx; c.h = dh; c.colsum = grad_b1; c.rows_dev = rows_dev; c.bwd = 1;
  return arb::launch_ffn_chain(c, static_cast<cudaStream_t>(stream));
}
