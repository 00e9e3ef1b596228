// Thin inline-PTX wrappers for the sm_90a features the scorer kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), warp-level tensor-core MMA (mma.sync) and the addressing of the 128-byte
// swizzled tiles TMA writes into shared memory.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace arb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must fault (trap), never hang the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();   // ~2 s at 2 GHz
  }
}

// ------------------------------------------------------------------ fences / barriers
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// until at most N of this thread's most recent store groups still read their shared-memory source
template <int N = 0>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }

// two fp32 -> packed bf16x2 (round to nearest even); `lo` lands in the low half
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// ------------------------------------------------------------------ 128-byte swizzled tiles
// TMA with CU_TENSOR_MAP_SWIZZLE_128B writes a box whose inner extent is 128 bytes as rows of 128 bytes; the 16-byte
// chunk j of row r lands at chunk j ^ (r % 8).  Byte offset of byte `b` of row `r`:
__device__ __forceinline__ uint32_t sw128(int r, int b) {
  return uint32_t(r) * 128u + ((uint32_t((b >> 4) ^ (r & 7))) << 4) + uint32_t(b & 15);
}
// 16-byte shared-memory load / store at a shared-window address (smem_u32)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// fp32 element (r, c) of a [rows][32] tile (c < 32: the contiguous dimension)
__device__ __forceinline__ float ld_f32(const uint8_t* tile, int r, int c) {
  return *reinterpret_cast<const float*>(tile + sw128(r, 4 * c));
}

// ------------------------------------------------------------------ warp-level tensor-core MMA
// fp32 -> tf32, round to nearest even; the tensor core itself ignores the low 13 mantissa bits.  (Ties away from zero
// -- cvt.rna -- measurably worsens the gradients of the deeper shipped configurations against the fp32 reference.)
__device__ __forceinline__ uint32_t cvt_tf32(float x) {
  uint32_t r;
  asm("cvt.rn.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
// D[16x8] += A[16x8] B[8x8], tf32 operands, fp32 accumulation.  Fragments (g = lane / 4, t = lane % 4):
//   a = {A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4]},  b = {B[t][g], B[t+4][g]},
//   d = {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// D[16x8] += A[16x16] B[16x8], bf16 operands (pairs along k, lower k in the low half), fp32 accumulation:
//   a = {A[g][2t..], A[g+8][2t..], A[g][2t+8..], A[g+8][2t+8..]},  b = {B[2t..][g], B[2t+8..][g]}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// Four 8x4 fp32 blocks from shared memory (ldmatrix of 8x8 b16 matrices): lanes 8j..8j+7 give the 16-byte row
// addresses of block j; lane (g = lane / 4, t = lane % 4) receives element (g, t) of every block.
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* row_addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(row_addr)));
}
// The tf32 A fragments (m16n8k8 layout above) of rows r0 .. r0+15 of a [rows][32 fp32] 128-byte-swizzled tile, one per
// k8 step of its 32-wide k-block: ldmatrix, then round to nearest tf32 unless `rnd` is 0 (the tensor core then
// truncates).  Every register-A tf32 wgmma loads its operand here, so the kernels that must agree bit for bit agree.
__device__ __forceinline__ void load_a_tf32(uint32_t (&a)[4][4], const uint8_t* tile, int r0, int rnd) {
  const int lane = threadIdx.x & 31, j = lane >> 3;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    // lanes 8j .. 8j+7 address block j: rows +8 (j & 1), k +4 (j >> 1) of the 16 x 8 fragment
    ldmatrix_x4(a[ks], tile + sw128(r0 + 8 * (j & 1) + (lane & 7), 32 * ks + 16 * (j >> 1)));
    if (rnd) {
#pragma unroll
      for (int e = 0; e < 4; ++e) a[ks][e] = cvt_tf32(__uint_as_float(a[ks][e]));
    }
  }
}

// ------------------------------------------------------------------ warpgroup MMA (wgmma)
// Shared-memory matrix descriptor of a K-major operand tile written by TMA with SWIZZLE_128B: rows of 128 bytes, 8-row
// swizzle atoms 1024 bytes apart (stride byte offset), the tile 1024-byte aligned.  A k-step inside the 128-byte row
// advances the start address by its byte offset (the hardware applies the swizzle to the final address).
__device__ __forceinline__ uint64_t wgmma_desc_sw128(const void* tile) {
  const uint64_t addr = smem_u32(tile);
  return ((addr & 0x3FFFFull) >> 4) | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Keeps the compiler from moving accumulator accesses across the asynchronous MMA (no code emitted).
template <int NT>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[NT][4]) {
#pragma unroll
  for (int j = 0; j < NT; ++j) asm volatile("" : "+f"(d[j][0]), "+f"(d[j][1]), "+f"(d[j][2]), "+f"(d[j][3])::"memory");
}

// D[64 x WN] += A[64 x 8] B[WN x 8]^T, tf32 operands, fp32 accumulation, issued by a whole warpgroup.  A comes from
// registers: warp w of the warpgroup holds rows 16w .. 16w+15 in the m16n8k8 A fragment layout above.  B is a K-major
// tile in shared memory (descriptor).  The accumulator of 8-column block j lives in d[J0 + j] in the m16n8k8 D layout.
#define ARB_D4(j) "+f"(d[J0 + j][0]), "+f"(d[J0 + j][1]), "+f"(d[J0 + j][2]), "+f"(d[J0 + j][3])
template <int J0, int NT>
__device__ __forceinline__ void wgmma_m64n32k8_tf32(float (&d)[NT][4], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : ARB_D4(0), ARB_D4(1), ARB_D4(2), ARB_D4(3)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}
template <int J0, int NT>
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[NT][4], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : ARB_D4(0), ARB_D4(1), ARB_D4(2), ARB_D4(3), ARB_D4(4), ARB_D4(5), ARB_D4(6), ARB_D4(7)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}
// The same with A also read from shared memory (a K-major tile, descriptor as for B); every warp's 16 rows of D are as
// above.
template <int J0, int NT>
__device__ __forceinline__ void wgmma_m64n32k8_tf32_ss(float (&d)[NT][4], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1;\n\t}"
      : ARB_D4(0), ARB_D4(1), ARB_D4(2), ARB_D4(3)
      : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <int J0, int NT>
__device__ __forceinline__ void wgmma_m64n64k8_tf32_ss(float (&d)[NT][4], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n\t}"
      : ARB_D4(0), ARB_D4(1), ARB_D4(2), ARB_D4(3), ARB_D4(4), ARB_D4(5), ARB_D4(6), ARB_D4(7)
      : "l"(desc_a), "l"(desc_b), "r"(1));
}
#undef ARB_D4

// An accumulator fragment {D[g][2t], D[g][2t+1], D[g+8][2t], D[g+8][2t+1]} of an 8-column block, reused as the tf32
// A fragment of the next product (contraction over those 8 columns): lane t needs columns t and t + 4 of its rows.
__device__ __forceinline__ void acc_to_a_tf32(const float (&c)[4], uint32_t (&a)[4], int lane) {
  const int t = lane & 3, base = lane & ~3;
  const int s1 = base + (t >> 1), s2 = base + 2 + (t >> 1);
  const float x0 = __shfl_sync(0xffffffffu, c[0], s1), x1 = __shfl_sync(0xffffffffu, c[1], s1);
  const float y0 = __shfl_sync(0xffffffffu, c[2], s1), y1 = __shfl_sync(0xffffffffu, c[3], s1);
  const float u0 = __shfl_sync(0xffffffffu, c[0], s2), u1 = __shfl_sync(0xffffffffu, c[1], s2);
  const float w0 = __shfl_sync(0xffffffffu, c[2], s2), w1 = __shfl_sync(0xffffffffu, c[3], s2);
  const bool odd = (t & 1) != 0;
  a[0] = __float_as_uint(odd ? x1 : x0);
  a[1] = __float_as_uint(odd ? y1 : y0);
  a[2] = __float_as_uint(odd ? u1 : u0);
  a[3] = __float_as_uint(odd ? w1 : w0);
}

}  // namespace ptx
}  // namespace arb
