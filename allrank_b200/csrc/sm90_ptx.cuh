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
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

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
