// Shared-memory accesses and mma.sync m16n8k8 tf32 fragment loads of the fused attention kernels
// (attention_fused.cu, attention_fused_bwd.cu).
#pragma once
#include <cstdint>

#include "sm90_ptx.cuh"

namespace arb {

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float round_tf32(float x) {
  // round-to-nearest (ties away) to tf32 as "+ half an ulp of the 10-bit mantissa, then let the tensor core ignore the
  // low 13 bits" -- one integer add instead of cvt.rna.tf32.f32.
  // Same result as cvt.rna for every finite value (probabilities and their gradients are finite).
  return __uint_as_float(__float_as_uint(x) + 0x1000u);
}

// Shared-memory accesses of the inner loops, by 32-bit shared-window address (ld.shared / ldmatrix / st.shared).
__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t a) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
// four 8 x 4 fp32 matrices (8 x 8 b16): lane l gives the address of row l % 8 of matrix l / 8, and receives word
// lane % 4 of row lane / 4 of each matrix
__device__ __forceinline__ void ldsm_x4(uint32_t a, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void sts128(uint32_t a, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts64(uint32_t a, uint2 v) {
  asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(v.x), "r"(v.y) : "memory");
}

// Operand rows in shared memory are 128 bytes (32 fp32; for dk = 16 TMA zero-fills columns 16..31), 128B-swizzled.
// Every product keeps the standard assignment of its contraction index to the MMA k-slots (head dimension: slot t of
// k-step ks is column 8 ks + t; queries / keys of an 8-row block: slot t is row t), so each output element is computed
// by the same sequence of tensor-core operations as a straightforward fragment layout would use.  Only the positions
// of output rows / columns inside an MMA are permuted, which changes where an element lands, not its value:
//  * the second operand of S^T = K Q^T (S = Q K^T) takes row sigma(n) of its 8-row block as column n,
//    sigma = {0, 4, 1, 5, 2, 6, 3, 7}: accumulator columns 2t, 2t + 1 are rows t, t + 4, which are exactly the k-slots
//    of the lane's A fragment for the next product -- P / dS feed it without shuffles;
//  * output column g of n-tile nt is head column 4 sigma(g) + nt (dk 32) or 2g + nt (dk 16): the B operand is one
//    conflict-free 128-bit (64-bit) load per row, and a lane's accumulator holds 16-byte runs of its two rows.
__device__ __forceinline__ int sigma8(int n) { return (n >> 1) + 4 * (n & 1); }
// A fragments over the head dimension of the 16 rows r0 ... r0 + 15:
// a[ks] = {X[r0 + g][8ks + t], X[r0 + g + 8][8ks + t], X[r0 + g][8ks + t + 4], X[r0 + g + 8][8ks + t + 4]}
template <int KS>
__device__ __forceinline__ void ld_a_head(uint32_t op, int r0, int lane, uint32_t (&a)[KS][4]) {
  const int m = lane >> 3, r = r0 + (lane & 7) + 8 * (m & 1);
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) ldsm_x4(op + uint32_t(r) * 128u + (uint32_t((2 * ks + (m >> 1)) ^ (r & 7)) << 4), a[ks]);
}
// a[ks] of ld_a_head alone (the wide streaming kernels re-read the tile's fragments one k-step at a time)
__device__ __forceinline__ void ld_a_step(uint32_t op, int r0, int lane, int ks, uint32_t (&a)[4]) {
  const int m = lane >> 3, r = r0 + (lane & 7) + 8 * (m & 1);
  ldsm_x4(op + uint32_t(r) * 128u + (uint32_t((2 * ks + (m >> 1)) ^ (r & 7)) << 4), a);
}
// B fragments over the head dimension of the 8 rows r0 + sigma(n): b[ks] = {X[r0 + sigma(g)][8ks + t], ...[8ks + t + 4]}
template <int KS>
__device__ __forceinline__ void ld_b_head(uint32_t op, int r0, int lane, uint32_t (&b)[KS][2]) {
  const int r = r0 + sigma8(lane & 7);
#pragma unroll
  for (int p = 0; p < KS / 2; ++p) {
    uint32_t x[4];
    ldsm_x4(op + uint32_t(r) * 128u + (uint32_t((4 * p + (lane >> 3)) ^ (r & 7)) << 4), x);
    b[2 * p][0] = x[0]; b[2 * p][1] = x[1]; b[2 * p + 1][0] = x[2]; b[2 * p + 1][1] = x[3];
  }
}
// the B operand of an output product from row r: v[nt] = X[r][column of output column g in n-tile nt]
template <int KS>
__device__ __forceinline__ void ld_b_out(uint32_t op, int r, int g, uint32_t (&v)[KS]) {
  if constexpr (KS == 4) {
    const uint4 x = lds128(op + uint32_t(r) * 128u + (uint32_t(sigma8(g) ^ (r & 7)) << 4));
    v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
  } else {
    const uint2 x = lds64(op + ptx::sw128(r, 8 * g));
    v[0] = x.x; v[1] = x.y;
  }
}

}  // namespace arb
