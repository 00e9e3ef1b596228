// Host-side description of one (batched) TF32 tensor-core GEMM launch.  See gemm_tf32.cu.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "dropout.cuh"

namespace arb {

// A strided view of up to 4 dimensions, dim[0] contiguous (stride[0] == 1), strides in elements.
// bf16 = 1: the elements are bfloat16 (2 bytes) -- the bf16 mode of the scorer (BASELINE config 3); else fp32.
struct TRef {
  const void* ptr = nullptr;
  int64_t dim[4] = {1, 1, 1, 1};
  int64_t stride[4] = {1, 0, 0, 0};
  int bf16 = 0;
};

enum : int {
  EPI_BIAS = 1,       // + bias[n]
  EPI_RELU = 2,       // max(., 0)
  EPI_ADD_AUX = 4,    // + Aux[m,n]          (residual; Aux may alias C)
  EPI_MASK_AUX = 8,   // . * (Aux[m,n] > 0)  (ReLU backward)
  EPI_ATOMIC = 16,    // atomic_out += C instead of storing C (split-K weight gradients; splits summed in order)
  EPI_DROPOUT = 32,   // inverted dropout on (alpha*acc + bias [relu]) before the aux tile is added
  EPI_COLSUM = 64,    // colsum_out[n] += sum_m C[m,n]  (bias gradient of the layer that produced C's input)
  EPI_RELU_BITS = 128,  // with EPI_RELU (fp32 output): also write bits[m, n/32] -- bit j = (C[m, 32*(n/32) + j] > 0)
  EPI_MASK_BITS = 256,  // . * bit of `bits` (ReLU backward from the forward's bit mask: 1 bit per element read instead
                        // of the 4-byte activation an EPI_MASK_AUX tile costs); fp32 output, N % 32 == 0
};

struct GemmDesc {
  int M = 0, N = 0, K = 0;      // C[M,N] = alpha * sum_k A[m,k] B[n,k]
  int a_mn = 0, b_mn = 0;       // 0: operand stored K-contiguous ("K-major"); 1: stored M/N-contiguous ("MN-major")
  int b_tf32 = 0;               // fp32 B already holds tf32-rounded values (the scorer's weight copy): not rounded again
  int dgrad = 0;                // an input-gradient product (label of the per-kernel profile only)
  TRef A, B, C, Aux;            // K-major operand: dim = (K, rows, b2, b3); MN-major: dim = (rows, K, b2, b3);
                                // C/Aux: dim = (N, M, b2, b3)
  int nb2 = 1, nb3 = 1;         // batch grid: blockIdx.z = b3 * nb2 + b2
  int a_b2 = 0, a_b3 = 0, b_b2 = 0, b_b3 = 0, c_b2 = 0, c_b3 = 0;   // does the operand move with b2 / b3 ?
  int block_n = 64;             // 32, 64 or 128 output columns per CTA
  int split_k = 1;              // >1 only with EPI_ATOMIC and nb2 == nb3 == 1
  int flags = 0;
  float alpha = 1.0f;
  const float* bias = nullptr;  // [N]
  float* atomic_out = nullptr;  // row-major [M, atomic_ld]
  int64_t atomic_ld = 0;
  DropSite drop{0u, 0u, 1.0f};  // EPI_DROPOUT: element index = m * drop_n + n (unbatched problems only)
  int drop_n = 0;               // EPI_DROPOUT: row width of the counter layout (0: N); a layer of n real columns stored
                                // at N = round_up(n, 4) counts over its real columns (DESIGN.md 4.16)
  float* colsum_out = nullptr;  // EPI_COLSUM: [N], += column sums (per-tile slots summed in order)
  uint32_t* bits = nullptr;     // EPI_RELU_BITS (written) / EPI_MASK_BITS (read): [M, N / 32] words, row-major
  const int* rows_dev = nullptr;   // packed rows (unbatched launches): device pointer to the live row count, a
                                   // multiple of 128.  It bounds M (tiles beyond it are not computed) or, with
                                   // EPI_ATOMIC, K (the weight gradients reduce over the live rows only); the host-side
                                   // M / K stay the upper bound the tensor maps and the grid are built from.
  // Element types come from the views: A and B must agree (both fp32 -> tf32 MMA, both bf16 -> bf16 MMA, fp32
  // accumulation either way); C may be fp32 or bf16; an Aux tile has C's type (fp32 residual into an fp32 stream,
  // bf16 ReLU-mask tile into a bf16 gradient).  bf16 outputs need block_n >= 64.
};

int launch_gemm_tf32(const GemmDesc& d, cudaStream_t stream);   // 0 or ARB_E_*

// The FFN sublayer's two linears chained in one kernel (ffn_chain.cu), fp32 operands on the tf32 tensor cores, all
// matrices row-major and dense:  Y[rows, d] = epi2( sum_j epi1( X[rows, d] A_j^T ) B_j^T ),  A [f, d], B [d, f].
//   forward (bwd = 0): A = W1, B = W2;  epi1 = + b1, ReLU (H -> h, bit words -> bits, either nullable);
//                      epi2 = + b2 + aux (the residual; may alias y)
//   backward (bwd = 1): X = dY, A = W2^T, B = W1^T;  epi1 = mask by bits (dH -> h, nullable);  colsum (nullable) +=
//                      the column sums of dH (the b1 gradient)
// The weights are read as given (the scorer's tf32-rounded copy); X and the chunk of the hidden layer are rounded as
// the GEMMs round their register operands.  Bit-identical to the two launch_gemm_tf32 products it replaces.
struct FfnChain {
  int rows = 0, d = 0, f = 0;
  const float* x = nullptr;
  const float* a = nullptr;
  const float* b = nullptr;
  const float* b1 = nullptr;
  const float* b2 = nullptr;
  const float* aux = nullptr;
  float* y = nullptr;
  float* h = nullptr;
  uint32_t* bits = nullptr;
  float* colsum = nullptr;
  const int* rows_dev = nullptr;   // packed rows: device-side live row count; tiles beyond it are not touched
  int bwd = 0;
};
bool ffn_chain_supported(int d, int f);   // d a multiple of 32 up to 256, f a multiple of 64
int launch_ffn_chain(const FfnChain& c, cudaStream_t stream);   // 0 or ARB_E_*

// 4-D tiled tensor map with 128-byte swizzle; box[0] must span 128 bytes (32 fp32 / 64 bf16 elements).
struct TmapBox { uint32_t b[4]; };
// unswizzled = 0: SWIZZLE_128B (16-byte chunks); 1: no swizzle (dense rows narrower than 128 bytes: the bf16 outputs
// of the attention kernels)
int make_tmap_4d(void* out_CUtensorMap, const TRef& t, TmapBox box, int unswizzled);

void set_tf32_round_on_load(int enable);
int tf32_round_on_load();   // 1: MMA kernels round fp32 operands to tf32 (nearest even) after loading them
void set_gemm_persistent(int on);

}  // namespace arb
