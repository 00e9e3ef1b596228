// Host launchers of the SIMT scorer kernels (scorer_kernels.cu).  All return 0 or ARB_E_*.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "dropout.cuh"

namespace arb {

// torch_mode = 0: the reference's custom LayerNorm (unbiased std, eps added to the std, transformer.py:73-81);
// torch_mode = 1: nn.LayerNorm (biased variance, eps under the root; FCModel.input_norm, model.py:27) -- `sd` then
// receives sqrt(var + eps) and ln_backward must be called with eps = 0 and torch_mode = 1
int ln_forward(const float* x, const float* a, const float* b, float eps, long long rows, int width, float* y,
               float* mean, float* sd, cudaStream_t st, int torch_mode = 0,
               void* y16 = nullptr,    // y16 != nullptr: write the output as bfloat16 there INSTEAD of y (bf16 mode)
               const int* rows_dev = nullptr,    // packed rows: device pointer to the live row count (<= rows)
               const int* rowmap_out = nullptr); // packed rows: write row r to y[rowmap_out[r]] (< 0: not at all); fp32
// dx = (dres ? dres : 0) + LayerNormBackward(dy); grad_a / grad_b (null: not computed) are accumulated
int ln_backward(const float* dy, const float* x, const float* a, const float* mean, const float* sd, float eps,
                const float* dres, long long rows, int width, float* dx, float* grad_a, float* grad_b,
                cudaStream_t st, float* dx_masked = nullptr, DropSite site = DropSite{0u, 0u, 1.0f},
                float* colsum_out = nullptr,    // colsum_out[c] += column sums of the emitted (masked) gradient
                int torch_mode = 0,
                const void* dy16_in = nullptr,  // bf16 mode: dy is read from this bfloat16 buffer instead
                void* dy16_out = nullptr,       // bf16 mode: bfloat16 copy of the emitted (masked) gradient
                const int* rows_dev = nullptr,
                const int* rowmap_in = nullptr);  // packed rows: dy of row r is dy[rowmap_in[r]] (< 0: zero); fp32
int pos_forward(float* x, const long long* indices, const uint8_t* mask, const float* pe, int pe_rows, float scale,
                long long rows, int width, cudaStream_t st);
int pos_backward(const float* dx, const long long* indices, const uint8_t* mask, float* dpe, int pe_rows, long long rows,
                 int width, cudaStream_t st);
// site.thresh != 0: inverted dropout on the probabilities (index ((b*h+head)*S+q)*S+key, as in the fused kernels);
// the backward then expects `prob` = the UNDROPPED probabilities and overwrites it with the dropped ones
// FC-block activations (model.py:41-43): h <- dropout(act(h)) in place; backward: dz = mul * dh * mask/(1-p) * act'
// from the stored output h, colsum_out[c] += column sums of dz.  act: ARB_ACT_*
int act_forward(float* h, long long rows, int width, int act, DropSite site, cudaStream_t st,
                const int* rows_dev = nullptr);
int act_backward(const float* dh, const float* h, float* dz, long long rows, int width, int act, DropSite site, float mul,
                 float* colsum_out, cudaStream_t st, const int* rows_dev = nullptr);
int softmax_forward(float* sc, const uint8_t* mask, int B, int h, int S, int pitch, cudaStream_t st,
                    DropSite site = DropSite{0u, 0u, 1.0f});
int softmax_backward(float* dp, float* prob, long long rows, int S, int pitch, cudaStream_t st,
                     DropSite site = DropSite{0u, 0u, 1.0f});
// extent[b] = 1 + the last item r of slate b that is a real key (mask == 0) or -- when `dscores` is given -- carries a
// non-zero score gradient (any of its n_out outputs); 0 for a slate without such an item.  Rows at or beyond the extent
// are padding whose activations gradients are exactly zero in every layer, and keys no query attends to.
int slate_extents(const uint8_t* mask, const float* dscores, int n_out, int B, int S, int* extent, cudaStream_t st);
// flat fp32 -> bfloat16 copy (the GEMM-operand shadow of the parameter buffer in bf16 mode); n multiple of 4
int convert_to_bf16(const float* src, void* dst, long long n, cudaStream_t st);
// The weight matrices inside the flat parameter buffer: FC layer i at fc_w[i] ([fc_out[i], fc_in[i]] row-major) and the
// four of encoder layer l at enc0 + l * enc_stride + {0, o_wo, o_w1, o_w2} ([3d, d], [d, d], [f, d], [d, f]).
struct WeightMats {
  int n_fc;
  long long fc_w[8];
  int fc_out[8], fc_in[8];
  int n_layers, d, f;
  long long enc0, enc_stride, o_wo, o_w1, o_w2;
};
// The GEMM-operand copy of the parameter buffer in TF32 mode, one launch: pr[i] = P[i] and, for every weight matrix
// W [out, in] at offset o, pt[o + c * out + r] = W[r][c] (W^T, the K-major B operand of the input gradient); values
// rounded to tf32 (nearest even) when rnd != 0, else copied as they are (the tensor core then truncates them).
int tf32_weight_copy(const float* P, long long n, const WeightMats& m, int rnd, float* pr, float* pt, cudaStream_t st);
// Padded heads (DESIGN.md 4.15): when the head width w = d / h is not a multiple of 4, every head of Q | K | V, the
// context and their gradients takes hs = round_up(w, 4) columns, the last hs - w of them exact zeros, so that the
// per-head tensor maps get a head stride of a multiple of 16 bytes.  The attention linears then read padded copies of
// their weights, one block of size() floats per layer (dp = h * hs):
//   wqkv [3 dp, d] (zero rows in the pads), wqkvt = wqkv^T [d, 3 dp], bqkv [3 dp], wo [d, dp] (zero columns in the
//   pads), wot = wo^T [dp, d]
// and write their weight and bias gradients to a padded block of gsize() floats: gwqkv [3 dp, d], gbqkv [3 dp],
// gwo [d, dp].  Every offset is a multiple of 4 floats (16 bytes, as TMA needs).
struct HeadPad {
  int n_layers, d, h, w, hs;
  long long enc0, enc_stride, o_bqkv, o_wo;   // flat parameters: layer l at enc0 + l * enc_stride; b_qkv, W_o inside it
  __host__ __device__ long long dp() const { return (long long)h * hs; }
  __host__ __device__ long long wqkv() const { return 0; }
  __host__ __device__ long long wqkvt() const { return 3 * dp() * d; }
  __host__ __device__ long long bqkv() const { return 6 * dp() * d; }
  __host__ __device__ long long wo() const { return 6 * dp() * d + 3 * dp(); }
  __host__ __device__ long long wot() const { return 7 * dp() * d + 3 * dp(); }
  __host__ __device__ long long size() const { return 8 * dp() * d + 3 * dp(); }
  __host__ __device__ long long gwqkv() const { return 0; }
  __host__ __device__ long long gbqkv() const { return 3 * dp() * d; }
  __host__ __device__ long long gwo() const { return 3 * dp() * d + 3 * dp(); }
  __host__ __device__ long long gsize() const { return 4 * dp() * d + 3 * dp(); }
};
// out[l * m.size() + ...] = the padded copies of every layer: weights from pr (the TF32 copy), the bias from P
int head_pad_copy(const float* pr, const float* P, const HeadPad& m, float* out, cudaStream_t st);
// G += the real rows and columns of layer l's padded gradient block gp (each element one addition: no atomics)
int head_pad_grads(const float* gp, const HeadPad& m, int l, float* G, cudaStream_t st);
int colsum_accumulate(const float* in, long long rows, int width, long long ld, float* out, cudaStream_t st);
int head_forward(const float* x, const float* a, const float* b, float eps, const float* w, const float* wb,
                 int has_norm, int act, long long rows, int width, float* score, float* mean, float* sd,
                 cudaStream_t st, const int* rows_dev = nullptr,
                 const int* rowmap = nullptr);   // packed rows: score[rowmap[row]] (rows with rowmap < 0 have no score)
int head_backward(const float* dscore, const float* score, const float* x, const float* a, const float* b,
                  const float* mean, const float* sd, float eps, const float* w, const float* wb, int has_norm,
                  int act, long long rows, int width, float* dx,
                  float* grad_a, float* grad_b, float* grad_w,   // (gradient outputs: null = not computed)
                  float* grad_wb, cudaStream_t st, float* dx_masked = nullptr,
                  DropSite site = DropSite{0u, 0u, 1.0f}, float* colsum_out = nullptr, void* dy16_out = nullptr,
                  const int* rows_dev = nullptr, const int* rowmap = nullptr);
// Packed rows (padding removal; see scorer_kernels.cu): from the slate extents build off [B+1], plan [2] and
// rowmap [B*S] and copy the features of the packed rows into xc
int pack_plan(const float* x, const int* ext, int B, int S, int F, int* off, int* plan, int* rowmap, float* xc,
              long long cap_rows,   // rows the packed buffers hold (B * round_up(S, 16))
              cudaStream_t st);
// Zero rows behind the packed rows of several buffers in one launch (pitch / width in floats): from = 0: n rows after
// the packed rows (plan[0]), capped at cap_rows; from = 1: the alignment rows between the slates' rows (plan[1]) and
// the packed row count (plan[0]).  See scorer_kernels.cu.
struct ZeroRegion { float* p; int pitch, width, from, n; };
struct ZeroRegions {
  static constexpr int MAX = 16;
  ZeroRegion r[MAX];
  int count = 0;
  bool add(float* p, int pitch, int width, int from, int n) {
    if (count >= MAX) return false;
    r[count++] = ZeroRegion{p, pitch, width, from, n};
    return true;
  }
};
int zero_rows(const ZeroRegions& z, const int* plan, long long cap_rows, cudaStream_t st);
// dst[rowmap[r]] = src[r] for the packed rows r below plan[1] (and cap_rows); dst is dense [B * S, width], zero-filled
// by the caller
int scatter_rows(const float* src, const int* plan, const int* rowmap, long long cap_rows, int width, float* dst,
                 cudaStream_t st);
// d_output = n > 1: scores [rows, n] from the (already normalised) rows xf; see scorer_kernels.cu
int head_multi_forward(const float* xf, const float* w, const float* wb, int act, long long rows, int width, int n,
                       float* score, cudaStream_t st);
int head_multi_backward(const float* dscore, const float* score, const float* xf, const float* w, int act,
                        long long rows, int width, int n, float* dxf, float* grad_w, float* grad_wb, cudaStream_t st,
                        float* dx_masked = nullptr, DropSite site = DropSite{0u, 0u, 1.0f},
                        float* colsum_out = nullptr);

}  // namespace arb
