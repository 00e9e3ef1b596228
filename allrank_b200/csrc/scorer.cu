// Scorer orchestration: LTRModel forward and backward as a fixed sequence of kernel launches on one stream.
//
//   forward : x -> FC -> N x [ LN -> QKV -> (Q K^T / sqrt(dk), key mask, softmax, P V) -> O + residual
//                               -> LN -> W1 + ReLU -> W2 + residual ] -> LN -> head
//   backward: the exact reverse, parameter gradients accumulated into a flat buffer.
//   encode  : the forward without the head: the final LayerNorm's output [B, S, d] (LTRModel.prepare_for_output);
//             backward_ex starts from its gradient instead of the score's and can also emit d loss / d x.
//
// Reference: allrank/models/model.py:62-92 (LTRModel), allrank/models/transformer.py:43-56,126-134,178-203,227.
// Every contraction is a launch of the tensor-core TF32 GEMM (gemm_tf32.cu) -- per-head attention products are
// batched launches over 4-D tensor maps (head and slate are TMA coordinates, so no transposes/copies exist:
// the reference's `transpose(1,2).contiguous()` at transformer.py:201 vanishes).  The host sequence contains no
// synchronisation and only stream-ordered allocations (the reduction slots, common.h: DetParts), so a training step can
// be captured into a CUDA graph by the host layer.
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

#include "attention_fused.h"
#include "common.h"
#include "defaults.h"
#include "gemm_tf32.h"
#include "scorer_kernels.h"

namespace arb {

static inline int64_t align_up(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

// 0: unfused attention (materialised [B,h,S,S] logits, generic GEMMs)   1: fused forward kernel, unfused backward
// 2 (default): fused forward and fused backward kernels
static int g_attn_mode = 2;
// 1 (default): the fused attention kernels skip the tiles that lie entirely in a slate's padding (exact: masked keys
// have probability 0 and padded rows a zero gradient); 0: dense tiles, for A/B measurements
static int g_skip_padding = ARB_DEFAULT_SKIP_PADDING;
// 1 (default): packed rows -- the encoder runs over the items below every slate's extent only (padding removal; exact
// for every real item and every parameter gradient; scores of padded items are then 0 instead of what the network
// computes for an all-zero feature row, which every consumer in allRank masks: DESIGN.md 4.12); 0: dense [B*S] rows
static int g_pack_rows = ARB_DEFAULT_PACK_ROWS;
static bool use_fused(const arb_scorer_config& c, int S) {
  return g_attn_mode >= 1 && c.n_layers > 0 && attn_fused_supported(S, c.d_model / c.n_heads);
}
static bool use_fused_bwd(const arb_scorer_config& c, int S) {
  return g_attn_mode >= 2 && use_fused(c, S) && attn_fused_bwd_supported(S, c.d_model / c.n_heads);
}

static inline int n_outputs(const arb_scorer_config& c) { return c.d_output > 1 ? c.d_output : 1; }

// The FFN's ReLU backward reads the forward's bit mask (1 bit per hidden unit, written by the W1 epilogue) instead of the
// fp32 hidden activation as a mask tile: 1 GB less read per layer at the headline shape.  TF32 mode without dropout
// (the dropout and bf16 epilogues keep the mask-tile path), d_ff a multiple of 32.
static int g_relu_bits = ARB_DEFAULT_RELU_BITS;
static bool relu_bits(const arb_scorer_config& c) {
  return g_relu_bits && c.n_layers > 0 && !c.bf16 && c.dropout == 0.0f && c.d_ff % 32 == 0;
}

// Packed rows need both fused attention kernels (they take per-slate row offsets) and, so far, a call without dropout
// (its counters index the dense layout), without a positional encoding and with a single output per item.
static bool pack_eligible(const arb_scorer_config& c, int S) {
  return c.n_layers > 0 && use_fused_bwd(c, S) && c.dropout == 0.0f && c.fc_dropout == 0.0f && c.pe_mode == 0 &&
         n_outputs(c) == 1;
}
static bool use_pack(const arb_scorer_config& c, int S) { return g_pack_rows && g_skip_padding && pack_eligible(c, S); }

struct ParamLayout {
  int n_fc;                                  // FC layers (>= 1)
  int fc_size[ARB_MAX_FC_LAYERS];            // output width of FC layer i; fc_size[n_fc-1] = d_model
  int64_t fc_w[ARB_MAX_FC_LAYERS], fc_b[ARB_MAX_FC_LAYERS];
  int64_t in_a, in_b;                        // nn.LayerNorm(F) of fc_model.input_norm (-1: none)
  struct Layer { int64_t wqkv, bqkv, wo, bo, w1, b1, w2, b2, ln1_a, ln1_b, ln2_a, ln2_b; };
  Layer layer[64];
  int64_t lnf_a, lnf_b, head_w, head_b, pe, total;
};

static int make_param_layout(const arb_scorer_config& c, ParamLayout& L) {
  if (c.n_layers < 0 || c.n_layers > 64) { arb_set_error("scorer: n_layers must be in [0,64]"); return ARB_E_UNSUPPORTED; }
  if (c.d_model <= 0 || c.d_model % 4 || c.n_features <= 0 || c.n_features % 4) {
    arb_set_error("scorer: d_model and (padded) n_features must be positive multiples of 4");
    return ARB_E_UNSUPPORTED;
  }
  if (c.n_layers > 0) {
    if (c.n_heads <= 0 || c.d_model % c.n_heads || (c.d_model / c.n_heads) % 4 || c.d_ff <= 0 || c.d_ff % 4) {
      arb_set_error("scorer: need d_model % h == 0, (d_model/h) % 4 == 0 and d_ff % 4 == 0");
      return ARB_E_UNSUPPORTED;
    }
    if (c.d_model / c.n_heads > 128) { arb_set_error("scorer: head width above 128 is not supported"); return ARB_E_UNSUPPORTED; }
  }
  if (c.d_model > 1024) { arb_set_error("scorer: d_model above 1024 is not supported"); return ARB_E_UNSUPPORTED; }
  if (c.bf16 && c.n_layers > 0 && (c.d_model % 8 || c.d_ff % 8 || c.d_model < 64 || c.d_ff < 64)) {
    arb_set_error("scorer: bf16 mode needs d_model and d_ff to be multiples of 8, at least 64");
    return ARB_E_UNSUPPORTED;
  }
  const int64_t d = c.d_model, F = c.n_features, f = c.d_ff;
  L.n_fc = c.n_fc_layers > 0 ? c.n_fc_layers : 1;
  if (L.n_fc > ARB_MAX_FC_LAYERS) { arb_set_error("scorer: at most 8 FC layers"); return ARB_E_UNSUPPORTED; }
  for (int i = 0; i < L.n_fc; ++i) {
    L.fc_size[i] = c.n_fc_layers > 0 ? c.fc_sizes[i] : c.d_model;
    if (L.fc_size[i] <= 0 || L.fc_size[i] % 4 || L.fc_size[i] > 8192) {
      arb_set_error("scorer: FC layer widths must be positive multiples of 4, at most 8192");
      return ARB_E_UNSUPPORTED;
    }
  }
  if (L.fc_size[L.n_fc - 1] != c.d_model) { arb_set_error("scorer: the last FC width must equal d_model"); return ARB_E_INVALID_ARG; }
  if (c.fc_act < ARB_ACT_NONE || c.fc_act > ARB_ACT_RELU) { arb_set_error("scorer: unknown FC activation"); return ARB_E_UNSUPPORTED; }
  if (c.fc_input_norm && F > 1024) { arb_set_error("scorer: input_norm supports up to 1024 features"); return ARB_E_UNSUPPORTED; }
  int64_t o = 0;
  for (int i = 0; i < L.n_fc; ++i) {
    const int64_t in = i == 0 ? F : L.fc_size[i - 1];
    L.fc_w[i] = o; o += int64_t(L.fc_size[i]) * in;
    L.fc_b[i] = o; o += L.fc_size[i];
  }
  L.in_a = L.in_b = -1;
  if (c.fc_input_norm) { L.in_a = o; o += F; L.in_b = o; o += F; }
  // the encoder's parameters start on a 32-byte boundary (8 elements): their bfloat16 shadow (bf16 mode) is read by TMA,
  // which needs 16-byte aligned bases; every size inside the encoder section is then a multiple of 8 elements
  if (c.n_layers > 0) o = align_up(o, 8);
  for (int l = 0; l < c.n_layers; ++l) {
    auto& y = L.layer[l];
    y.wqkv = o; o += 3 * d * d;
    y.bqkv = o; o += 3 * d;
    y.wo = o; o += d * d;
    y.bo = o; o += d;
    y.w1 = o; o += f * d;
    y.b1 = o; o += f;
    y.w2 = o; o += d * f;
    y.b2 = o; o += d;
    y.ln1_a = o; o += d;
    y.ln1_b = o; o += d;
    y.ln2_a = o; o += d;
    y.ln2_b = o; o += d;
  }
  if (c.n_layers > 0) { L.lnf_a = o; o += d; L.lnf_b = o; o += d; } else { L.lnf_a = L.lnf_b = -1; }
  if (c.d_output < 0 || c.d_output > 64) { arb_set_error("scorer: d_output must be in [1,64]"); return ARB_E_UNSUPPORTED; }
  const int64_t n_out = n_outputs(c);
  L.head_w = o; o += n_out * d;      // nn.Linear(d, d_output).weight, row-major [d_output, d]
  L.head_b = o; o += n_out;
  L.pe = -1;
  if (c.pe_mode != 0) {
    if (c.n_layers == 0 || c.pe_rows < 2 || c.pe_mode < 0 || c.pe_mode > 2) {
      arb_set_error("scorer: positional encoding needs a transformer and a table of >= 2 rows");
      return ARB_E_UNSUPPORTED;
    }
    if (c.pe_mode == 2) { o = align_up(o, 4); L.pe = o; o += int64_t(c.pe_rows) * d; }
  }
  L.total = o;
  return ARB_OK;
}

struct WsLayout {
  int64_t x0;
  int64_t fch[ARB_MAX_FC_LAYERS];   // outputs of the FC layers before the last (training: kept for backward)
  int64_t fc_last;                  // last FC output before the positional encoding overwrites x0 (activated FC + PE)
  int64_t xnorm, in_mean, in_std;   // input_norm output and row statistics
  struct Layer { int64_t xn1, mean1, std1, qkv, prob, smax, ssum, ctx, xmid, xn2, mean2, std2, hdn, xout, hbits; };
  Layer layer[64];
  int64_t kext;                     // [B] ints: key extent of every slate (keys at or beyond it are all masked)
  int64_t xc, poff, plan, rowmap;   // packed rows: features of the packed rows, off [B+1], plan [2], rowmap [B*S] (ints)
  int64_t wb16;                     // bf16 mode: bfloat16 shadow of the whole parameter buffer (same element offsets)
  int64_t meanf, stdf, xf, total;   // xf: final-norm output, kept only for the multi-output head
  int Sp;
  bool fused;
};

// Rows the activation buffers hold: B * S, or -- when the call can run over packed rows, whose slates occupy multiples
// of 16 rows -- B * round_up(S, 16).
static int64_t buffer_rows(const arb_scorer_config& c, int B, int S) {
  return int64_t(B) * (pack_eligible(c, S) ? align_up(S, 16) : int64_t(S));
}

static void make_ws_layout(const arb_scorer_config& c, const ParamLayout& L, int B, int S, int training, WsLayout& W) {
  const int64_t R = buffer_rows(c, B, S), d = c.d_model, f = c.d_ff, h = c.n_heads;
  W.Sp = int(align_up(S, 4));
  W.fused = use_fused(c, S);
  int64_t o = 0;
  auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
  W.x0 = take(R * d);
  {
    int64_t ping[2] = {0, 0};
    if (!training && L.n_fc > 1) {   // eval: two buffers of the widest hidden layer, used alternately
      int64_t widest = 0;
      for (int i = 0; i + 1 < L.n_fc; ++i) widest = std::max<int64_t>(widest, L.fc_size[i]);
      ping[0] = take(R * widest);
      ping[1] = L.n_fc > 2 ? take(R * widest) : ping[0];
    }
    for (int i = 0; i < ARB_MAX_FC_LAYERS; ++i)
      W.fch[i] = (i + 1 < L.n_fc) ? (training ? take(R * L.fc_size[i]) : ping[i & 1]) : 0;
  }
  W.fc_last = (training && c.fc_act != ARB_ACT_NONE && c.pe_mode != 0) ? take(R * d) : 0;
  W.xnorm = W.in_mean = W.in_std = 0;
  if (c.fc_input_norm) { W.xnorm = take(R * c.n_features); W.in_mean = take(R); W.in_std = take(R); }
  // bf16 mode: tensors that only feed products (LayerNorm outputs, context, FFN hidden) are bfloat16: half the floats
  const int64_t op = (c.bf16 && c.n_layers > 0) ? 2 : 1;
  W.wb16 = op == 2 ? take((L.total + 1) / 2) : 0;
  WsLayout::Layer shared{};
  for (int l = 0; l < c.n_layers; ++l) {
    auto& y = W.layer[l];
    if (training || l == 0) {
      y.xn1 = take(R * d / op); y.mean1 = take(R); y.std1 = take(R);
      y.qkv = take(R * 3 * d);
      y.prob = W.fused ? 0 : take(int64_t(B) * h * S * W.Sp);
      y.smax = take(int64_t(B) * h * S);
      y.ssum = take(int64_t(B) * h * S);
      y.ctx = take(R * d / op);
      y.xn2 = training ? take(R * d / op) : y.xn1;
      y.mean2 = training ? take(R) : y.mean1;
      y.std2 = training ? take(R) : y.std1;
      y.hdn = take(R * f / op);
      y.hbits = (training && relu_bits(c)) ? take(R * (f / 32)) : 0;   // ReLU bit mask of the hidden layer: 1 bit per unit
      y.xmid = training ? take(R * d) : W.x0;    // eval: the residual stream is updated in place
      y.xout = training ? take(R * d) : W.x0;
      shared = y;
    } else {
      y = shared;
    }
  }
  W.kext = take(B);
  W.xc = W.poff = W.plan = W.rowmap = 0;
  if (pack_eligible(c, S)) { W.xc = take(R * c.n_features); W.poff = take(B + 1); W.plan = take(2); W.rowmap = take(R); }
  W.meanf = take(R);
  W.stdf = take(R);
  W.xf = (n_outputs(c) > 1 && c.n_layers > 0) ? take(R * d) : 0;
  W.total = o;
}

struct Ctx {
  const arb_scorer_config& c;
  int B, S;
  int64_t R;
  cudaStream_t st;
  const int* rows_dev = nullptr;   // packed rows: device pointer to the live row count (plan[0]); R is the upper bound
};

// ---- GEMM helpers ------------------------------------------------------------------------------
// A pointer with its element type: fp32 (implicitly, from any float*) or bfloat16 (b16(...)) -- bf16 mode.
struct V {
  const void* p;
  int bf16;
  V(const float* q = nullptr) : p(q), bf16(0) {}
  V(const void* q, int is16) : p(q), bf16(is16) {}
};
static inline V b16(const void* q) { return V(q, 1); }

static TRef rows_view(V v, int64_t inner, int64_t rows, int64_t pitch) {
  TRef t; t.ptr = v.p; t.bf16 = v.bf16; t.dim[0] = inner; t.dim[1] = rows; t.stride[0] = 1; t.stride[1] = pitch; return t;
}
static int pick_block_n(int n) { return n <= 32 ? 32 : (n < 128 ? 64 : 128); }

// Y[R,out] = epi( X[R,in] W[out,in]^T + bias )
static int linear_fwd(const Ctx& k, V X, int64_t x_pitch, int in, V Wt, const float* bias, int out,
                      V Y, int64_t y_pitch, int flags, V aux, int64_t aux_pitch,
                      DropSite drop = DropSite{0u, 0u, 1.0f}, uint32_t* relu_bits_out = nullptr) {
  GemmDesc g;
  g.M = int(k.R); g.N = out; g.K = in;
  g.drop = drop;
  if (drop.thresh != 0) flags |= EPI_DROPOUT;
  g.A = rows_view(X, in, k.R, x_pitch);
  g.B = rows_view(Wt, in, out, in);
  g.C = rows_view(Y, out, k.R, y_pitch);
  if (aux.p) g.Aux = rows_view(aux, out, k.R, aux_pitch);
  g.bias = bias; g.flags = flags | (bias ? EPI_BIAS : 0);
  if (relu_bits_out) { g.flags |= EPI_RELU_BITS; g.bits = relu_bits_out; }
  g.block_n = pick_block_n(out);
  if (Y.bf16 && g.block_n < 64) g.block_n = 64;
  g.rows_dev = k.rows_dev;
  return launch_gemm_tf32(g, k.st);
}
// dX[R,in] = epi( dY[R,out] W[out,in] )      (W read as an MN-major B operand)
static int linear_bwd_input(const Ctx& k, V dY, int64_t dy_pitch, int out, V Wt, int in, V dX,
                            int64_t dx_pitch, int flags, V aux, int64_t aux_pitch, float alpha = 1.0f,
                            float* colsum_out = nullptr, const uint32_t* mask_bits = nullptr) {
  GemmDesc g;
  g.alpha = alpha;
  g.colsum_out = colsum_out;
  if (!colsum_out) flags &= ~EPI_COLSUM;     // (no parameter gradients requested)
  g.M = int(k.R); g.N = in; g.K = out; g.b_mn = 1;
  g.A = rows_view(dY, out, k.R, dy_pitch);
  g.B = rows_view(Wt, in, out, in);          // dim0 = in (N, contiguous), dim1 = out (K)
  g.C = rows_view(dX, in, k.R, dx_pitch);
  if (aux.p) g.Aux = rows_view(aux, in, k.R, aux_pitch);
  g.flags = flags;
  if (mask_bits) { g.flags |= EPI_MASK_BITS; g.bits = const_cast<uint32_t*>(mask_bits); }
  g.block_n = pick_block_n(in);
  if (dX.bf16 && g.block_n < 64) g.block_n = 64;
  g.rows_dev = k.rows_dev;
  return launch_gemm_tf32(g, k.st);
}
// dW[out,in] += dY[R,out]^T X[R,in]          (both operands MN-major, reduction over all rows, split-K)
static int linear_bwd_weight(const Ctx& k, V dY, int64_t dy_pitch, int out, V X, int64_t x_pitch,
                             int in, float* dW) {
  GemmDesc g;
  g.M = out; g.N = in; g.K = int(k.R); g.a_mn = 1; g.b_mn = 1;
  g.A = rows_view(dY, out, k.R, dy_pitch);
  g.B = rows_view(X, in, k.R, x_pitch);
  g.flags = EPI_ATOMIC; g.atomic_out = dW; g.atomic_ld = in;
  g.block_n = pick_block_n(in);
  const int tiles = ((out + 127) / 128) * ((in + g.block_n - 1) / g.block_n);
  const int kel = dY.bf16 ? 64 : 32;          // rows of the batch per k-block
  const int kb = int((k.R + kel - 1) / kel);
  // 4-stage ring => 1 CTA per SM: one wave of ~132 CTAs (H100 SXM) (fewer splits = fewer L2 reductions of the dW tile)
  g.split_k = std::max(1, std::min(kb / 8 + 1, std::max(1, 132 / tiles)));
  g.rows_dev = k.rows_dev;
  return launch_gemm_tf32(g, k.st);
}

// per-head strided view of a [R, pitch] activation: dims (dk, S, h, B)
static TRef head_view(V v, int dk, int S, int h, int B, int64_t pitch) {
  TRef t; t.ptr = v.p; t.bf16 = v.bf16;
  t.dim[0] = dk; t.dim[1] = S; t.dim[2] = h; t.dim[3] = B;
  t.stride[0] = 1; t.stride[1] = pitch; t.stride[2] = dk; t.stride[3] = int64_t(S) * pitch;
  return t;
}
// [B,h,S,Sp] probability / logit buffers: dims (S, S, h, B)
static TRef prob_view(const float* p, int S, int Sp, int h, int B) {
  TRef t; t.ptr = p;
  t.dim[0] = S; t.dim[1] = S; t.dim[2] = h; t.dim[3] = B;
  t.stride[0] = 1; t.stride[1] = Sp; t.stride[2] = int64_t(S) * Sp; t.stride[3] = int64_t(h) * S * Sp;
  return t;
}
static void batch_all(GemmDesc& g, int h, int B) {
  g.nb2 = h; g.nb3 = B;
  g.a_b2 = g.a_b3 = g.b_b2 = g.b_b3 = g.c_b2 = g.c_b3 = 1;
}

#define ARB_TRY(expr) do { int rc__ = (expr); if (rc__ != ARB_OK) return rc__; } while (0)

// Exactly one of `scores` (the model's output) and `hidden` (the encoder's output, [B, S, d]; the head is not run) is
// non-null.
static int forward_impl(const arb_scorer_config& c, const float* P, const float* x, const uint8_t* mask,
                        const int64_t* indices, const float* pe_table, int B, int S,
                        float* scores, float* hidden, float* ws, int64_t ws_floats, int training, uint64_t seed,
                        cudaStream_t st) {
  ParamLayout L;
  ARB_TRY(make_param_layout(c, L));
  WsLayout W;
  make_ws_layout(c, L, B, S, training, W);
  if (ws_floats < W.total) { arb_set_error("arb_scorer_forward: workspace too small"); return ARB_E_WORKSPACE; }
  Ctx k{c, B, S, int64_t(B) * S, st};
  const int d = c.d_model, F = c.n_features, f = c.d_ff, h = c.n_heads;
  const int dk = c.n_layers > 0 ? d / h : 0;

  // dropout follows the module's train()/eval() mode (the host zeroes these in eval); `training` only selects
  // whether activations are kept for a backward pass
  const float p_drop = c.dropout, p_fc = c.fc_dropout;
  // bf16 mode (cfg.bf16): encoder linears as bfloat16 products; see include/allrank_b200.h
  const bool bf = c.bf16 && c.n_layers > 0;
  uint16_t* Pb = bf ? reinterpret_cast<uint16_t*>(ws + W.wb16) : nullptr;
  if (bf) {
    if (!use_fused_bwd(c, S)) {
      arb_set_error("scorer: bf16 mode needs the fused attention kernels (slate_length <= 256, head width 16 or 32)");
      return ARB_E_UNSUPPORTED;
    }
    ARB_TRY(convert_to_bf16(P, Pb, L.total, st));      // refresh the GEMM-operand shadow of the master weights
  }
  auto wt = [&](int64_t off) { return bf ? b16(Pb + off) : V(P + off); };
  auto act = [&](float* q) { return bf ? b16(q) : V(q); };   // a product-only activation buffer of this mode
  float* xcur = ws + W.x0;
  int* kext = reinterpret_cast<int*>(ws + W.kext);
  if (c.n_layers > 0 && W.fused && g_skip_padding)
    ARB_TRY(slate_extents(mask, nullptr, 0, B, S, kext, st));   // once per call, shared by every layer
  if (c.n_layers > 0 && W.fused && g_skip_padding && arb_prof_enabled()) {
    // per-launch accounting (bench.py): the attention kernels stop at the extents, so their flops are counted over the
    // real items -- sum_b round_up(extent_b, 16)^2 of the dense B * S^2 (read back here: profiling only)
    std::vector<int> he(static_cast<size_t>(B));
    if (cudaStreamSynchronize(st) != cudaSuccess ||
        cudaMemcpy(he.data(), kext, size_t(B) * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) {
      arb_set_error("scorer: reading the slate extents failed"); return ARB_E_CUDA;
    }
    double sq = 0.0;
    for (int e : he) { const double r = double((std::max(0, std::min(S, e)) + 15) & ~15); sq += r * r; }
    arb_set_attn_frac(sq / (double(B) * double(S) * double(S)));
  } else if (arb_prof_enabled()) {
    arb_set_attn_frac(1.0);
  }
  // Packed rows: every kernel below runs over the rows below the slates' extents only (scorer_kernels.cu: pack_plan)
  const bool pack = use_pack(c, S);
  const int* plan = nullptr;
  const int* rowmap = nullptr;
  const int* poff = nullptr;
  if (pack) {
    plan = reinterpret_cast<const int*>(ws + W.plan);
    rowmap = reinterpret_cast<const int*>(ws + W.rowmap);
    poff = reinterpret_cast<const int*>(ws + W.poff);
    ARB_TRY(pack_plan(x, kext, B, S, F, reinterpret_cast<int*>(ws + W.poff), reinterpret_cast<int*>(ws + W.plan),
                      reinterpret_cast<int*>(ws + W.rowmap), ws + W.xc, buffer_rows(c, B, S), st));
    // items beyond their slate's extent get the score 0 (encoder output: a zero row)
    float* const out = hidden ? hidden : scores;
    const size_t out_floats = size_t(B) * S * (hidden ? d : 1);
    if (cudaMemsetAsync(out, 0, out_floats * sizeof(float), st) != cudaSuccess) { arb_set_error("scorer: memset failed"); return ARB_E_CUDA; }
    k.R = buffer_rows(c, B, S);       // upper bound of the packed row count (grids, tensor maps)
    if (arb_prof_enabled()) {     // per-launch accounting (bench.py) needs the live row count on the host
      int live = 0;
      if (cudaStreamSynchronize(st) != cudaSuccess || cudaMemcpy(&live, plan, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) {
        arb_set_error("scorer: reading the packed row count failed"); return ARB_E_CUDA;
      }
      arb_set_row_frac(double(live) / double(k.R));   // launches account with k.R nominal rows
    }
    k.rows_dev = plan;
    x = ws + W.xc;
  }
  {   // FCModel (model.py:35-44): [nn.LayerNorm(F)] then dropout(act(Linear)) per layer
    const float* hin = x;
    int in = F;
    if (c.fc_input_norm) {
      ARB_TRY(ln_forward(x, P + L.in_a, P + L.in_b, 1e-5f, k.R, F, ws + W.xnorm, ws + W.in_mean, ws + W.in_std, st, 1,
                         nullptr, plan));
      hin = ws + W.xnorm;
    }
    for (int i = 0; i < L.n_fc; ++i) {
      const int out = L.fc_size[i];
      const bool last = i + 1 == L.n_fc;
      float* hout = last ? (W.fc_last ? ws + W.fc_last : xcur) : ws + W.fch[i];
      const DropSite site = make_drop_site(seed, i, SITE_FC, p_fc);
      if (c.fc_act == ARB_ACT_NONE || c.fc_act == ARB_ACT_RELU) {
        ARB_TRY(linear_fwd(k, hin, in, in, P + L.fc_w[i], P + L.fc_b[i], out, hout, out,
                           c.fc_act == ARB_ACT_RELU ? EPI_RELU : 0, nullptr, 0, site));
      } else {
        ARB_TRY(linear_fwd(k, hin, in, in, P + L.fc_w[i], P + L.fc_b[i], out, hout, out, 0, nullptr, 0));
        ARB_TRY(act_forward(hout, k.R, out, c.fc_act, site, st, plan));
      }
      hin = hout; in = out;
    }
    if (W.fc_last) {   // keep the activated FC output for backward: the positional encoding rewrites x0 in place
      if (cudaMemcpyAsync(xcur, ws + W.fc_last, size_t(k.R) * d * sizeof(float), cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
        arb_set_error("scorer: device copy failed"); return ARB_E_CUDA;
      }
    }
  }
  if (c.pe_mode != 0) {   // x = sqrt(d) x + pe[indices]   (transformer.py:51-52, positional.py)
    const float* table = c.pe_mode == 2 ? P + L.pe : pe_table;
    if (!indices || !table) { arb_set_error("scorer: positional encoding needs indices and a table"); return ARB_E_INVALID_ARG; }
    ARB_TRY(pos_forward(xcur, reinterpret_cast<const long long*>(indices), mask, table, c.pe_rows, sqrtf(float(d)), k.R, d, st));
  }
  if (pack) {
    // The attention kernels' 128-row boxes overrun the last slates: 256 finite rows behind the packed rows of every
    // layer's Q|K|V; and the context of the alignment rows (no slate writes them) feeds the output projection: zero.
    // Nothing else writes those rows, so one launch serves all layers (eval mode: the layers share one buffer set).
    ZeroRegions z;
    for (int l = 0; l < c.n_layers; ++l) {
      if (l > 0 && !training) break;
      const auto& wl = W.layer[l];
      if (!z.add(ws + wl.qkv, 3 * d, 3 * d, 0, 256) || !z.add(ws + wl.ctx, bf ? d / 2 : d, bf ? d / 2 : d, 1, 0)) {
        ARB_TRY(zero_rows(z, plan, k.R, st));
        z = ZeroRegions{};
        z.add(ws + wl.qkv, 3 * d, 3 * d, 0, 256);
        z.add(ws + wl.ctx, bf ? d / 2 : d, bf ? d / 2 : d, 1, 0);
      }
    }
    if (z.count) ARB_TRY(zero_rows(z, plan, k.R, st));
  }
  // per-head views: dense (dk, S, h, B), or packed (dk, rows, h, 1) with per-slate row offsets inside the kernels
  auto hview = [&](V v, int64_t pitch) { return pack ? head_view(v, dk, int(k.R), h, 1, pitch) : head_view(v, dk, S, h, B, pitch); };
  for (int l = 0; l < c.n_layers; ++l) {
    const auto& pl = L.layer[l];
    const auto& wl = W.layer[l];
    float* xn1 = ws + wl.xn1; float* qkv = ws + wl.qkv; float* prob = ws + wl.prob; float* ctx = ws + wl.ctx;
    float* xmid = ws + wl.xmid; float* xn2 = ws + wl.xn2; float* hdn = ws + wl.hdn; float* xout = ws + wl.xout;
    // ---- self-attention sublayer: x + O(attn(LN(x)))   (transformer.py:133, :105-106)
    ARB_TRY(ln_forward(xcur, P + pl.ln1_a, P + pl.ln1_b, c.ln_eps, k.R, d, xn1, ws + wl.mean1, ws + wl.std1, st, 0,
                       bf ? xn1 : nullptr, plan));
    ARB_TRY(linear_fwd(k, act(xn1), d, d, wt(pl.wqkv), P + pl.bqkv, 3 * d, qkv, 3 * d, 0, nullptr, 0));
    if (W.fused) {
      AttnFwdArgs a;   // QK^T, key mask, softmax, PV in one kernel; the S x S tile never leaves registers
      a.q = hview(qkv, 3 * d);
      a.k = hview(qkv + d, 3 * d);
      a.v = hview(qkv + 2 * d, 3 * d);
      a.o = hview(act(ctx), d);
      a.pack_off = poff;
      a.mask = mask; a.stat_max = ws + wl.smax; a.stat_sum = ws + wl.ssum;
      a.B = B; a.h = h; a.S = S; a.dk = dk; a.scale = 1.0f / sqrtf(float(dk));
      a.drop = make_drop_site(seed, l, SITE_ATTN_P, p_drop);
      a.extent = g_skip_padding ? kext : nullptr;
      ARB_TRY(launch_attn_fwd(a, st));
    } else {
      {
        GemmDesc g;   // logits = Q K^T / sqrt(dk)      (transformer.py:148)
        g.M = S; g.N = S; g.K = dk; g.alpha = 1.0f / sqrtf(float(dk));
        g.A = head_view(qkv, dk, S, h, B, 3 * d);
        g.B = head_view(qkv + d, dk, S, h, B, 3 * d);
        g.C = prob_view(prob, S, W.Sp, h, B);
        batch_all(g, h, B); g.block_n = 64;
        ARB_TRY(launch_gemm_tf32(g, st));
      }
      // key mask + softmax + dropout on the probabilities (transformer.py:150-155); with dropout the buffer holds the
      // dropped probabilities (what P V needs) and the backward recomputes the undropped ones
      ARB_TRY(softmax_forward(prob, mask, B, h, S, W.Sp, st, make_drop_site(seed, l, SITE_ATTN_P, p_drop)));
      {
        GemmDesc g;   // ctx = P V, written straight into the concatenated-heads layout (transformer.py:156, :201-202)
        g.M = S; g.N = dk; g.K = S; g.b_mn = 1;
        g.A = prob_view(prob, S, W.Sp, h, B);
        g.B = head_view(qkv + 2 * d, dk, S, h, B, 3 * d);
        g.C = head_view(ctx, dk, S, h, B, d);
        batch_all(g, h, B); g.block_n = pick_block_n(dk);
        ARB_TRY(launch_gemm_tf32(g, st));
      }
    }
    ARB_TRY(linear_fwd(k, act(ctx), d, d, wt(pl.wo), P + pl.bo, d, xmid, d, EPI_ADD_AUX, xcur, d,
                       make_drop_site(seed, l, SITE_ATTN_OUT, p_drop)));
    // ---- feed-forward sublayer: x + W2 relu(W1 LN(x))   (transformer.py:134, :227)
    ARB_TRY(ln_forward(xmid, P + pl.ln2_a, P + pl.ln2_b, c.ln_eps, k.R, d, xn2, ws + wl.mean2, ws + wl.std2, st, 0,
                       bf ? xn2 : nullptr, plan));
    ARB_TRY(linear_fwd(k, act(xn2), d, d, wt(pl.w1), P + pl.b1, f, act(hdn), f, EPI_RELU, nullptr, 0,
                       make_drop_site(seed, l, SITE_FFN_HID, p_drop),
                       wl.hbits ? reinterpret_cast<uint32_t*>(ws + wl.hbits) : nullptr));
    ARB_TRY(linear_fwd(k, act(hdn), f, f, wt(pl.w2), P + pl.b2, d, xout, d, EPI_ADD_AUX, xmid, d,
                       make_drop_site(seed, l, SITE_FFN_OUT, p_drop)));
    xcur = xout;
  }
  const int has_norm = c.n_layers > 0;
  if (hidden) {   // encoder output (model.py:62-70): the final norm's output, written at the items' places
    if (has_norm)
      return ln_forward(xcur, P + L.lnf_a, P + L.lnf_b, c.ln_eps, k.R, d, hidden, ws + W.meanf, ws + W.stdf, st, 0,
                        nullptr, plan, rowmap);
    // no encoder: the reference's encoder is the identity (model.py:59), so this is the activated FC output
    if (cudaMemcpyAsync(hidden, xcur, size_t(k.R) * d * sizeof(float), cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
      arb_set_error("scorer: device copy failed"); return ARB_E_CUDA;
    }
    return ARB_OK;
  }
  if (n_outputs(c) > 1) {   // d_output > 1: final norm as its own kernel, then one dot product per output (model.py:116)
    const float* xf = xcur;
    if (has_norm) {
      ARB_TRY(ln_forward(xcur, P + L.lnf_a, P + L.lnf_b, c.ln_eps, k.R, d, ws + W.xf, ws + W.meanf, ws + W.stdf, st));
      xf = ws + W.xf;
    }
    return head_multi_forward(xf, P + L.head_w, P + L.head_b, c.out_act, k.R, d, n_outputs(c), scores, st);
  }
  ARB_TRY(head_forward(xcur, has_norm ? P + L.lnf_a : nullptr, has_norm ? P + L.lnf_b : nullptr, c.ln_eps, P + L.head_w,
                       P + L.head_b, has_norm, c.out_act, k.R, d, scores, ws + W.meanf, ws + W.stdf, st, plan, rowmap));
  return ARB_OK;
}

struct ScratchLayout { int64_t dxa, dxb, dxn, dxm, dqkv, dctx, dprob, prob, delta, dfa, dfb, ext, dy16, dxin, total; };
// want_dx: room for d loss / d x over packed rows (backward_ex), after everything the plain backward uses
static void make_scratch_layout(const arb_scorer_config& c, const ParamLayout& L, int B, int S, ScratchLayout& Z,
                                bool want_dx = false) {
  const int64_t R = buffer_rows(c, B, S), d = c.d_model;
  const int Sp = int(align_up(S, 4));
  int64_t o = 0;
  auto take = [&](int64_t n) { int64_t at = o; o += align_up(n, 64); return at; };
  Z.dxa = take(R * d); Z.dxb = take(R * d); Z.dxn = take(R * d);
  Z.dxm = (c.dropout > 0.0f || c.fc_dropout > 0.0f || c.pe_mode != 0) ? take(R * d) : 0;
  if (c.n_layers > 0) {
    Z.dqkv = take(R * 3 * d); Z.dctx = take(R * d);
    const bool fb = use_fused_bwd(c, S);
    Z.dprob = fb ? 0 : take(int64_t(B) * c.n_heads * S * Sp);
    Z.prob = (use_fused(c, S) && !fb) ? take(int64_t(B) * c.n_heads * S * Sp) : 0;
    Z.delta = fb ? take(int64_t(B) * c.n_heads * S) : 0;
  } else {
    Z.dqkv = Z.dctx = Z.dprob = Z.prob = Z.delta = 0;
  }
  // FC-block backward: two gradient buffers of the widest tensor it differentiates through
  int64_t widest = c.fc_input_norm ? c.n_features : 0;
  for (int i = 0; i + 1 < L.n_fc; ++i) widest = std::max<int64_t>(widest, L.fc_size[i]);
  if (c.fc_act != ARB_ACT_NONE) widest = std::max<int64_t>(widest, d);
  Z.dfa = widest ? take(R * widest) : 0;
  Z.dfb = widest ? take(R * widest) : 0;
  Z.ext = take(B);      // [B] ints: gradient extent of every slate
  Z.dy16 = (c.bf16 && c.n_layers > 0) ? take(R * d / 2) : 0;   // bf16 copy of the residual-stream gradient
  Z.dxin = (want_dx && pack_eligible(c, S)) ? take(R * c.n_features) : 0;
  Z.total = o;
}

// The gradient arrives as d loss / d scores (after a forward call) or as d loss / d hidden (after an encode call):
// exactly one of dscores / dhidden is non-null.  G == null: no parameter gradient is computed (no weight-gradient
// product, no gain / bias / column-sum output); dX != null: d loss / d x [B, S, F] is written there.
static int backward_impl(const arb_scorer_config& c, const float* P, const float* x, const uint8_t* mask,
                         const int64_t* indices, int B, int S,
                         const float* scores, const float* dscores, const float* dhidden, float* G, float* dX,
                         float* ws, int64_t ws_floats, float* scratch, int64_t scratch_floats, uint64_t seed,
                         cudaStream_t st) {
  ParamLayout L;
  ARB_TRY(make_param_layout(c, L));
  WsLayout W;
  make_ws_layout(c, L, B, S, 1, W);
  ScratchLayout Z;
  make_scratch_layout(c, L, B, S, Z, dX != nullptr);
  if (ws_floats < W.total) { arb_set_error("arb_scorer_backward: workspace too small"); return ARB_E_WORKSPACE; }
  if (scratch_floats < Z.total) { arb_set_error("arb_scorer_backward: scratch too small"); return ARB_E_WORKSPACE; }
  Ctx k{c, B, S, int64_t(B) * S, st};
  const int d = c.d_model, F = c.n_features, f = c.d_ff, h = c.n_heads;
  const int dk = c.n_layers > 0 ? d / h : 0;
  const float alpha = c.n_layers > 0 ? 1.0f / sqrtf(float(dk)) : 1.0f;
  auto g = [&](int64_t off) { return G ? G + off : nullptr; };   // a parameter's gradient, or null
  float* dx = scratch + Z.dxa;      // gradient w.r.t. the residual stream at the current depth
  float* dx_alt = scratch + Z.dxb;
  float* dxn = scratch + Z.dxn;
  float* dqkv = scratch + Z.dqkv;
  float* dctx = scratch + Z.dctx;
  float* dprob = scratch + Z.dprob;
  float* dxm = scratch + Z.dxm;      // dx seen through the dropout of the sublayer below (masked copy)
  const float p_drop = c.dropout, p_fc = c.fc_dropout;
  const bool drop_on = p_drop > 0.0f;
  // bf16 mode: products read bfloat16 operands -- the weights' shadow (written by the forward call into the
  // workspace), the saved bf16 activations, and bf16 copies of the gradients (dy16: the residual-stream gradient as
  // the sublayer below receives it; dxn / dqkv: gradients that only feed products are bfloat16 outright)
  const bool bf = c.bf16 && c.n_layers > 0;
  if (bf && !use_fused_bwd(c, S)) {
    arb_set_error("scorer: bf16 mode needs the fused attention kernels (slate_length <= 256, head width 16 or 32)");
    return ARB_E_UNSUPPORTED;
  }
  const uint16_t* Pb = bf ? reinterpret_cast<const uint16_t*>(ws + W.wb16) : nullptr;
  void* dy16 = bf ? static_cast<void*>(scratch + Z.dy16) : nullptr;
  auto wt = [&](int64_t off) { return bf ? b16(Pb + off) : V(P + off); };
  auto act = [&](const float* q) { return bf ? b16(q) : V(q); };
  // site whose mask the gradient of the residual stream must pass through right below the head / final norm
  // The last FC layer's dropout mask (and its bias gradient) is folded into the kernel that emits the gradient of the
  // FC output -- unless the FC block has an activation: then act_backward below does both.
  const bool fc_act = c.fc_act != ARB_ACT_NONE;
  const DropSite none_site{0u, 0u, 1.0f};
  const DropSite fc_site = make_drop_site(seed, L.n_fc - 1, SITE_FC, p_fc);
  float* const fc_bias_grad = fc_act ? nullptr : g(L.fc_b[L.n_fc - 1]);
  const DropSite top_site = c.n_layers > 0 ? make_drop_site(seed, c.n_layers - 1, SITE_FFN_OUT, p_drop)
                                           : (fc_act ? none_site : fc_site);

  // rows at or beyond this extent are masked keys with a zero score gradient: their gradients stay exactly zero in
  // every layer, which lets the fused attention backward skip their tiles
  int* gext = reinterpret_cast<int*>(scratch + Z.ext);
  const bool skip = g_skip_padding && c.n_layers > 0 && use_fused_bwd(c, S);
  // Packed rows: the forward call left the plan in the workspace (row count, row map, slate offsets, packed features,
  // key extents); the items it dropped have the constant score 0, so their score gradient is not read.
  const bool pack = use_pack(c, S);
  const int* plan = pack ? reinterpret_cast<const int*>(ws + W.plan) : nullptr;
  const int* rowmap = pack ? reinterpret_cast<const int*>(ws + W.rowmap) : nullptr;
  const int* poff = pack ? reinterpret_cast<const int*>(ws + W.poff) : nullptr;
  if (pack) { k.rows_dev = plan; k.R = buffer_rows(c, B, S); x = ws + W.xc; gext = reinterpret_cast<int*>(ws + W.kext); }
  else if (skip) ARB_TRY(slate_extents(mask, dhidden ? dhidden : dscores, dhidden ? d : n_outputs(c), B, S, gext, st));
  auto hview = [&](V v, int64_t pitch) { return pack ? head_view(v, dk, int(k.R), h, 1, pitch) : head_view(v, dk, S, h, B, pitch); };
  if (pack) {
    // 256 finite rows of d ctx behind the packed rows (the attention backward's boxes overrun the last slates), and
    // zero dQ | dK | dV in the alignment rows no slate writes (the QKV weight gradient sums over them): both buffers
    // are shared by all layers and nothing else writes those rows -- once per call
    ZeroRegions z;
    z.add(dctx, d, d, 0, 256);
    z.add(dqkv, bf ? 3 * d / 2 : 3 * d, bf ? 3 * d / 2 : 3 * d, 1, 0);
    ARB_TRY(zero_rows(z, plan, k.R, st));
  }
  const int has_norm = c.n_layers > 0;
  const float* xlast = c.n_layers > 0 ? ws + W.layer[c.n_layers - 1].xout : ws + W.x0;
  float* top_bias_grad = c.n_layers > 0 ? g(L.layer[c.n_layers - 1].b2) : fc_bias_grad;
  const float* dy = top_site.thresh ? dxm : dx;   // gradient w.r.t. the output of the linear below the dropout
  if (dhidden) {
    if (has_norm) {   // the final norm's backward from the given gradient (packed rows: read at the items' places)
      ARB_TRY(ln_backward(dhidden, xlast, P + L.lnf_a, ws + W.meanf, ws + W.stdf, c.ln_eps, nullptr, k.R, d, dx,
                          g(L.lnf_a), g(L.lnf_b), st, dxm, top_site, top_bias_grad, 0, nullptr, dy16, plan, rowmap));
    } else if (!fc_act) {   // FC-only model: d hidden through the FC dropout; the FC bias gradient is its column sums
      if (fc_site.thresh || fc_bias_grad)
        ARB_TRY(act_backward(dhidden, ws + W.x0, dx, k.R, d, ARB_ACT_NONE, fc_site, 1.0f, fc_bias_grad, st));
      dy = (fc_site.thresh || fc_bias_grad) ? dx : dhidden;
    }   // (FC-only with an activation: act_backward below reads dhidden)
  } else if (n_outputs(c) > 1) {
    if (has_norm) {   // d xf into dxn, then the final norm's backward emits dx (+ its masked copy and the b2 gradient)
      ARB_TRY(head_multi_backward(dscores, scores, ws + W.xf, P + L.head_w, c.out_act, k.R, d, n_outputs(c), dxn,
                                  g(L.head_w), g(L.head_b), st));
      ARB_TRY(ln_backward(dxn, xlast, P + L.lnf_a, ws + W.meanf, ws + W.stdf, c.ln_eps, nullptr, k.R, d, dx,
                          g(L.lnf_a), g(L.lnf_b), st, dxm, top_site, top_bias_grad, 0, nullptr, dy16));
    } else {
      ARB_TRY(head_multi_backward(dscores, scores, xlast, P + L.head_w, c.out_act, k.R, d, n_outputs(c), dx,
                                  g(L.head_w), g(L.head_b), st, dxm, top_site, top_bias_grad));
    }
  } else {
    ARB_TRY(head_backward(dscores, scores, xlast, has_norm ? P + L.lnf_a : nullptr, has_norm ? P + L.lnf_b : nullptr,
                          ws + W.meanf, ws + W.stdf, c.ln_eps, P + L.head_w, P + L.head_b, has_norm, c.out_act, k.R, d,
                          dx, has_norm ? g(L.lnf_a) : nullptr, has_norm ? g(L.lnf_b) : nullptr, g(L.head_w),
                          g(L.head_b), st, dxm, top_site, top_bias_grad, dy16, plan, rowmap));
  }
  for (int l = c.n_layers - 1; l >= 0; --l) {
    const auto& pl = L.layer[l];
    const auto& wl = W.layer[l];
    const float* xin = (l == 0) ? ws + W.x0 : ws + W.layer[l - 1].xout;
    float* xn1 = ws + wl.xn1; float* qkv = ws + wl.qkv; float* ctx = ws + wl.ctx;
    float* prob = W.fused ? scratch + Z.prob : ws + wl.prob;
    float* xmid = ws + wl.xmid; float* xn2 = ws + wl.xn2; float* hdn = ws + wl.hdn;
    // ---- feed-forward sublayer backward:  xout = xmid + W2 relu(W1 xn2 + b1) + b2
    const V dyv = bf ? b16(dy16) : V(dy);      // what the sublayer's products read as the incoming gradient
    if (G) ARB_TRY(linear_bwd_weight(k, dyv, d, d, act(hdn), f, f, G + pl.w2));   // (b2 gradient: fused into the kernel that emitted dy)
    // hdn <- d hdn in place; hdn > 0 <=> ReLU active AND kept by the hidden dropout, so the mask tile also carries
    // the dropout mask and only the 1/(1-p) scale is needed
    if (wl.hbits)    // ReLU mask from the forward's bit mask (1 bit per unit) instead of the fp32 activation tile
      ARB_TRY(linear_bwd_input(k, dyv, d, d, wt(pl.w2), f, act(hdn), f, EPI_COLSUM, nullptr, 0, 1.0f, g(pl.b1),
                               reinterpret_cast<const uint32_t*>(ws + wl.hbits)));
    else
    ARB_TRY(linear_bwd_input(k, dyv, d, d, wt(pl.w2), f, act(hdn), f, EPI_MASK_AUX | EPI_COLSUM, act(hdn), f,
                             drop_on ? 1.0f / (1.0f - p_drop) : 1.0f, g(pl.b1)));   // b1 gradient in the epilogue
    if (G) ARB_TRY(linear_bwd_weight(k, act(hdn), f, f, act(xn2), d, d, G + pl.w1));
    ARB_TRY(linear_bwd_input(k, act(hdn), f, f, wt(pl.w1), d, act(dxn), d, 0, nullptr, 0));
    const DropSite site_ao = make_drop_site(seed, l, SITE_ATTN_OUT, p_drop);
    ARB_TRY(ln_backward(dxn, xmid, P + pl.ln2_a, ws + wl.mean2, ws + wl.std2, c.ln_eps, dx, k.R, d, dx_alt,
                        g(pl.ln2_a), g(pl.ln2_b), st, dxm, site_ao, g(pl.bo), 0, bf ? dxn : nullptr, dy16, plan));
    // dx_alt = d loss / d xmid ; dy = the same through the dropout on the attention sublayer output
    dy = site_ao.thresh ? dxm : dx_alt;
    // ---- attention sublayer backward:  xmid = xin + Wo ctx + bo
    const V dyo = bf ? b16(dy16) : V(dy);
    if (G) ARB_TRY(linear_bwd_weight(k, dyo, d, d, act(ctx), d, d, G + pl.wo));   // (bo gradient: fused into the LayerNorm backward above)
    ARB_TRY(linear_bwd_input(k, dyo, d, d, wt(pl.wo), d, dctx, d, 0, nullptr, 0));
    if (use_fused_bwd(c, S)) {
      AttnBwdArgs a;   // dQ, dK, dV from d ctx in one kernel; P is recomputed from the saved row statistics
      a.q = hview(qkv, 3 * d);
      a.k = hview(qkv + d, 3 * d);
      a.v = hview(qkv + 2 * d, 3 * d);
      a.d_o = hview(dctx, d);
      if (bf) {   // dQ | dK | dV as one packed bfloat16 [R, 3d] buffer
        uint16_t* g16 = reinterpret_cast<uint16_t*>(dqkv);
        a.dq = hview(b16(g16), 3 * d);
        a.dk_ = hview(b16(g16 + d), 3 * d);
        a.dv = hview(b16(g16 + 2 * d), 3 * d);
      } else {
        a.dq = hview(dqkv, 3 * d);
        a.dk_ = hview(dqkv + d, 3 * d);
        a.dv = hview(dqkv + 2 * d, 3 * d);
      }
      a.pack_off = poff; a.rows_dev = plan; a.rowmap = rowmap;
      a.o_ptr = ctx; a.o_bf16 = bf ? 1 : 0; a.do_ptr = dctx; a.o_pitch = d;
      a.mask = mask; a.stat_max = ws + wl.smax; a.stat_sum = ws + wl.ssum; a.delta = scratch + Z.delta;
      a.B = B; a.h = h; a.S = S; a.dk = dk; a.scale = alpha;
      a.drop = make_drop_site(seed, l, SITE_ATTN_P, p_drop);
      a.dbias_qkv = g(pl.bqkv); a.d_model = d;           // bias gradient of the QKV projection, fused
      a.extent = (skip || pack) ? gext : nullptr;
      ARB_TRY(launch_attn_bwd(a, st));
    } else {
      const DropSite site_p = make_drop_site(seed, l, SITE_ATTN_P, p_drop);
      if (W.fused || site_p.thresh) {
        // no undropped probabilities were kept (the fused forward keeps none; under dropout the unfused forward kept
        // the dropped ones): recompute P = softmax(mask(alpha Q K^T))
        GemmDesc g;
        g.M = S; g.N = S; g.K = dk; g.alpha = alpha;
        g.A = head_view(qkv, dk, S, h, B, 3 * d);
        g.B = head_view(qkv + d, dk, S, h, B, 3 * d);
        g.C = prob_view(prob, S, W.Sp, h, B);
        batch_all(g, h, B); g.block_n = 64;
        ARB_TRY(launch_gemm_tf32(g, st));
        ARB_TRY(softmax_forward(prob, mask, B, h, S, W.Sp, st));
      }
      {
        GemmDesc g;   // dP~ = dctx V^T   (gradient w.r.t. the dropped probabilities)
        g.M = S; g.N = S; g.K = dk;
        g.A = head_view(dctx, dk, S, h, B, d);
        g.B = head_view(qkv + 2 * d, dk, S, h, B, 3 * d);
        g.C = prob_view(dprob, S, W.Sp, h, B);
        batch_all(g, h, B); g.block_n = 64;
        ARB_TRY(launch_gemm_tf32(g, st));
      }
      // dprob <- dS (pre-scale); under dropout the mask is regenerated and prob <- dropped probabilities
      ARB_TRY(softmax_backward(dprob, prob, int64_t(B) * h * S, S, W.Sp, st, site_p));
      {
        GemmDesc g;   // dV = P~^T dctx     (P~ read as an MN-major A operand, dctx as an MN-major B operand)
        g.M = S; g.N = dk; g.K = S; g.a_mn = 1; g.b_mn = 1;
        g.A = prob_view(prob, S, W.Sp, h, B);
        g.B = head_view(dctx, dk, S, h, B, d);
        g.C = head_view(dqkv + 2 * d, dk, S, h, B, 3 * d);
        batch_all(g, h, B); g.block_n = pick_block_n(dk);
        ARB_TRY(launch_gemm_tf32(g, st));
      }
      {
        GemmDesc g;   // dQ = alpha dS K
        g.M = S; g.N = dk; g.K = S; g.b_mn = 1; g.alpha = alpha;
        g.A = prob_view(dprob, S, W.Sp, h, B);
        g.B = head_view(qkv + d, dk, S, h, B, 3 * d);
        g.C = head_view(dqkv, dk, S, h, B, 3 * d);
        batch_all(g, h, B); g.block_n = pick_block_n(dk);
        ARB_TRY(launch_gemm_tf32(g, st));
      }
      {
        GemmDesc g;   // dK = alpha dS^T Q
        g.M = S; g.N = dk; g.K = S; g.a_mn = 1; g.b_mn = 1; g.alpha = alpha;
        g.A = prob_view(dprob, S, W.Sp, h, B);
        g.B = head_view(qkv, dk, S, h, B, 3 * d);
        g.C = head_view(dqkv + d, dk, S, h, B, 3 * d);
        batch_all(g, h, B); g.block_n = pick_block_n(dk);
        ARB_TRY(launch_gemm_tf32(g, st));
      }
    }
    if (G) ARB_TRY(linear_bwd_weight(k, act(dqkv), 3 * d, 3 * d, act(xn1), d, d, G + pl.wqkv));
    if (G && !use_fused_bwd(c, S)) ARB_TRY(colsum_accumulate(dqkv, k.R, 3 * d, 3 * d, G + pl.bqkv, st));
    ARB_TRY(linear_bwd_input(k, act(dqkv), 3 * d, 3 * d, wt(pl.wqkv), d, act(dxn), d, 0, nullptr, 0));
    DropSite site_below = l > 0 ? make_drop_site(seed, l - 1, SITE_FFN_OUT, p_drop) : (fc_act ? none_site : fc_site);
    // with a positional encoding the encoder input is sqrt(d) * fc_out + pe: the gradient that reaches the FC
    // (through its dropout mask, if any) carries the extra sqrt(d)
    if (l == 0 && c.pe_mode != 0 && !fc_act) site_below.scale *= sqrtf(float(d));
    ARB_TRY(ln_backward(dxn, xin, P + pl.ln1_a, ws + wl.mean1, ws + wl.std1, c.ln_eps, dx_alt, k.R, d, dx,
                        g(pl.ln1_a), g(pl.ln1_b), st, dxm, site_below, l > 0 ? g(L.layer[l - 1].b2) : fc_bias_grad,
                        0, bf ? dxn : nullptr, l > 0 ? dy16 : nullptr, plan));   // (the FC block below layer 0 stays TF32)
    // dx = d loss / d xin ; dy = the same through the dropout that produced xin's last summand
    dy = (site_below.thresh || site_below.scale != 1.0f) ? dxm : dx;
  }
  if (c.pe_mode == 2 && G) {   // learned table: d pe[idx] += d x0
    if (!indices) { arb_set_error("scorer: positional encoding needs indices"); return ARB_E_INVALID_ARG; }
    ARB_TRY(pos_backward(dx, reinterpret_cast<const long long*>(indices), mask, G + L.pe, c.pe_rows, k.R, d, st));
  }
  // ---- FC-block backward (model.py:35-44), last layer first.  dz = gradient w.r.t. the linear's output.
  const float* dz = dy;            // identity activation: mask + bias gradient were fused into the kernel that emitted dy
  float* dfa = scratch + Z.dfa;
  float* dfb = scratch + Z.dfb;
  if (fc_act) {
    const float* h_last = W.fc_last ? ws + W.fc_last : ws + W.x0;
    const float* dh = (dhidden && c.n_layers == 0) ? dhidden : dx;   // d loss / d (activated FC output)
    ARB_TRY(act_backward(dh, h_last, dfa, k.R, d, c.fc_act, fc_site, c.pe_mode != 0 ? sqrtf(float(d)) : 1.0f,
                         g(L.fc_b[L.n_fc - 1]), st, plan));
    dz = dfa; std::swap(dfa, dfb);
  }
  for (int i = L.n_fc - 1; i >= 0; --i) {
    const int out = L.fc_size[i];
    const int in = i > 0 ? L.fc_size[i - 1] : F;
    const float* hin = i > 0 ? ws + W.fch[i - 1] : (c.fc_input_norm ? ws + W.xnorm : x);
    if (G) ARB_TRY(linear_bwd_weight(k, dz, out, out, hin, in, in, G + L.fc_w[i]));
    if (i > 0) {
      const DropSite site = make_drop_site(seed, i - 1, SITE_FC, p_fc);
      if (c.fc_act == ARB_ACT_RELU) {        // h > 0 <=> ReLU active and kept by the dropout: mask tile + 1/(1-p)
        ARB_TRY(linear_bwd_input(k, dz, out, out, P + L.fc_w[i], in, dfa, in, EPI_MASK_AUX | EPI_COLSUM, hin, in,
                                 site.scale, g(L.fc_b[i - 1])));
      } else if (c.fc_act == ARB_ACT_NONE && site.thresh == 0) {
        ARB_TRY(linear_bwd_input(k, dz, out, out, P + L.fc_w[i], in, dfa, in, EPI_COLSUM, nullptr, 0, 1.0f, g(L.fc_b[i - 1])));
      } else {
        ARB_TRY(linear_bwd_input(k, dz, out, out, P + L.fc_w[i], in, dfa, in, 0, nullptr, 0));
        ARB_TRY(act_backward(dfa, hin, dfa, k.R, in, c.fc_act, site, 1.0f, g(L.fc_b[i - 1]), st, plan));
      }
      dz = dfa; std::swap(dfa, dfb);
      continue;
    }
    // the first layer's input: d loss / d x goes to dX (dense rows) or to a packed buffer scattered into dX below
    float* const dxin = dX ? (pack ? scratch + Z.dxin : dX) : nullptr;
    if (c.fc_input_norm && (G || dX)) {      // the LayerNorm's backward emits d x (kept only when asked for)
      ARB_TRY(linear_bwd_input(k, dz, out, out, P + L.fc_w[0], in, dfa, in, 0, nullptr, 0));
      ARB_TRY(ln_backward(dfa, x, P + L.in_a, ws + W.in_mean, ws + W.in_std, 0.0f, nullptr, k.R, F, dxin ? dxin : dfb,
                          g(L.in_a), g(L.in_b), st, nullptr, none_site, nullptr, 1, nullptr, nullptr, plan));
    } else if (dX) {                         // dX = dZ0 W0
      ARB_TRY(linear_bwd_input(k, dz, out, out, P + L.fc_w[0], in, dxin, in, 0, nullptr, 0));
    }
  }
  if (dX && pack) {   // items beyond their slate's packed rows get 0, like their score
    if (cudaMemsetAsync(dX, 0, size_t(B) * S * F * sizeof(float), st) != cudaSuccess) { arb_set_error("scorer: memset failed"); return ARB_E_CUDA; }
    ARB_TRY(scatter_rows(scratch + Z.dxin, plan, rowmap, k.R, F, dX, st));
  }
  return ARB_OK;
}

}  // namespace arb

using namespace arb;

extern "C" void arb_set_attention_mode(int32_t mode) { g_attn_mode = mode; }
extern "C" void arb_set_attention_skip_padding(int32_t on) { g_skip_padding = on; }
extern "C" void arb_set_attention_bwd_persistent(int32_t on) { set_attn_bwd_persistent(on); }
extern "C" void arb_set_relu_bits(int32_t on) { g_relu_bits = on; }
extern "C" int32_t arb_get_relu_bits(void) { return g_relu_bits; }
extern "C" void arb_set_pack_rows(int32_t on) { g_pack_rows = on; }
extern "C" int32_t arb_get_pack_rows(void) { return g_pack_rows; }
extern "C" void arb_set_attention_fwd_two_pass(int32_t on) { set_attn_fwd_two_pass(on); }

extern "C" int64_t arb_scorer_param_count(const arb_scorer_config* cfg) {
  ParamLayout L;
  if (!cfg || make_param_layout(*cfg, L) != ARB_OK) return -1;
  return L.total;
}
extern "C" int64_t arb_scorer_workspace_floats(const arb_scorer_config* cfg, int32_t B, int32_t S, int32_t training) {
  ParamLayout L;
  if (!cfg || B <= 0 || S <= 0 || make_param_layout(*cfg, L) != ARB_OK) return -1;
  WsLayout W;
  make_ws_layout(*cfg, L, B, S, training, W);
  return W.total;
}
extern "C" int64_t arb_scorer_backward_scratch_floats(const arb_scorer_config* cfg, int32_t B, int32_t S) {
  ParamLayout L;
  if (!cfg || B <= 0 || S <= 0 || make_param_layout(*cfg, L) != ARB_OK) return -1;
  ScratchLayout Z;
  make_scratch_layout(*cfg, L, B, S, Z);
  return Z.total;
}
extern "C" int64_t arb_scorer_backward_ex_scratch_floats(const arb_scorer_config* cfg, int32_t B, int32_t S,
                                                         int32_t want_dx) {
  ParamLayout L;
  if (!cfg || B <= 0 || S <= 0 || make_param_layout(*cfg, L) != ARB_OK) return -1;
  ScratchLayout Z;
  make_scratch_layout(*cfg, L, B, S, Z, want_dx != 0);
  return Z.total;
}
extern "C" int32_t arb_scorer_forward(const arb_scorer_config* cfg, const float* params, const float* x,
                                      const uint8_t* mask, const int64_t* indices, const float* pe_table, int32_t B,
                                      int32_t S, float* scores, float* workspace, int64_t workspace_floats,
                                      int32_t training, uint64_t seed, void* stream) {
  if (!cfg || !params || !x || !mask || !scores || !workspace || B <= 0 || S <= 0) {
    arb_set_error("arb_scorer_forward: null pointer or bad shape");
    return ARB_E_INVALID_ARG;
  }
  return forward_impl(*cfg, params, x, mask, indices, pe_table, B, S, scores, nullptr, workspace, workspace_floats,
                      training, seed, static_cast<cudaStream_t>(stream));
}
extern "C" int32_t arb_scorer_encode(const arb_scorer_config* cfg, const float* params, const float* x,
                                     const uint8_t* mask, const int64_t* indices, const float* pe_table, int32_t B,
                                     int32_t S, float* hidden, float* workspace, int64_t workspace_floats,
                                     int32_t training, uint64_t seed, void* stream) {
  if (!cfg || !params || !x || !mask || !hidden || !workspace || B <= 0 || S <= 0) {
    arb_set_error("arb_scorer_encode: null pointer or bad shape");
    return ARB_E_INVALID_ARG;
  }
  return forward_impl(*cfg, params, x, mask, indices, pe_table, B, S, nullptr, hidden, workspace, workspace_floats,
                      training, seed, static_cast<cudaStream_t>(stream));
}
extern "C" int32_t arb_scorer_backward(const arb_scorer_config* cfg, const float* params, const float* x,
                                       const uint8_t* mask, const int64_t* indices, int32_t B, int32_t S,
                                       const float* scores,
                                       const float* d_scores, float* grads, float* workspace, int64_t workspace_floats,
                                       float* scratch, int64_t scratch_floats, uint64_t seed, void* stream) {
  if (!cfg || !params || !x || !mask || !scores || !d_scores || !grads || !workspace || !scratch || B <= 0 || S <= 0) {
    arb_set_error("arb_scorer_backward: null pointer or bad shape");
    return ARB_E_INVALID_ARG;
  }
  return backward_impl(*cfg, params, x, mask, indices, B, S, scores, d_scores, nullptr, grads, nullptr, workspace,
                       workspace_floats, scratch, scratch_floats, seed, static_cast<cudaStream_t>(stream));
}
extern "C" int32_t arb_scorer_backward_ex(const arb_scorer_config* cfg, const float* params, const float* x,
                                          const uint8_t* mask, const int64_t* indices, int32_t B, int32_t S,
                                          const float* scores, const float* d_scores, const float* d_hidden,
                                          float* grads, float* d_x, float* workspace, int64_t workspace_floats,
                                          float* scratch, int64_t scratch_floats, uint64_t seed, void* stream) {
  if (!cfg || !params || !x || !mask || !workspace || !scratch || B <= 0 || S <= 0 || (!d_scores == !d_hidden) ||
      (d_scores && !scores)) {
    arb_set_error("arb_scorer_backward_ex: null pointer, bad shape, or not exactly one of d_scores / d_hidden");
    return ARB_E_INVALID_ARG;
  }
  return backward_impl(*cfg, params, x, mask, indices, B, S, scores, d_scores, d_hidden, grads, d_x, workspace,
                       workspace_floats, scratch, scratch_floats, seed, static_cast<cudaStream_t>(stream));
}
