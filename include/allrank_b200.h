/* allrank_b200 -- C ABI of the H100 (sm_90a) scoring + listwise-loss + metric path.
 *
 * This is the drop-in boundary (DESIGN.md section 2).  allRank is pure Python, so there is no
 * existing FFI to mirror; each entry point below replaces one *Python call surface* of the
 * reference and cites it.  The Python host layer (allrank_b200/{losses,metrics,model}.py) binds
 * these with ctypes and re-exports the reference's names/signatures; INTEGRATION.md shows the
 * stub a maintainer adds on the allRank side.
 *
 * Conventions
 *   - plain pointers + sizes only; no torch types.  All pointers are DEVICE pointers unless the
 *     parameter name ends in `_host`.  Tensors are row-major, contiguous, fp32 unless stated.
 *   - outputs and workspaces are caller-owned (the host layer allocates them with PyTorch's caching allocator).
 *     The one allocation the library makes is stream-ordered scratch for its gradient reductions: a call that sums
 *     partial results across blocks takes per-block slots with cudaMallocAsync on `stream`, adds them in a fixed
 *     order (so gradients are bitwise reproducible) and releases them with cudaFreeAsync on the same stream before it
 *     returns.  Calls on different streams never share slots; under stream capture the slots become memory nodes
 *     owned by the graph.  No device memory is held between calls.
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*; NULL = legacy default
 *     stream) of the CURRENT device and returns without synchronising; calls are re-entrant.
 *   - return value: 0 = ok, <0 = ARB_E_* below; arb_last_error() gives a thread-local message.
 *   - inputs are const: the caller's y_pred / y_true / x / mask are never modified
 *     (the reference clones before masking: listNet.py:17-18, lambdaLoss.py:25-26, metrics.py:53-54).
 */
#ifndef ALLRANK_B200_H
#define ALLRANK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ARB_OK 0
#define ARB_E_INVALID_ARG (-1)
#define ARB_E_UNSUPPORTED (-2)
#define ARB_E_CUDA (-3)
#define ARB_E_WORKSPACE (-4)

#define ARB_MAX_ATS 32

/* lambdaLoss weighing schemes: allrank/models/losses/lambdaLoss.py:84-114 (selected by name at :61) */
#define ARB_SCHEME_NONE 0
#define ARB_SCHEME_NDCGLOSS1 1
#define ARB_SCHEME_NDCGLOSS2 2
#define ARB_SCHEME_LAMBDARANK 3
#define ARB_SCHEME_NDCGLOSS2PP 4
#define ARB_SCHEME_RANKNET 5
#define ARB_SCHEME_RANKNET_GTDIFF 6
#define ARB_SCHEME_RANKNET_GTDIFF_POWED 7

#define ARB_REDUCTION_SUM 0
#define ARB_REDUCTION_MEAN 1
#define ARB_LOG_BINARY 0
#define ARB_LOG_NATURAL 1

#define ARB_GAIN_POW2 0     /* 2^x - 1 : default gain_function of metrics.dcg (metrics.py:41)          */
#define ARB_GAIN_IDENTITY 1 /* x       : what neuralNDCG passes when powered_relevancies=False (:58)   */

const char* arb_last_error(void);
/* 4 (round 2): packed rows (arb_set_pack_rows / arb_get_pack_rows; the scorer workspace layout depends on the call's
 * dropout rates), arb_set_attention_bwd_persistent; 3: general FC block, bf16 mode */
int32_t arb_abi_version(void);
/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
int64_t arb_launch_count(void);

/* ---------------------------------------------------------------- metrics
 * Replaces allrank.models.metrics.{dcg,ndcg,mrr} (allrank/models/metrics.py:41-77, :7-28, :80-113),
 * called from train_utils.metric_on_batch (allrank/training/train_utils.py:32-34).
 * One launch computes any subset of the outputs (NULL pointer = not wanted):
 *   out_dcg   [B,n_ats]  DCG@at of labels ranked by y_pred          (ats_dcg_host: already min(at,S))
 *   out_idcg  [B,n_ats]  DCG@at of labels ranked by themselves
 *   out_ndcg  [B,n_ats]  out_dcg/out_idcg, `filler` where out_idcg == 0
 *   out_mrr   [B,n_ats]  reciprocal rank of the first max-label item if rank < at (ats_mrr_host, unclipped);
 *                        all zeros if the batch-wide sum of per-slate max labels is 0 (metrics.py:108-109)
 *   out_order [B,S] i32  the descending argsort of the masked scores (stable; bit-exact on tie-free input)
 * `discounts` is the [S] fp32 table 1/log2(j+2) that the reference evaluates on the HOST (metrics.py:64);
 * the host layer builds it the same way so DCG values can match bit for bit.
 * `mrr_scratch` : >= 2*B floats. */
int32_t arb_rank_metrics(const float* y_pred, const float* y_true, int32_t B, int32_t S,
                         const float* discounts, const int32_t* ats_dcg_host, const int32_t* ats_mrr_host,
                         int32_t n_ats, int32_t gain_mode, float pad_value, float filler,
                         float* out_dcg, float* out_idcg, float* out_ndcg, float* out_mrr, int32_t* out_order,
                         float* mrr_scratch, void* stream);

/* ---------------------------------------------------------------- losses (forward + backward in one launch)
 * Each replaces `loss_func(y_pred, y_true)` at allrank/training/train_utils.py:20 for one member of
 * allrank.models.losses.  `loss` is a device scalar; `grad` ([B,S], may be NULL for eval) receives
 * d loss / d y_pred.  `scratch` : >= 2*B floats. */

/* listNet(y_pred, y_true, eps, padded_value_indicator)            allrank/models/losses/listNet.py:8-30 */
int32_t arb_listnet(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps, float pad_value,
                    float* loss, float* grad, float* scratch, void* stream);

/* listMLE(...)                                                    allrank/models/losses/listMLE.py:7-38
 * `perm` [S] i64: the column shuffle the reference draws with torch.randperm (:17) -- drawn by the host
 * layer from the same global CPU RNG.  `order` (nullable [B,S] i32): debug hook feeding a realised sort
 * order of the shuffled labels (SURVEY.md 8c L1); NULL = stable descending sort on the device. */
int32_t arb_listmle(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps, float pad_value,
                    const int64_t* perm, const int32_t* order, float* loss, float* grad, float* scratch,
                    void* stream);

/* approxNDCGLoss(y_pred, y_true, eps, padded_value_indicator, alpha)   .../losses/approxNDCG.py:7-53 */
int32_t arb_approx_ndcg(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps,
                        float pad_value, float alpha, float* loss, float* grad, float* scratch, void* stream);

/* lambdaLoss(y_pred, y_true, eps, pad, weighing_scheme, k, sigma, mu, reduction, reduction_log)
 *                                                                  .../losses/lambdaLoss.py:7-114
 * k <= 0 means "None" (no truncation). */
int32_t arb_lambda_loss(const float* y_pred, const float* y_true, int32_t B, int32_t S, float eps,
                        float pad_value, int32_t scheme, int32_t k, float sigma, float mu, int32_t reduction,
                        int32_t log_base, float* loss, float* grad, float* scratch, void* stream);

/* --- SURVEY.md 8(f) rank-1 "next" losses, built on the same machinery ---
 * rankNet / rankNet_weightByGTDiff / rankNet_weightByGTDiff_pow            .../losses/rankNet.py:9-79
 * weight_mode 0: unweighted, 1: |t_i - t_j|, 2: |t_i^2 - t_j^2|; mean over all selected pairs of the batch. */
int32_t arb_ranknet(const float* y_pred, const float* y_true, int32_t B, int32_t S, float pad_value,
                    int32_t weight_mode, float* loss, float* grad, float* scratch, void* stream);
/* mode 0: binary_listNet(eps)            .../losses/binary_listNet.py:8-33
 * mode 1: pointwise_rmse(no_of_levels = param)   .../losses/pointwise.py:6-32
 * mode 2: bce (y_pred are probabilities)          .../losses/bce.py:8-32
 * Any slate length: one warp streams each slate and uses no shared memory.  The other losses are bounded by the
 * shared memory of one CTA: neuralNDCG serves S <= 4096 exactly, lambdaLoss about 5570, approxNDCG (and
 * arb_rank_metrics) about 6680, listMLE 8192, listNet and rankNet about 29 000, ordinal any length; a longer slate
 * returns ARB_E_UNSUPPORTED without a launch. */
int32_t arb_pointwise_loss(const float* y_pred, const float* y_true, int32_t B, int32_t S, float pad_value,
                           int32_t mode, float param, float eps, float* loss, float* grad, float* scratch,
                           void* stream);

/* ordinal(y_pred, y_true, n, pad)                                          .../losses/ordinal.py:8-50
 * y_pred [B,S,n] are probabilities (the scorer's d_output = n, Sigmoid head); target level j of an item with
 * label t is 1[t >= j+1] (with_ordinals, :8-22).  loss = sum of the n*valid BCE terms / number of valid items. */
int32_t arb_ordinal(const float* y_pred, const float* y_true, int32_t B, int32_t S, int32_t n, float pad_value,
                    float* loss, float* grad, float* scratch, void* stream);

/* neuralNDCG(y_pred, y_true, pad, temperature, powered_relevancies, k, stochastic=False)
 *                            .../losses/neuralNDCG.py:10-70 + loss_utils.py:8-67 (NeuralSort, Sinkhorn)
 * max_iter / tol are the Sinkhorn parameters the reference hard-codes to 50 / 1e-6 (neuralNDCG.py:41-42).
 * `discounts`: the same host-evaluated [S] table 1/log2(j+2) as arb_rank_metrics (neuralNDCG.py:52).
 * `workspace`: arb_neural_ndcg_workspace_bytes(B,S,max_iter) bytes (0 when every slate fits in shared memory). */
size_t arb_neural_ndcg_workspace_bytes(int32_t B, int32_t S, int32_t max_iter);
int32_t arb_neural_ndcg(const float* y_pred, const float* y_true, int32_t B, int32_t S,
                        const float* discounts, float pad_value, float temperature, int32_t powered_relevancies, int32_t k, int32_t max_iter, float tol,
                        float* loss, float* grad, float* scratch, void* workspace, size_t workspace_bytes,
                        void* stream);

/* Parity hook for deterministic_neural_sort / sinkhorn_scaling (allrank/models/losses/loss_utils.py:34-67, :8-31), which
 * arb_neural_ndcg fuses: the kernel's own matrices for slates of at most 128 items.  p0_out, p_out: zero-filled
 * [B,S,S] buffers; entries [b, rank j, item i] of the real items receive NeuralSort's P_hat and its Sinkhorn scaling
 * (max_iter iterations at most, per-slate tolerance test).  Slates without a relevant item are left untouched.
 * scratch: >= 2*B floats. */
int32_t arb_neural_sort_debug(const float* y_pred, const float* y_true, int32_t B, int32_t S, const float* discounts,
                              float pad_value, float temperature, int32_t max_iter, float tol, float* p0_out,
                              float* p_out, float* scratch, void* stream);

/* ---------------------------------------------------------------- scorer: LTRModel(x, mask, indices) -> scores
 * Replaces allrank.models.model.LTRModel.forward / .score (allrank/models/model.py:72-92) for the model family
 * make_model builds (model.py:131-151): one input Linear (FCModel, model.py:12-44) -> N pre-norm Transformer
 * encoder blocks (allrank/models/transformer.py:28-227: custom LayerNorm, MultiHeadedAttention with key-padding
 * mask, PositionwiseFeedForward, residuals) -> final LayerNorm -> Linear(d_model -> 1) head (model.py:95-128).
 * Called from allrank/training/train_utils.py:20 (`model(xb, mask, indices)`) and :34 (`model.score`).
 *
 * Every matrix product runs on the tensor cores in TF32 with fp32 accumulation (csrc/gemm_tf32.cu);
 * LayerNorm / softmax / head are fp32 SIMT kernels (csrc/scorer_kernels.cu).  Dropout masks are a counter-based
 * hash of (seed, layer, site, element index) fused into the producing kernels and regenerated in backward
 * (csrc/dropout.cuh); `seed` must be the same in the forward and the backward call of a step.
 *
 *  Parameters live in ONE flat fp32 buffer (the host layer makes the nn.Parameters views of it), laid out as
 *   per FC layer i: fc_w[s_i, s_{i-1}] fc_b[s_i] (s_{-1} = F) | in_norm_w[F] in_norm_b[F] if fc_input_norm |
 *   (pad to a multiple of 8 elements) | per layer: wq wk wv [3d,d] bq bk bv [3d] wo[d,d] bo[d] w1[dff,d] b1[dff] w2[d,dff] b2[d]
 *   ln1_a ln1_b ln2_a ln2_b [d each] | lnf_a lnf_b [d] head_w[d] head_b[1] (pad to 4) | pe[pe_rows,d] if pe_mode == 2
 * (a fixed sinusoidal table, pe_mode == 1, is a buffer, not a parameter: it is passed separately as `pe_table`)
 * arb_scorer_param_count() gives the total; gradients use the same layout and are ACCUMULATED into `grads`.
 */
#define ARB_ACT_NONE 0
#define ARB_ACT_TANH 1
#define ARB_ACT_SIGMOID 2
#define ARB_ACT_RELU 3

typedef struct arb_scorer_config {
  int32_t n_features;   /* F (row pitch of x; must be a multiple of 4 -- the host layer pads)            */
  int32_t d_model;      /* fc_model.sizes[-1] (model.py:142); multiple of 32 * n_heads                    */
  int32_t n_layers;     /* transformer N; 0 = FC-only model (no encoder, no final LayerNorm)              */
  int32_t n_heads;      /* h                                                                             */
  int32_t d_ff;         /* PositionwiseFeedForward hidden width                                           */
  int32_t out_act;      /* ARB_ACT_*: post_model.output_activation (model.py:105-107)                     */
  float ln_eps;         /* 1e-6 (transformer.py:63)                                                       */
  float dropout;        /* transformer.dropout: on attention probabilities, both sublayer outputs and the FFN
                           hidden layer (transformer.py:105,155,227); applied only when training != 0          */
  float fc_dropout;     /* fc_model.dropout on the input FC output (model.py:43)                          */
  int32_t pe_mode;      /* positional encoding (allrank/models/positional.py): 0 none, 1 fixed table, 2 learned     */
  int32_t pe_rows;      /* rows of the table = max_indices + 1; the last row is the padding row              */
  int32_t d_output;     /* post_model.d_output (model.py:104,108): outputs per item; 0 or 1 = one score per item.
                           > 1 (ordinal loss): scores are [B,S,d_output], head weight [d_output,d_model]           */
  /* --- ABI v3: the general FCModel input block (model.py:16-44): [nn.LayerNorm(F)] -> n x dropout(act(Linear)) */
  int32_t n_fc_layers;  /* len(fc_model.sizes), 1..ARB_MAX_FC_LAYERS; 0 = one layer of width d_model (v2 behaviour)  */
  int32_t fc_sizes[8];  /* fc_model.sizes (multiples of 4, <= 8192); fc_sizes[n_fc_layers-1] must equal d_model       */
  int32_t fc_act;       /* ARB_ACT_*: fc_model.activation applied after every FC linear, before its dropout          */
  int32_t fc_input_norm;/* fc_model.input_norm: nn.LayerNorm(n_features) (eps 1e-5, biased variance) on x first;
                           needs n_features % 4 == 0 (no feature padding)                                             */
  int32_t bf16;         /* 1: bf16 mode of the encoder (BASELINE config 3): every encoder linear runs as a tensor-core
                           product of bfloat16 operands with fp32 accumulation -- weights from a bfloat16
                           shadow of the fp32 master parameters (refreshed by every forward call), activations that only
                           feed products (LayerNorm outputs, attention context, FFN hidden layer) and the gradients that
                           only feed products stored as bfloat16; residual stream, LayerNorm statistics, softmax,
                           attention scores (TF32 products on fp32 Q/K/V), head, loss and parameter gradients stay fp32.
                           Needs the fused attention kernels (slate_length <= 256), head width 8, 16, 24 or 32
                           (a bfloat16 head of w columns spans 2w bytes, which TMA needs to be a multiple of 16) and
                           d_model, d_ff multiples of 8.  0: TF32 products on fp32 data everywhere.                  */
} arb_scorer_config;
#define ARB_MAX_FC_LAYERS 8

int64_t arb_scorer_param_count(const arb_scorer_config* cfg);
/* floats of activation workspace for a [B,S] batch; `training` != 0 keeps what backward needs.  Query it with the
 * configuration of the call itself (the dropout rates in particular: a call without dropout may run over packed rows,
 * arb_set_pack_rows, whose buffers differ). */
int64_t arb_scorer_workspace_floats(const arb_scorer_config* cfg, int32_t B, int32_t S, int32_t training);
/* x [B,S,F] fp32, mask [B,S] uint8 (1 = padded, train_utils.py:19) -> scores [B,S] fp32.
 * indices [B,S] int64 (original item ranks, -1 = padded; positional.py:45-50) and pe_table are only read when
 * cfg->pe_mode != 0 (pe_table: the fixed table for mode 1; ignored for mode 2, whose table lives in params). */
int32_t arb_scorer_forward(const arb_scorer_config* cfg, const float* params, const float* x, const uint8_t* mask,
                           const int64_t* indices, const float* pe_table,
                           int32_t B, int32_t S, float* scores, float* workspace, int64_t workspace_floats,
                           int32_t training, uint64_t seed, void* stream);
/* d_scores [B,S] -> grads += d loss / d params.  `workspace` is the one the training forward filled;
 * `scratch`: arb_scorer_backward_scratch_floats(cfg,B,S) floats. */
int64_t arb_scorer_backward_scratch_floats(const arb_scorer_config* cfg, int32_t B, int32_t S);
int32_t arb_scorer_backward(const arb_scorer_config* cfg, const float* params, const float* x, const uint8_t* mask,
                            const int64_t* indices, int32_t B, int32_t S, const float* scores, const float* d_scores, float* grads,
                            float* workspace, int64_t workspace_floats, float* scratch, int64_t scratch_floats,
                            uint64_t seed, void* stream);

/* The encoder output (LTRModel.prepare_for_output, model.py:62-70): the arguments of arb_scorer_forward, but instead
 * of scores it writes hidden [B,S,d_model] fp32 -- the final LayerNorm's output, or with n_layers == 0 the FC block's
 * output after its activation and dropout (the reference's encoder is then the identity).  The head is not run.
 * training != 0 keeps the workspace for arb_scorer_backward_ex(d_hidden = ...), as the forward does.
 * Packed rows (arb_set_pack_rows): items at or beyond their slate's packed rows get a zero row, as they get the score 0. */
int32_t arb_scorer_encode(const arb_scorer_config* cfg, const float* params, const float* x, const uint8_t* mask,
                          const int64_t* indices, const float* pe_table,
                          int32_t B, int32_t S, float* hidden, float* workspace, int64_t workspace_floats,
                          int32_t training, uint64_t seed, void* stream);
/* The backward with a choice of starting point and outputs.  Exactly one of
 *   d_scores [B,S] (or [B,S,d_output]; after arb_scorer_forward, `scores` its output) and
 *   d_hidden [B,S,d_model] (after arb_scorer_encode; `scores` may be NULL)
 * is non-null.  grads: accumulated as by arb_scorer_backward; NULL computes and writes no parameter gradient (no
 * weight-gradient product, no gain / bias / column-sum output).  d_x: NULL, or [B,S,cfg->n_features] fp32, overwritten
 * with d loss / d x (packed rows: items at or beyond their slate's packed rows get 0, and d_hidden sent to them is
 * ignored).  `scratch`: arb_scorer_backward_ex_scratch_floats(cfg, B, S, d_x != NULL) floats.
 * arb_scorer_backward(..., d_scores, grads, ...) is arb_scorer_backward_ex(..., d_scores, NULL, grads, NULL, ...). */
int64_t arb_scorer_backward_ex_scratch_floats(const arb_scorer_config* cfg, int32_t B, int32_t S, int32_t want_dx);
int32_t arb_scorer_backward_ex(const arb_scorer_config* cfg, const float* params, const float* x, const uint8_t* mask,
                               const int64_t* indices, int32_t B, int32_t S, const float* scores,
                               const float* d_scores, const float* d_hidden, float* grads, float* d_x,
                               float* workspace, int64_t workspace_floats, float* scratch, int64_t scratch_floats,
                               uint64_t seed, void* stream);

/* The dropout seed read from device memory: the three calls above with `const uint64_t* seed_dev` (device memory,
 * non-null) in place of `seed`.  The kernels read *seed_dev when they execute, not when they are enqueued, and give
 * exactly the masks of the host-seeded call with seed = *seed_dev.  So a CUDA graph that captures them draws new
 * masks on every replay once the word is advanced (in stream order) between replays.  The word must hold the same
 * value when a step's backward executes as when its forward did: to advance it between the two, pass the backward a
 * copy taken before.  With dropout off (cfg->dropout and cfg->fc_dropout 0) the word is not read. */
int32_t arb_scorer_forward_dseed(const arb_scorer_config* cfg, const float* params, const float* x, const uint8_t* mask,
                                 const int64_t* indices, const float* pe_table,
                                 int32_t B, int32_t S, float* scores, float* workspace, int64_t workspace_floats,
                                 int32_t training, const uint64_t* seed_dev, void* stream);
int32_t arb_scorer_encode_dseed(const arb_scorer_config* cfg, const float* params, const float* x, const uint8_t* mask,
                                const int64_t* indices, const float* pe_table,
                                int32_t B, int32_t S, float* hidden, float* workspace, int64_t workspace_floats,
                                int32_t training, const uint64_t* seed_dev, void* stream);
int32_t arb_scorer_backward_ex_dseed(const arb_scorer_config* cfg, const float* params, const float* x,
                                     const uint8_t* mask, const int64_t* indices, int32_t B, int32_t S,
                                     const float* scores, const float* d_scores, const float* d_hidden, float* grads,
                                     float* d_x, float* workspace, int64_t workspace_floats, float* scratch,
                                     int64_t scratch_floats, const uint64_t* seed_dev, void* stream);

/* 0: unfused attention (materialised logits + generic GEMMs); 1: fused tensor-core attention forward kernel, unfused
 * backward; 2 (default): fused forward and backward kernels.  Fused kernels serve slates of <= 256 items at head width
 * 8, 16, 24 or 32 in bf16 mode and, in TF32 mode, slates of 1 ... 4096 items at every head width 4 ... 256 in steps of
 * 4; other shapes use the unfused path automatically (slate_length <= 1536).  Process-wide; exists for A/B tests. */
void arb_set_attention_mode(int32_t mode);

/* 1 (default): the fused attention kernels stop at each slate's extent -- the 16-row strips of keys (and, where their
 * gradients are exactly zero, of query rows) beyond round_up(last real item + 1, 16) are skipped: keys beyond the last
 * real item have probability exactly 0 and rows beyond the last item that is real or carries a score gradient have
 * exactly zero activation gradients, so results are unchanged; 0: all keys and all queries.  For A/B measurements. */
void arb_set_attention_skip_padding(int32_t on);

/* Packed rows (padding removal).  1: the encoder -- every LayerNorm, linear, attention and head kernel and every
 * gradient product -- runs over the items below each slate's extent only (extent = last unmasked item + 1, rounded up to
 * 16 rows; the live row count stays on the device, nothing synchronises).  Exact for every real item's score and every
 * parameter gradient; the scores of the items beyond a slate's extent are then 0 (and carry no gradient) instead of
 * what the network computes for a padded feature row -- values every consumer in allRank masks (losses.py: the
 * padded_value_indicator masks, metrics.py:31-35, inference_utils.py:51).  Applies to calls with a transformer whose
 * attention runs in the fused kernels (slate_length <= 256, head width 16 / 32), no dropout, no positional encoding
 * and d_output = 1; other calls use the dense layout.  0: dense [B*S] rows everywhere, i.e. padded items scored like
 * the reference does.  Process-wide. */
void arb_set_pack_rows(int32_t on);

/* Fused attention backward: 1: one CTA per SM walks the (slate, head) items and loads the next item's operands while it
 * computes the current one (when both fit its shared-memory pool, else as soon as the current one is done); 0: one CTA
 * per item, no prefetch.  Same results.  Process-wide; exists for A/B measurements. */
void arb_set_attention_bwd_persistent(int32_t on);
int32_t arb_get_pack_rows(void);

/* 1 (default): the kernels of a step are chained with programmatic dependent launch -- a kernel's prologue (barrier
 * init, tensor-map prefetch) overlaps its predecessor's last wave, and it blocks in griddepcontrol.wait
 * before its first global-memory access; 0: every launch fully serialised.  For A/B measurements. */
void arb_set_pdl(int32_t on);

/* Accepted for compatibility: every setting runs the same fused attention forward kernel. */
void arb_set_attention_fwd_two_pass(int32_t on);

/* GEMM kernel choice.  0: one CTA per output tile everywhere; 1: the persistent, decoupled-pipeline kernel (one CTA per
 * SM walking all tiles) wherever it is supported (not for fp32 products whose operands are both MN-major); 2 (default): persistent for every unbatched, non-split product except
 * short-K ones (K < 256) with a residual / mask tile.  Process-wide; exists
 * for A/B measurements. */
void arb_set_gemm_persistent(int32_t on);

/* 1 (default): MMA operands are rounded fp32 -> tf32 (nearest even) as the kernels load them; 0: the tensor core
 * truncates.  Process-wide; exists for the precision tests. */
void arb_set_tf32_round_on_load(int32_t enable);

/* Building block exposed for tests: C = epilogue(alpha * A op B) on row-major fp32 matrices (csrc/gemm_tf32.cu). */
int32_t arb_gemm_tf32(const float* A, const float* B, float* C, const float* aux, const float* bias, int32_t M,
                      int32_t N, int32_t K, int32_t a_mn, int32_t b_mn, int32_t batch, int64_t a_bstride,
                      int64_t b_bstride, int64_t c_bstride, int32_t block_n, int32_t flags, float alpha,
                      int32_t split_k, void* stream);

/* The same building block with bf16 operands (tensor-core bf16 MMA, fp32 accumulation) -- the matrix products of the
 * scorer's bf16 mode (BASELINE config 3).  A and B are bfloat16; C (and aux) bfloat16 when out_bf16 != 0, else fp32;
 * flags as for arb_gemm_tf32 (the ARB_GEMM_* values below); colsum_out: optional [N] bias-gradient accumulator. */
int32_t arb_gemm_bf16(const void* A, const void* B, void* C, const void* aux, const float* bias, int32_t M, int32_t N,
                      int32_t K, int32_t a_mn, int32_t b_mn, int32_t block_n, int32_t flags, float alpha,
                      int32_t split_k, int32_t out_bf16, float* colsum_out, void* stream);

/* The whole launch descriptor of the GEMM (csrc/gemm_tf32.h, GemmDesc), field for field, for tests that build the
 * launches the scorer builds: pitched and 4-D batched views, dropout, column sums, ReLU bit words and device-side row
 * counts.  A view has up to 4 dimensions, dim[0] contiguous, strides in elements; bf16 = 1: bfloat16 elements.
 * K-major operand: dim = (K, rows, b2, b3); MN-major: dim = (rows, K, b2, b3); C / aux: dim = (N, M, b2, b3).
 * flags are the EPI_* values of csrc/gemm_tf32.h: 1 bias, 2 ReLU, 4 add aux, 8 mask by aux > 0, 16 split-K into
 * atomic_out, 32 dropout, 64 column sums into colsum_out, 128 ReLU bit words written, 256 bit words read as the mask.
 * drop_call_seed: null, or a device word from which the kernel derives the seed
 * (drop_key as for the scorer's sites); else drop_seed is used.  rows_dev: null, or a device pointer to the live row
 * count.  Returns 0 or ARB_E_* without launching anything when the descriptor breaks a rule of the GEMM. */
typedef struct arb_gemm_view {
  const void* ptr;
  int64_t dim[4];
  int64_t stride[4];
  int32_t bf16;
} arb_gemm_view;
typedef struct arb_gemm_desc {
  int32_t M, N, K;
  int32_t a_mn, b_mn, b_tf32, dgrad;
  arb_gemm_view A, B, C, aux;
  int32_t nb2, nb3;
  int32_t a_b2, a_b3, b_b2, b_b3, c_b2, c_b3;
  int32_t block_n, split_k, flags;
  float alpha;
  const float* bias;
  float* atomic_out;
  int64_t atomic_ld;
  uint32_t drop_seed, drop_thresh;
  float drop_scale;
  uint32_t drop_key;
  const uint64_t* drop_call_seed;
  float* colsum_out;
  uint32_t* bits;
  const int32_t* rows_dev;
} arb_gemm_desc;
int32_t arb_gemm_launch(const arb_gemm_desc* d, void* stream);

/* Building blocks exposed for tests: the fused attention kernels of one encoder layer, dense layout, launched with the
 * descriptors the scorer uses (csrc/attention_fused.cu, attention_fused_bwd.cu, attention_long.cu).  Shapes: B slates
 * of S <= 4096 items, h heads of width dk 4 ... 256 in steps of 4, with an fp32 context; a bf16 context needs S <= 256
 * and dk 8, 16, 24 or 32 (otherwise ARB_E_UNSUPPORTED); d = h * dk.
 *   qkv       [B*S, 3d] fp32: the QKV linear's output, Q | K | V, head j at columns j*dk ... j*dk + dk - 1 of each
 *   mask      [B, S] uint8, 1 = padded item (a masked key)
 *   extent    nullable [B] int32: keys at or beyond extent[b] must be masked; the kernels skip their work (forward:
 *             keys; backward: keys and queries -- the rows of d_ctx at or beyond it must be zero).  Null: all rows.
 *   ctx       [B*S, d]: fp32, or bfloat16 (round to nearest even) when ctx_bf16
 *   stat_max  [B, h, S] fp32: the row maximum of the raw logits Q K^T over the unmasked keys (-inf: none)
 *   stat_sum  [B, h, S] fp32: sum over the unmasked keys of exp((s - max) / sqrt(dk))
 *   d_ctx     [B*S, d] fp32;  d_qkv [B*S, 3d], dQ | dK | dV in the layout of qkv, of the context's element type
 *   dbias_qkv nullable [3d] fp32: the column sums of d_qkv are ADDED to it (the bias gradient of the QKV linear)
 *   delta_scratch [B, h, S] fp32
 * Dropout on the probabilities with rate p uses the scorer's site of encoder layer `layer` under the call seed `seed`:
 * element ((b*h + head)*S + query)*S + key.  The backward reads the forward's statistics and context.  An all-padded
 * slate gets NaN context rows (as the reference) and zero gradients.  Returns ARB_E_UNSUPPORTED for other shapes. */
int32_t arb_attention_forward(const float* qkv, const uint8_t* mask, const int32_t* extent, int32_t B, int32_t S,
                              int32_t h, int32_t dk, float p, uint64_t seed, int32_t layer, int32_t ctx_bf16,
                              void* ctx, float* stat_max, float* stat_sum, void* stream);
int32_t arb_attention_backward(const float* qkv, const void* ctx, int32_t ctx_bf16, const float* d_ctx,
                               const uint8_t* mask, const int32_t* extent, const float* stat_max,
                               const float* stat_sum, int32_t B, int32_t S, int32_t h, int32_t dk, float p,
                               uint64_t seed, int32_t layer, void* d_qkv, float* dbias_qkv, float* delta_scratch,
                               void* stream);
/* The same kernels over padded heads, as the scorer runs a head width w = d_model / h that is not a multiple of 4:
 * every head takes hs = round_up(w, 4) columns of the buffers (any w from 1 to 256; hs = w when w is a multiple of 4),
 * and the probabilities are softmax(Q K^T / sqrt(w)).  dp = h * hs; fp32 context only.
 *   qkv    [B*S, 3 dp]: Q | K | V, head j at columns j*hs ... j*hs + hs - 1 of each; columns w ... hs - 1 of every
 *          head must be zero (the scorer's padded QKV weights and bias give exact zeros there)
 *   ctx, d_ctx [B*S, dp]; d_qkv [B*S, 3 dp]; dbias_qkv nullable [3 dp]
 * The pad columns of ctx and d_qkv come out as +0 (a zero column adds exact zeros to every product) and the pad
 * entries of dbias_qkv receive +0.  Everything else as arb_attention_forward / arb_attention_backward. */
int32_t arb_attention_padded_forward(const float* qkv, const uint8_t* mask, const int32_t* extent, int32_t B, int32_t S,
                                     int32_t h, int32_t w, float p, uint64_t seed, int32_t layer, float* ctx,
                                     float* stat_max, float* stat_sum, void* stream);
int32_t arb_attention_padded_backward(const float* qkv, const float* ctx, const float* d_ctx, const uint8_t* mask,
                                      const int32_t* extent, const float* stat_max, const float* stat_sum, int32_t B,
                                      int32_t S, int32_t h, int32_t w, float p, uint64_t seed, int32_t layer,
                                      float* d_qkv, float* dbias_qkv, float* delta_scratch, void* stream);

/* Building blocks exposed for tests: the encoder's feed-forward sublayer as the scorer runs it in TF32 mode without
 * dropout, both linears chained in one kernel per direction (csrc/ffn_chain.cu).  All matrices are dense row-major
 * fp32; d is a multiple of 32 up to 256 and d_ff a multiple of 64 (else ARB_E_UNSUPPORTED).  The weights are read as
 * given: pass them tf32-rounded, as the scorer's weight copy holds them.  The activations are rounded (or truncated,
 * arb_set_tf32_round_on_load(0)) as the GEMMs round their operands, so the results equal bit for bit those of the two
 * arb_gemm_tf32 products they replace.
 *   forward:  h = relu(x w1^T + b1), bits[r][u / 32] bit u % 32 = (h[r][u] > 0), y = h w2^T + b2 + res
 *             x, res, y [rows, d] (res may alias y); w1 [d_ff, d]; w2 [d, d_ff]; h [rows, d_ff] and bits
 *             [rows, d_ff / 32] are nullable (not written).
 *   backward: dh = (dy w2) masked by bits, dx = dh w1;  w2t = w2^T [d_ff, d], w1t = w1^T [d, d_ff]; dh nullable;
 *             grad_b1 (nullable) += the column sums of dh, per 128-row tile in the EPI_COLSUM epilogue's order.
 *   rows_dev (nullable, device int32): the live row count; the 128-row tiles at or beyond it are neither read nor
 *   written. */
int32_t arb_ffn_forward(const float* x, const float* w1, const float* b1, const float* w2, const float* b2,
                        const float* res, int32_t rows, int32_t d, int32_t d_ff, float* y, float* h, uint32_t* bits,
                        const int32_t* rows_dev, void* stream);
int32_t arb_ffn_backward_input(const float* dy, const float* w2t, const float* w1t, const uint32_t* bits,
                               int32_t rows, int32_t d, int32_t d_ff, float* dx, float* dh, float* grad_b1,
                               const int32_t* rows_dev, void* stream);

/* Building blocks exposed for tests: the SIMT row kernels (csrc/scorer_kernels.cu), launched by the scorer's own
 * launchers, so that the steps per warp, the row layout and the reduction slots depend on `rows` as in the scorer
 * (launches of 2^17 rows or more take the large-launch path).  Rows are `width` floats apart; width is a multiple of 4,
 * at most 1024 (else ARB_E_UNSUPPORTED).  Nullable arguments: y16, dy16_in, dy16_out, dres, dx_masked, colsum_out, the
 * gradient outputs grad_*, rows_dev and rowmap (both device int32); a null output is not computed.
 *   - Gradients and column sums are ACCUMULATED: grad_*, colsum_out and the multi-head grad_w / grad_wb += their sums.
 *   - rows_dev: rows at or beyond *rows_dev (live rows <= rows) are not read and not written.
 *   - rowmap [rows]: layer norm forward writes row r to y[rowmap[r]], its backward reads dy[rowmap[r]]; the head reads
 *     and writes score / dscore [rowmap[r]].  rowmap[r] < 0: no destination, or a zero gradient.  fp32 rows only.
 *   - Dropout with rate p uses make_drop_site(seed, layer, site) as the scorer does; the row kernels' element counter
 *     is row * width + column.  dx_masked = dx through that mask (not written when p = 0); dy16_out is the bfloat16
 *     copy (nearest even) of dx_masked, or of dx when p = 0; dy16_in replaces dy with bfloat16 values.
 *   - torch_mode: nn.LayerNorm (biased variance, eps under the root); sd receives sqrt(var + eps), and the backward is
 *     then called with eps = 0 as the scorer calls it.  Otherwise the reference's LayerNorm (unbiased std, eps added to
 *     the std).  A row with sd = 0 (a constant row) gets y = b, and in the backward the std term of dx is 0.
 *   - act: ARB_ACT_*; has_norm = 0 is the FC-only head score = act(w . x + wb[0]).
 *   - the multi-output head: score [rows, n] = act(xf w^T + wb), w [n, width]; grad_w and grad_wb both or neither.
 * Softmax: in place on scores [B, h, S] rows of `pitch` >= S floats (S <= 1536, else ARB_E_UNSUPPORTED), keys with
 * mask [B, S] = 1 get probability 0, an all-masked slate gets NaN rows.  Dropout on the probabilities with the
 * attention site of `layer`, counter row * S + key (independent of pitch), as in the fused kernels.  The backward
 * turns dprob (the gradient w.r.t. the dropped probabilities) into dS = P (dP - sum P dP) in place and overwrites
 * prob (the undropped P) with the dropped probabilities.  Columns from S to pitch are neither read nor written. */
int32_t arb_layernorm_forward(const float* x, const float* a, const float* b, float eps, int32_t torch_mode,
                              int64_t rows, int32_t width, float* y, void* y16, float* mean, float* sd,
                              const int32_t* rows_dev, const int32_t* rowmap, void* stream);
int32_t arb_layernorm_backward(const float* dy, const void* dy16_in, const float* x, const float* a, const float* mean,
                               const float* sd, float eps, int32_t torch_mode, const float* dres, int64_t rows,
                               int32_t width, float* dx, float* grad_a, float* grad_b, float* dx_masked,
                               void* dy16_out, float* colsum_out, float p, uint64_t seed, int32_t layer, int32_t site,
                               const int32_t* rows_dev, const int32_t* rowmap, void* stream);
int32_t arb_head_forward(const float* x, const float* a, const float* b, float eps, const float* w, const float* wb,
                         int32_t has_norm, int32_t act, int64_t rows, int32_t width, float* score, float* mean,
                         float* sd, const int32_t* rows_dev, const int32_t* rowmap, void* stream);
int32_t arb_head_backward(const float* dscore, const float* score, const float* x, const float* a, const float* b,
                          const float* mean, const float* sd, float eps, const float* w, int32_t has_norm, int32_t act,
                          int64_t rows, int32_t width, float* dx, float* grad_a, float* grad_b, float* grad_w,
                          float* grad_wb, float* dx_masked, void* dy16_out, float* colsum_out, float p, uint64_t seed,
                          int32_t layer, int32_t site, const int32_t* rows_dev, const int32_t* rowmap, void* stream);
int32_t arb_head_multi_forward(const float* xf, const float* w, const float* wb, int32_t act, int64_t rows,
                               int32_t width, int32_t n, float* score, void* stream);
int32_t arb_head_multi_backward(const float* dscore, const float* score, const float* xf, const float* w, int32_t act,
                                int64_t rows, int32_t width, int32_t n, float* dxf, float* grad_w, float* grad_wb,
                                float* dx_masked, float* colsum_out, float p, uint64_t seed, int32_t layer,
                                int32_t site, void* stream);
/* out[c] += sum over rows r of in[r * ld + c], c < width; ld >= width, a multiple of 4 */
int32_t arb_column_sums(const float* in, int64_t rows, int32_t width, int64_t ld, float* out, void* stream);
int32_t arb_softmax_forward(float* scores, const uint8_t* mask, int32_t B, int32_t h, int32_t S, int32_t pitch,
                            float p, uint64_t seed, int32_t layer, void* stream);
int32_t arb_softmax_backward(float* dprob, float* prob, int64_t rows, int32_t S, int32_t pitch, float p,
                             uint64_t seed, int32_t layer, void* stream);

/* ---------------------------------------------------------------- optimiser + profiling helpers
 * Flat Adam over the scorer's flat parameter/gradient buffers: torch.optim.Adam semantics (the optimiser the
 * reference instantiates from its config, allrank/main.py:82), one launch.  grads are multiplied by grad_scale
 * first (1/world_size after a sum all-reduce).  `step` is the 1-based step count. */
int32_t arb_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                      float beta1, float beta2, float eps, float weight_decay, int32_t step, float grad_scale,
                      void* stream);
/* The same with the step counter on the device: state[0] (a float, initially 0) is incremented by a one-thread prep
 * launch and the step's bias corrections are computed there -- what a CUDA-graph replay of a training step needs
 * (allrank_b200.graph.GraphedTrainStep); state holds 3 floats. */
int32_t arb_adam_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                          float beta1, float beta2, float eps, float weight_decay, float* state, float grad_scale,
                          void* stream);

/* ---------------------------------------------------------------- slate movers (SURVEY.md 8(f) ranks 3-4)
 * arb_assemble_slates: the per-slate FixLength transform + ToTensor + DataLoader collation of
 * allrank/data/dataset_loading.py:32-93,:230-247 for a batch of queries, from a corpus resident in HBM:
 *   docs_x [N,F] fp32 and docs_y [N] fp32 grouped by query, offsets [n_queries+1] int64 (CSR), queries [B] int64
 *   (a query number outside [0, n_queries) produces an all-padding slate).
 * Query shorter than S: rows in order, then zero rows with y = -1 and index = -1 (bit-identical to the reference).
 * Otherwise: S items sampled uniformly without replacement in random order; a sample without any relevant item is
 * redrawn while the query has one (the query's only relevant item, if its labels sum to 1, replaces the last
 * sampled item instead) -- :55-74.  The sample stream is a counter hash of (seed, slate, attempt, item).
 * max_query_len: longest query of the corpus (sizes the shared-memory sort; arb_assemble_slates_smem_bytes).
 * Outputs: x_out [B,S,F], y_out [B,S] fp32, idx_out [B,S] int64 (positions inside the query, -1 = padded). */
size_t arb_assemble_slates_smem_bytes(int32_t max_query_len, int32_t S);
int32_t arb_assemble_slates(const float* docs_x, const float* docs_y, const int64_t* offsets, int64_t n_queries,
                            const int64_t* queries, int32_t B, int32_t S, int32_t F, int32_t max_query_len,
                            uint64_t seed, float* x_out, float* y_out, int64_t* idx_out, void* stream);
/* inference_utils.__rank_slates (allrank/inference/inference_utils.py:37-60): x_out[b,r,:] = x[b,order[b,r],:],
 * y_out[b,r] = y[b,order[b,r]], with `order` the descending score ranking (arb_rank_metrics' out_order). */
int32_t arb_gather_slates(const float* x, const float* y, const int32_t* order, int32_t B, int32_t S, int32_t F,
                          float* x_out, float* y_out, void* stream);

/* ---------------------------------------------------------------- click models (allrank/click_models)
 * A click model is a tree of at most ARB_CLICK_MAX_NODES nodes.  Node 0 is the root; the children of a node are the
 * contiguous nodes [first_child, first_child + n_children), each with a larger index than its parent, and every
 * non-root node has exactly one parent.  Every model sees the REAL items of a slate (y != pad) in slate order, like
 * MaskedRemainMasked (click_utils.py:30-53); n is their number and "position" is the index among them.
 *   FIXED       click the positions list[list_offset .. +n_list] (integers stored as doubles; negative = from the end);
 *               a position outside [-n, n) sets status ARB_CLICK_INDEX_ERROR
 *   RANDOM      exactly iparam distinct items, uniformly (the iparam smallest per-item hash keys); iparam > n sets
 *               status ARB_CLICK_VALUE_ERROR
 *   RELEVANT    click iff y >= fparam0 (compared in fp32)
 *   CASCADE     observed iff observe_tables[iparam * S + p] >= u (u a per-item uniform); click iff
 *               (observed ? y : 0*y) >= fparam1 (fp32).  The table holds 1 / (p+1)**eta, evaluated by the caller.
 *   MULTIPLE    evaluate only child argmax(u < list[list_offset + k]) (cumulative probabilities, n_list = n_children;
 *               child 0 when none holds), u one uniform per slate
 *   CONDITIONED iparam 0: all children click, 1: any child clicks
 *   MAXCLICKS   the child's clicks whose running count is <= fparam0 (+inf passes everything)
 *   DUPLICATES  item j clicks iff min_{i<j} dist(i, j) > fparam0, metric iparam (ARB_CLICK_METRIC_*); n = 0 sets status
 *               ARB_CLICK_VALUE_ERROR
 *   DIVERSE     margin = linear quantile fparam0 of all pairwise euclidean distances (0 when n < 2); the child's clicks
 *               are walked top to bottom and kept iff their distance to every kept item is > margin
 * Distances are computed in fp64 from the fp32 features, summed over the features in order without FMA (scipy's cdist).
 * Uniforms are counter-based: 53 bits of a hash of (seed, node, slate_offset + slate, position). */
#define ARB_CLICK_MAX_NODES 32
#define ARB_CLICK_MAX_SLATE 4096
#define ARB_CLICK_FIXED 0
#define ARB_CLICK_RANDOM 1
#define ARB_CLICK_RELEVANT 2
#define ARB_CLICK_CASCADE 3
#define ARB_CLICK_MULTIPLE 4
#define ARB_CLICK_CONDITIONED 5
#define ARB_CLICK_MAXCLICKS 6
#define ARB_CLICK_DUPLICATES 7
#define ARB_CLICK_DIVERSE 8
#define ARB_CLICK_METRIC_EUCLIDEAN 0
#define ARB_CLICK_METRIC_SQEUCLIDEAN 1
#define ARB_CLICK_METRIC_CITYBLOCK 2
#define ARB_CLICK_METRIC_CHEBYSHEV 3
/* per-slate status codes */
#define ARB_CLICK_OK 0
#define ARB_CLICK_INDEX_ERROR 1
#define ARB_CLICK_VALUE_ERROR 2

typedef struct arb_click_node {
  int32_t kind, first_child, n_children, iparam, list_offset, n_list;
  double fparam0, fparam1;
} arb_click_node;

/* Device workspace bytes for processing all B slates in one launch: one fp64 upper triangle of pairwise distances
 * per slate when the tree has a DIVERSE node, 0 otherwise (the tree itself travels with the launch).  A smaller
 * workspace is processed in chunks of slates; it must hold at least one slate's triangle. */
size_t arb_click_workspace_bytes(const arb_click_node* nodes_host, int32_t n_nodes, int32_t B, int32_t S, int32_t F);
/* y [B,S] fp32 (pad marks padding), x [B,S,F] fp32 (may be NULL when no node measures distances), observe_tables
 * device fp64 [n_tables, S] for CASCADE nodes (may be NULL without them).  Writes clicks [B,S] fp32 (0/1, pad value
 * `pad` at padded positions) and status [B] int32 (ARB_CLICK_*).  Never synchronises. */
int32_t arb_click_slates(const arb_click_node* nodes_host, int32_t n_nodes, const double* list_host, int32_t n_list,
                         const double* observe_tables, const float* x, const float* y, int32_t B, int32_t S, int32_t F,
                         float pad, int64_t slate_offset, uint64_t seed, float* clicks, int32_t* status,
                         void* workspace, size_t ws_bytes, void* stream);

/* Per-launch device timing for bench.py's roofline: enable, run steps, collect per kernel class
 * (0 = tensor-core GEMM [work = flops], 1 = scorer SIMT, 2 = losses, 3 = metrics, 4 = optimiser, 5 = slate assembly /
 * gather [work = bytes]). */
void arb_prof_enable(int32_t on);
int32_t arb_prof_collect(int32_t cls, double* total_ms, double* total_work, int64_t* launches);
/* algorithmic HBM bytes (operands + outputs, each counted once) summed by the last arb_prof_collect(cls, ...) */
double arb_prof_last_bytes(int32_t cls);
/* Per-kernel table since arb_prof_enable(1), one text line per distinct launch name:
 *   name \t class \t launches \t total_ms \t total_work \t total_algorithmic_bytes
 * (GEMM launches are named by shape and operand layout, the other kernels by their launcher).  Writes at most
 * cap - 1 bytes + NUL into buf and returns the count; buf == NULL returns the size needed. */
int64_t arb_prof_report(char* buf, int64_t cap);

#ifdef __cplusplus
}
#endif
#endif /* ALLRANK_B200_H */
