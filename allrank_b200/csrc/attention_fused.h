// Fused attention core (attention_fused.cu): launch descriptors.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "gemm_tf32.h"

namespace arb {

struct AttnFwdArgs {
  TRef q, k, v, o;            // per-head views: dim = (dk, S, h, B)
  const uint8_t* mask;        // [B,S], 1 = padded key
  float* stat_max;            // [B,h,S] row max of the raw logits Q K^T (before the 1/sqrt(dk) scale)
  float* stat_sum;            // [B,h,S] sum_j exp((s_j - max)/sqrt(dk)) over real keys
  int B, h, S, dk;
  float scale;                // 1/sqrt(dk)
  DropSite drop{0u, 0u, 1.0f};   // dropout on the probabilities (transformer.py:154-155); index ((b*h+head)*S+q)*S+key
  const int* extent = nullptr;   // optional [B]: every key >= extent[b] is masked (slate_extents); work beyond it is
                                 // skipped -- those keys have probability exactly 0, so the result is unchanged
  const int* pack_off = nullptr; // packed rows (needs extent): q/k/v/o are views (dk, rows, h, 1) of activations that hold
                                 // only the first round_up(extent[b], 16) rows of every slate, slate b at row pack_off[b]
};

bool attn_fused_supported(int S, int dk);
void set_attn_fwd_two_pass(int on);   // accepted for the C ABI; every setting runs the same kernel
int launch_attn_fwd(const AttnFwdArgs& a, cudaStream_t st);

}  // namespace arb

namespace arb {

struct AttnBwdArgs {
  TRef q, k, v, d_o;          // per-head views (dk, S, h, B): saved Q/K/V and the incoming d ctx
  TRef dq, dk_, dv;           // per-head views of the outputs (into the packed d qkv buffer)
  const void* o_ptr;          // ctx [B*S, d_model] (for delta = rowsum(dO * O)); bfloat16 when o_bf16
  int o_bf16 = 0;
  const float* do_ptr;        // d ctx [B*S, d_model]
  int64_t o_pitch;
  const uint8_t* mask;        // [B,S]
  const float* stat_max;      // [B,h,S] from the fused forward
  const float* stat_sum;      // [B,h,S]
  float* delta;               // [B,h,S] scratch
  float* dbias_qkv = nullptr; // optional [3*d_model]: += column sums of dQ | dK | dV (bias gradient of the QKV linear)
  int d_model = 0;
  int B, h, S, dk;
  float scale;
  DropSite drop{0u, 0u, 1.0f};
  const int* extent = nullptr;   // optional [B]: rows >= extent[b] are masked keys whose d ctx rows are exactly zero
                                 // (slate_extents over the mask and the incoming score gradient): their tiles are
                                 // skipped and their dQ / dK / dV rows written as zeros -- exactly what the dense
                                 // computation produces
  const int* pack_off = nullptr; // packed rows (needs extent = the forward's key extents): see AttnFwdArgs
  const int* rows_dev = nullptr; // packed rows: plan[0] (live packed rows, for the delta kernel)
  const int* rowmap = nullptr;   // packed rows: item index of every packed row (for the delta kernel)
};

bool attn_fused_bwd_supported(int S, int dk);
void set_attn_bwd_persistent(int on);   // 1: one CTA per SM walks the (slate, head) items; 0: one CTA per item
int launch_attn_bwd(const AttnBwdArgs& a, cudaStream_t st);

}  // namespace arb
