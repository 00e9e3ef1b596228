// Default settings of the process-wide A/B switches (each has a setter in include/allrank_b200.h and an environment
// variable read by allrank_b200/_lib.py).  Kept in one place so that a setting that has not been validated on the GPU
// can be turned off with one edit.
#pragma once
#define ARB_DEFAULT_PDL 1                 // programmatic dependent launch (arb_set_pdl, ARB_PDL)
#define ARB_DEFAULT_SKIP_PADDING 1        // attention kernels stop at the slate extent (arb_set_attention_skip_padding)
#define ARB_DEFAULT_GEMM_PERSISTENT 2     // 0 never, 1 everywhere, 2 all unbatched non-split shapes but short-K + aux tile (arb_set_gemm_persistent)
#define ARB_DEFAULT_PACK_ROWS 1           // encoder over the unpadded rows only (arb_set_pack_rows, ARB_PACK_ROWS)
#define ARB_DEFAULT_ATTN_BWD_PERSISTENT 1 // attention backward: one CTA per SM walks the (slate, head) items (arb_set_attention_bwd_persistent)
#define ARB_DEFAULT_RELU_BITS 1           // FFN ReLU backward from a 1-bit-per-unit mask written by the W1 epilogue (arb_set_relu_bits)
