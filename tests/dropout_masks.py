"""Host restatement of the scorer's counter-based dropout masks (allrank_b200/csrc/dropout.cuh), shared by the GPU
tests that compare the CUDA scorer with the eager reference maths UNDER THE SAME MASKS."""
import numpy as np
import torch

M32 = np.uint64(0xFFFFFFFF)


def _mix32(h):
    h = h ^ (h >> np.uint64(16)); h = (h * np.uint64(0x85ebca6b)) & M32
    h = h ^ (h >> np.uint64(13)); h = (h * np.uint64(0xc2b2ae35)) & M32
    return h ^ (h >> np.uint64(16))


def _site(call_seed, layer, site, p):
    """Host restatement of make_drop_site / drop_keep (csrc/dropout.cuh)."""
    m64 = (1 << 64) - 1
    z = (call_seed + 0x9e3779b97f4a7c15 * (layer * 8 + site + 1)) & m64
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & m64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & m64
    z ^= z >> 31
    seed = (z & 0xFFFFFFFF) ^ (z >> 32)
    # the library takes the rate as a float: p = 0.1 gives thresh 429496736, not the 429496729 of the double 0.1
    thresh = max(1, min(int(float(np.float32(p)) * 4294967296.0), 0xFFFFFFFF))
    return np.uint64(seed), np.uint64(thresh), 1.0 / (1.0 - p)


def mask_tensor(shape, call_seed, layer, site, p):
    if p <= 0:
        return None
    seed, thresh, scale = _site(call_seed, layer, site, p)
    idx = np.arange(int(np.prod(shape)), dtype=np.uint64)
    h = _mix32((idx & M32) ^ seed)
    h = _mix32((h + (idx >> np.uint64(32)) * np.uint64(0x9e3779b1) + np.uint64(0x7f4a7c15)) & M32)
    keep = (h >= thresh).astype(np.float32) * scale
    return torch.tensor(keep.reshape(shape))


SITE_FC, SITE_ATTN_P, SITE_ATTN_OUT, SITE_FFN_HID, SITE_FFN_OUT = 0, 1, 2, 3, 4


def scorer_masks(call_seed, B, S, fc_sizes, n_layers, heads, d_ff, p, p_fc):
    """{(layer, site name): scaled keep mask} for oracle.tf32_emulation.scorer_forward: one "fc" entry per FC layer
    (keyed by the layer index, model.py:43) and the four encoder sites per block (transformer.py:105,155,227)."""
    R, d = B * S, fc_sizes[-1]
    drop = {}
    for i, width in enumerate(fc_sizes):
        drop[(i, "fc")] = mask_tensor((R, width), call_seed, i, SITE_FC, p_fc)
    for l in range(n_layers):
        drop[(l, "attn_p")] = mask_tensor((B, heads, S, S), call_seed, l, SITE_ATTN_P, p)
        drop[(l, "attn_out")] = mask_tensor((R, d), call_seed, l, SITE_ATTN_OUT, p)
        drop[(l, "ffn_hid")] = mask_tensor((R, d_ff), call_seed, l, SITE_FFN_HID, p)
        drop[(l, "ffn_out")] = mask_tensor((R, d), call_seed, l, SITE_FFN_OUT, p)
    return drop
