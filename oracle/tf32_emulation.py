"""TF32-faithful variant of the oracle scorer (TEST INFRASTRUCTURE).

Same maths as oracle/scorer_ref.py (reference: allrank/models/{model,transformer}.py), but every matrix
product -- forward and backward -- sees its operands with the mantissa cut to 10 bits, which is what the
tensor-core tf32 datapath does to fp32 operands; accumulation stays fp32/fp64.  It separates "TF32 rounding"
from "kernel bug" when the CUDA scorer is compared with the fp32 reference: the CUDA path must agree with this
emulation much more tightly than with the fp32 oracle.
"""
import math

import torch


def tf32_trunc(t, mode="trunc"):
    """Cut an fp32 tensor to TF32 precision (1+8+10 bits). mode: 'trunc' (toward zero) or 'rna' (round to nearest);
    mode 'bf16': round to nearest even to bfloat16 precision (1+8+7 bits) -- the operands of the bf16 mode."""
    t = t.float().contiguous()
    if mode == "bf16":
        return t.bfloat16().float()
    bits = t.view(torch.int32)
    if mode == "rna":
        bits = bits + 0x1000
    return (bits & ~0x1FFF).view(torch.float32)


class _RoundGrad(torch.autograd.Function):
    """Identity whose GRADIENT is rounded to bfloat16: the bf16 mode stores the gradient of a LayerNorm output as
    bfloat16 (it is produced by an input-gradient product and only then read by the LayerNorm backward)."""

    @staticmethod
    def forward(ctx, x):
        return x

    @staticmethod
    def backward(ctx, g):
        return g.bfloat16().float()


class _MM(torch.autograd.Function):
    """C = A @ B with TF32 operands in the forward and in both backward products."""

    @staticmethod
    def forward(ctx, a, b, mode, acc_dtype):
        ctx.save_for_backward(a, b)
        ctx.mode, ctx.acc = mode, acc_dtype
        return (tf32_trunc(a, mode).to(acc_dtype) @ tf32_trunc(b, mode).to(acc_dtype)).float()

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        m, acc = ctx.mode, ctx.acc
        gt = tf32_trunc(g, m).to(acc)
        da = (gt @ tf32_trunc(b, m).to(acc).transpose(-1, -2)).float()
        db = (tf32_trunc(a, m).to(acc).transpose(-1, -2) @ gt).float()
        while da.dim() > a.dim():
            da = da.sum(0)
        while db.dim() > b.dim():
            db = db.sum(0)
        if da.shape != a.shape:
            da = da.sum(tuple(range(da.dim() - a.dim())) or 0).reshape(a.shape) if da.numel() != a.numel() else da.reshape(a.shape)
        if db.shape != b.shape:
            # weight shared across a leading batch of rows: reduce the broadcast dimensions
            extra = db.dim() - b.dim()
            db = db.sum(tuple(range(extra))) if extra > 0 else db
            if db.shape != b.shape:
                db = db.reshape(-1, *b.shape).sum(0)
        return da, db, None, None


def mm(a, b, mode="trunc", acc_dtype=torch.float64):
    return _MM.apply(a, b, mode, acc_dtype)


def row_norm(x, a, b, eps=1e-6):
    mu = x.mean(-1, keepdim=True)
    sd = x.std(-1, keepdim=True)
    return a * (x - mu) / (sd + eps) + b


def _activation(t, name):
    if name is None:
        return t
    return {"ReLU": torch.relu, "Tanh": torch.tanh, "Sigmoid": torch.sigmoid}[name](t)


def scorer_forward(sd, x, mask, n_layers, heads, out_act=None, mode="trunc", drop=None, fc_act=None, bf16=False):
    """Functional forward from a reference-keyed state_dict (tensors may require grad).
    `drop`: optional {(layer, site): already-scaled mask tensor} with sites fc / attn_p / attn_out / ffn_hid /
    ffn_out (shapes [R,width], [B,h,S,S], [R,d], [R,d_ff], [R,d]) -- the dropout sites of transformer.py:105,155,227
    and model.py:43 (site "fc" is keyed by the FC layer index).
    bf16=True emulates the CUDA scorer's bf16 mode: encoder linears with bfloat16-rounded operands (weights,
    LayerNorm outputs, context, hidden layer, incoming gradients), LayerNorm-output gradients stored as bfloat16,
    attention score / context products and the input FC block in TF32 (`mode`) on fp32 data.
    General FCModel (model.py:35-44): `input_layer.input_norm.*` if present in `sd`, then every
    `input_layer.layers.{i}` followed by `fc_act` and dropout; `output_layer.w_1.weight` with n > 1 rows gives
    [B,S,n] outputs (model.py:111-117)."""
    B, S, F = x.shape
    R = B * S
    drop = drop or {}

    def dr(t, layer, site):
        m = drop.get((layer, site))
        return t if m is None else t * m

    def lin(inp, w, b, m=None):   # inp [R, in]
        return mm(inp, w.t(), m or mode) + b

    enc = "bf16" if bf16 else mode          # operand rounding of the encoder linears

    def normed(t, a, b_):
        y = row_norm(t, a, b_)
        return _RoundGrad.apply(y) if bf16 else y

    h = x.reshape(R, F)
    if "input_layer.input_norm.weight" in sd:    # nn.LayerNorm(F): biased variance, eps = 1e-5 under the root
        h = torch.nn.functional.layer_norm(h, (F,), sd["input_layer.input_norm.weight"], sd["input_layer.input_norm.bias"])
    i = 0
    while f"input_layer.layers.{i}.weight" in sd:
        h = dr(_activation(lin(h, sd[f"input_layer.layers.{i}.weight"], sd[f"input_layer.layers.{i}.bias"]), fc_act), i, "fc")
        i += 1
    d = h.shape[-1]
    dk = d // heads if n_layers else 0
    for l in range(n_layers):
        p = f"encoder.layers.{l}."
        xn = normed(h, sd[p + "sublayer.0.norm.a_2"], sd[p + "sublayer.0.norm.b_2"])
        q, k, v = (lin(xn, sd[p + f"self_attn.linears.{i}.weight"], sd[p + f"self_attn.linears.{i}.bias"], enc)
                   .view(B, S, heads, dk).transpose(1, 2) for i in range(3))
        logits = mm(q, k.transpose(-1, -2), mode) * (1.0 / math.sqrt(dk))
        logits = logits.masked_fill(mask[:, None, None, :], float("-inf"))
        prob = dr(torch.softmax(logits, dim=-1), l, "attn_p")
        ctx = mm(prob, v, mode).transpose(1, 2).reshape(R, d)
        h = h + dr(lin(ctx, sd[p + "self_attn.linears.3.weight"], sd[p + "self_attn.linears.3.bias"], enc), l, "attn_out")
        xn = normed(h, sd[p + "sublayer.1.norm.a_2"], sd[p + "sublayer.1.norm.b_2"])
        hid = dr(torch.relu(lin(xn, sd[p + "feed_forward.w_1.weight"], sd[p + "feed_forward.w_1.bias"], enc)), l, "ffn_hid")
        h = h + dr(lin(hid, sd[p + "feed_forward.w_2.weight"], sd[p + "feed_forward.w_2.bias"], enc), l, "ffn_out")
    if n_layers:
        h = row_norm(h, sd["encoder.norm.a_2"], sd["encoder.norm.b_2"])
    hw = sd["output_layer.w_1.weight"]
    n_out = hw.shape[0]
    z = (h[:, None, :] * hw[None, :, :]).sum(-1) + sd["output_layer.w_1.bias"]   # fp32 head (SIMT), [R, n_out]
    z = z.view(B, S) if n_out == 1 else z.view(B, S, n_out)
    return _activation(z, out_act)
