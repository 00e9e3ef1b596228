"""Drop-in replacement for allrank.models.model.make_model / LTRModel on the GPU.

Same call surface as the reference (/root/reference/allrank/models/model.py):

    model = make_model(fc_model=..., transformer=..., post_model=..., n_features=...)      # model.py:131
    scores = model(x, mask, indices)            # [B,S] ([B,S,d_output] when d_output > 1; model.py:72-80)
    scores = model.score(x, mask, indices)      # [B,S]   (model.py:82-92,  train_utils.py:34)
    hidden = model.prepare_for_output(x, mask, indices)   # [B,S,d_model], the encoder output (model.py:62-70)
    model.parameters() / .state_dict() / .load_state_dict() / .train() / .eval() / .to(device)

and the same state_dict keys and shapes as the reference's module tree (so a reference `model.pkl` loads):
`input_layer.layers.{i}.{weight,bias}` (+ `input_layer.input_norm.{weight,bias}`), `encoder.layers.{l}.self_attn.linears.{0..3}.{weight,bias}`,
`encoder.layers.{l}.feed_forward.w_{1,2}.{weight,bias}`, `encoder.layers.{l}.sublayer.{0,1}.norm.{a_2,b_2}`,
`encoder.norm.{a_2,b_2}`, `output_layer.w_1.{weight,bias}`; same initialisation order (nn.Linear defaults,
clones share the prototype's bias, xavier_uniform_ on every parameter with dim > 1: model.py:148-150).

The forward and backward passes are fixed launch sequences inside liballrank_b200.so (csrc/scorer.cu): tensor-core
TF32 GEMMs + fp32 SIMT kernels.  The nn.Parameters are views of ONE flat fp32 buffer and their .grad are views of
one flat gradient buffer -- which is what makes the single-bucket NCCL all-reduce (allrank_b200/ddp.py) and
flat optimisers possible.  There is no eager fallback: CPU tensors raise.

Dropout (transformer.dropout on attention probabilities, sublayer outputs and the FFN hidden layer; fc_model.dropout
on the input FC) is fused into the kernels with counter-based masks that backward regenerates; like nn.Dropout it is
active in train() mode only.  The mask stream differs from torch's Philox stream: parity under dropout is statistical.
The per-call seed is drawn on the host, or inside `with model.dropout_seed_from(seed_tensor):` read by the kernels from
a device tensor -- what a CUDA-graph replay of a training step needs (allrank_b200.graph).

Positional encodings (allrank/models/positional.py: fixed sinusoidal buffer or learned embedding indexed by `indices`,
padding row for padded items) are applied by a SIMT kernel after the input FC; the learned table is part of the flat
parameter buffer.

The input block is the reference's general FCModel (model.py:16-44): optional nn.LayerNorm on the features, then any
number of Linear layers each followed by the activation (None / ReLU / Tanh / Sigmoid) and dropout.  With
`transformer=None` the model is that MLP plus the output head (the `*_mlp.json` configurations of the paper).
Autograd reaches `x` as well as the parameters: x.grad (in x's dtype and shape) comes from the CUDA backward, which
then also runs the first FC layer's input-gradient product; with every parameter frozen it computes no parameter
gradient at all.  In the default packed-row layout (include/allrank_b200.h: arb_set_pack_rows) items at or beyond their
slate's packed rows get 0 in `prepare_for_output` and in x.grad, and a gradient sent to their hidden rows is ignored --
the same contract as their score.  Double backward is not supported (it raises).
Attention runs on the fused kernels at every head width d_model / h from 1 to 256, for slates of up to 4096 items.  A
width that is not a multiple of 4 (d_model 144 with h = 8: 18 columns) runs on heads padded with zero columns to the
next multiple of 4 inside the CUDA scorer (DESIGN.md 4.15); the parameters and the state_dict keep the reference's
shapes.
Not supported (raise NotImplementedError rather than fall back): `fc_model=None`, other activation classes,
attention heads wider than 256 columns (d_model / h; raised when the parameters are first packed on the GPU) and
padded heads beyond 1024 columns in all (h * round_up(d_model / h, 4)); compute_dtype="bf16" at head widths other than
8, 16, 24 and 32.
"""
import contextlib
import copy
import ctypes

import torch
import torch.nn as nn

from . import _lib

_ACTS = {None: 0, "Tanh": 1, "Sigmoid": 2, "ReLU": 3}


class ScorerConfig(ctypes.Structure):
    _fields_ = [("n_features", ctypes.c_int32), ("d_model", ctypes.c_int32), ("n_layers", ctypes.c_int32),
                ("n_heads", ctypes.c_int32), ("d_ff", ctypes.c_int32), ("out_act", ctypes.c_int32),
                ("ln_eps", ctypes.c_float), ("dropout", ctypes.c_float), ("fc_dropout", ctypes.c_float),
                ("pe_mode", ctypes.c_int32), ("pe_rows", ctypes.c_int32), ("d_output", ctypes.c_int32),
                ("n_fc_layers", ctypes.c_int32), ("fc_sizes", ctypes.c_int32 * 8), ("fc_act", ctypes.c_int32),
                ("fc_input_norm", ctypes.c_int32), ("bf16", ctypes.c_int32)]


c_p, c_i, c_i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
_lib.register("arb_scorer_param_count", c_i64, [c_p])
_lib.register("arb_scorer_workspace_floats", c_i64, [c_p, c_i, c_i, c_i])
_lib.register("arb_scorer_backward_scratch_floats", c_i64, [c_p, c_i, c_i])
_lib.register("arb_scorer_forward", c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_i64, c_i, ctypes.c_uint64,
                                          c_p])
_lib.register("arb_scorer_backward", c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_i64, c_p, c_i64,
                                           ctypes.c_uint64, c_p])
_lib.register("arb_scorer_encode", c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_i64, c_i, ctypes.c_uint64,
                                         c_p])
_lib.register("arb_scorer_backward_ex_scratch_floats", c_i64, [c_p, c_i, c_i, c_i])
_lib.register("arb_scorer_backward_ex", c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_p, c_p, c_i64, c_p,
                                              c_i64, ctypes.c_uint64, c_p])
# the same calls with the dropout seed read from a device word (include/allrank_b200.h)
_lib.register("arb_scorer_forward_dseed", c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_i64, c_i, c_p, c_p])
_lib.register("arb_scorer_encode_dseed", c_i, [c_p, c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_i64, c_i, c_p, c_p])
_lib.register("arb_scorer_backward_ex_dseed", c_i, [c_p, c_p, c_p, c_p, c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_p, c_p,
                                                    c_i64, c_p, c_i64, c_p, c_p])


def _seed_arg(seed, device):
    """The C argument of a dropout seed: a host value, or the address of a one-element int64 tensor on `device`."""
    if not isinstance(seed, torch.Tensor):
        return ctypes.c_uint64(seed)
    if seed.device != device:
        raise ValueError(f"the dropout seed tensor is on {seed.device}, the batch on {device}")
    return _lib.ptr(seed)


# ------------------------------------------------------------------------------------------------ module tree
class _Norm(nn.Module):
    """Parameter holder for the reference's custom LayerNorm (transformer.py:59-81)."""

    def __init__(self, width):
        super().__init__()
        self.a_2 = nn.Parameter(torch.ones(width))
        self.b_2 = nn.Parameter(torch.zeros(width))


class _Sublayer(nn.Module):
    def __init__(self, width):
        super().__init__()
        self.norm = _Norm(width)


class _SelfAttn(nn.Module):
    def __init__(self, proto):
        super().__init__()
        self.linears = nn.ModuleList([_clone_linear(proto) for _ in range(4)])


class _FeedForward(nn.Module):
    def __init__(self, w1, w2):
        super().__init__()
        self.w_1 = _clone_linear(w1)
        self.w_2 = _clone_linear(w2)


class _EncoderLayer(nn.Module):
    def __init__(self, width, attn_proto, w1, w2):
        super().__init__()
        self.self_attn = _SelfAttn(attn_proto)
        self.feed_forward = _FeedForward(w1, w2)
        self.sublayer = nn.ModuleList([_Sublayer(width), _Sublayer(width)])


class _FixedPE(nn.Module):
    """Sinusoidal table + one zero padding row, a buffer named `pe` (positional.py:15-37)."""

    def __init__(self, width, max_len):
        super().__init__()
        import math
        pe = torch.zeros(max_len, width)
        position = torch.arange(0.0, max_len).unsqueeze(1)
        div_term = torch.exp(torch.arange(0.0, width, 2) * -(math.log(10000.0) / width))
        pe[:, 0::2] = torch.sin(position * div_term)
        pe[:, 1::2] = torch.cos(position * div_term)
        pe = torch.cat((pe, torch.zeros([1, width])))
        self.register_buffer("pe", pe)


class _LearnedPE(nn.Module):
    """nn.Embedding(max_len + 1, d, padding_idx=-1) named `pe` (positional.py:53-64)."""

    def __init__(self, width, max_len):
        super().__init__()
        self.pe = nn.Embedding(max_len + 1, width, padding_idx=-1)


class _Encoder(nn.Module):
    def __init__(self, n_layers, width, attn_proto, w1, w2, position=None):
        super().__init__()
        self.layers = nn.ModuleList([_EncoderLayer(width, attn_proto, w1, w2) for _ in range(n_layers)])
        self.norm = _Norm(width)
        self.position = position


class _InputFC(nn.Module):
    """Parameter holder with FCModel's attribute order (model.py:27-33): input_norm, then layers."""

    def __init__(self, linears, n_features, input_norm):
        super().__init__()
        self.input_norm = nn.LayerNorm(n_features) if input_norm else nn.Identity()
        self.layers = nn.ModuleList(linears)
        self.output_size = linears[-1].out_features


class _Head(nn.Module):
    def __init__(self, lin):
        super().__init__()
        self.w_1 = lin
        self.d_output = lin.out_features


def _clone_linear(proto):
    return copy.deepcopy(proto)   # like the reference's clones(): no RNG draw, clones share the prototype's init


# ------------------------------------------------------------------------------------------------ autograd glue
# `anchor` requires grad exactly when some parameter does (it stands for all of them: they are views of one flat buffer
# that the C backward fills); `x` is the caller's tensor, padded to the C layout inside the Function.
class _ScorerFn(torch.autograd.Function):
    """x -> scores (arb_scorer_forward / arb_scorer_backward_ex from d_scores)."""

    @staticmethod
    def forward(ctx, anchor, x, mask, model, indices):
        keep = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        xin = model._pad_features(x)
        seed, drop = model._call_seed()
        scores, ws = model._launch_forward(xin, mask, keep, seed, indices)
        if keep:
            ctx.model, ctx.ws, ctx.seed, ctx.drop, ctx.indices = model, ws, seed, drop, indices
            ctx.x_meta = (x.shape, x.dtype)
            ctx.save_for_backward(xin, mask, scores)
        return scores

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_scores):
        xin, mask, scores = ctx.saved_tensors
        dx = ctx.model._launch_backward(xin, mask, scores, d_scores.contiguous().float(), ctx.ws, ctx.seed, ctx.drop,
                                        ctx.indices, want_params=ctx.needs_input_grad[0],
                                        want_dx=ctx.needs_input_grad[1])
        ctx.ws = None
        return None, ctx.model._input_grad(dx, ctx.x_meta), None, None, None


class _EncodeFn(torch.autograd.Function):
    """x -> hidden [B,S,d_model] (arb_scorer_encode / arb_scorer_backward_ex from d_hidden)."""

    @staticmethod
    def forward(ctx, anchor, x, mask, model, indices):
        keep = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        xin = model._pad_features(x)
        seed, drop = model._call_seed()
        hidden, ws = model._launch_forward(xin, mask, keep, seed, indices, encode=True)
        if keep:
            ctx.model, ctx.ws, ctx.seed, ctx.drop, ctx.indices = model, ws, seed, drop, indices
            ctx.x_meta = (x.shape, x.dtype)
            ctx.save_for_backward(xin, mask)
        return hidden

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_hidden):
        xin, mask = ctx.saved_tensors
        dx = ctx.model._launch_backward(xin, mask, None, d_hidden.contiguous().float(), ctx.ws, ctx.seed, ctx.drop,
                                        ctx.indices, want_params=ctx.needs_input_grad[0],
                                        want_dx=ctx.needs_input_grad[1], from_hidden=True)
        ctx.ws = None
        return None, ctx.model._input_grad(dx, ctx.x_meta), None, None, None


class LTRModel(nn.Module):
    """CUDA scorer with the reference LTRModel's surface (model.py:47-92)."""

    def __init__(self, n_features, d_model, n_layers, n_heads, d_ff, dropout, output_activation, fc_dropout=0.0,
                 positional=None, d_output=1, fc_sizes=None, fc_activation=None, input_norm=False,
                 compute_dtype="tf32"):
        super().__init__()
        fc_sizes = [int(d_model)] if fc_sizes is None else [int(v) for v in fc_sizes]
        d_model = fc_sizes[-1]
        if not 1 <= len(fc_sizes) <= 8:
            raise NotImplementedError("fc_model.sizes must list 1 to 8 layers")
        if fc_activation not in _ACTS:
            raise NotImplementedError(f"fc_model.activation {fc_activation!r}: supported {sorted(map(str, _ACTS))}")
        if input_norm and n_features % 4:
            raise NotImplementedError("fc_model.input_norm needs n_features % 4 == 0 (no feature padding under the norm)")
        self.fc_sizes, self.fc_activation, self.input_norm_on = fc_sizes, fc_activation, bool(input_norm)
        self.d_output = int(d_output)
        if not 1 <= self.d_output <= 64:
            raise NotImplementedError("d_output must be in [1, 64]")
        if output_activation not in _ACTS:
            raise NotImplementedError(f"output activation {output_activation!r}: supported {sorted(map(str, _ACTS))}")
        self.n_features, self.d_model, self.n_layers = int(n_features), int(d_model), int(n_layers)
        self.n_heads, self.d_ff, self.dropout_p = int(n_heads), int(d_ff), float(dropout or 0.0)
        self.fc_dropout_p = float(fc_dropout or 0.0)
        self.output_activation = output_activation
        if n_layers > 0:
            assert d_model % n_heads == 0   # transformer.py:170
        # --- build in the reference's construction order so that a seeded init reproduces (model.py:139-150)
        dims = [int(n_features)] + fc_sizes
        self.input_layer = _InputFC([nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])], int(n_features), input_norm)
        if n_layers > 0:
            attn_proto = nn.Linear(d_model, d_model)
            w1 = nn.Linear(d_model, d_ff)
            w2 = nn.Linear(d_ff, d_model)
            position = None
            if positional is not None:                      # positional.py:80-94
                strategy, max_len = positional
                if strategy == "fixed":
                    position = _FixedPE(d_model, max_len)
                elif strategy == "learned":
                    position = _LearnedPE(d_model, max_len)
                else:
                    raise ValueError("Invalid positional encoding type: {}".format(strategy))
            self.encoder = _Encoder(n_layers, d_model, attn_proto, w1, w2, position)
        else:
            self.encoder = None
        self.output_layer = _Head(nn.Linear(d_model, self.d_output))
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        self._Fp = (self.n_features + 3) // 4 * 4
        self._cfg = ScorerConfig(self._Fp, self.d_model, self.n_layers, max(self.n_heads, 1), max(self.d_ff, 4),
                                 _ACTS[output_activation], 1e-6, self.dropout_p, self.fc_dropout_p, 0, 0, self.d_output,
                                 len(fc_sizes), (ctypes.c_int32 * 8)(*fc_sizes), _ACTS[fc_activation],
                                 1 if input_norm else 0, 0)
        self.compute_dtype = compute_dtype
        pos = self.encoder.position if self.encoder is not None else None
        if pos is not None:
            self._cfg.pe_mode = 1 if isinstance(pos, _FixedPE) else 2
            self._cfg.pe_rows = (pos.pe if isinstance(pos, _FixedPE) else pos.pe.weight).shape[0]
        self._flat = None
        self._flat_grad = None
        self._views = None
        self._anchor = None
        self._dropout_seed = None      # the seed tensor of dropout_seed_from(), or None: seeds drawn on the host

    # ---- arithmetic of the encoder's matrix products ------------------------------------------------
    @property
    def compute_dtype(self):
        """"tf32" (default): tensor-core tf32 products on fp32 data.  "bf16": every encoder linear is a tensor-core
        product of bfloat16 operands with fp32 accumulation -- bfloat16 shadow of the fp32 master weights, bfloat16
        LayerNorm outputs / attention context / FFN hidden layer and product-only gradients; residual stream,
        normalisation statistics, softmax, attention scores, head, loss and parameter gradients stay fp32
        (BASELINE config 3; include/allrank_b200.h: arb_scorer_config.bf16)."""
        return "bf16" if self._cfg.bf16 else "tf32"

    @compute_dtype.setter
    def compute_dtype(self, value):
        if value not in ("tf32", "bf16"):
            raise ValueError("compute_dtype must be 'tf32' or 'bf16'")
        if value == "bf16" and self.n_layers > 0 and (self.d_model % 8 or self.d_ff % 8 or
                                                      self.d_model // max(self.n_heads, 1) not in (8, 16, 24, 32)):
            raise NotImplementedError("bf16 mode needs d_model, d_ff multiples of 8 and a head width of 8, 16, 24 or 32 "
                                      "(a bfloat16 head must span a multiple of 16 bytes)")
        self._cfg.bf16 = 1 if value == "bf16" else 0

    # ---- flat parameter storage -------------------------------------------------------------------
    def _ordered(self):
        """(parameter, flat shape) in the C ABI's layout order (include/allrank_b200.h)."""
        Fp = self._Fp
        out = []
        for i, lin in enumerate(self.input_layer.layers):   # layer 0's weight rows are padded to Fp features
            out += [(lin.weight, (lin.out_features, Fp) if i == 0 else None), (lin.bias, None)]
        if self.input_norm_on:
            out += [(self.input_layer.input_norm.weight, None), (self.input_layer.input_norm.bias, None)]
        if self.encoder is not None:
            out += [(None, "align8")]      # the encoder section starts on a 32-byte boundary (include/allrank_b200.h)
        if self.encoder is not None:
            for lyr in self.encoder.layers:
                lin = lyr.self_attn.linears
                out += [(lin[0].weight, None), (lin[1].weight, None), (lin[2].weight, None),
                        (lin[0].bias, None), (lin[1].bias, None), (lin[2].bias, None),
                        (lin[3].weight, None), (lin[3].bias, None),
                        (lyr.feed_forward.w_1.weight, None), (lyr.feed_forward.w_1.bias, None),
                        (lyr.feed_forward.w_2.weight, None), (lyr.feed_forward.w_2.bias, None),
                        (lyr.sublayer[0].norm.a_2, None), (lyr.sublayer[0].norm.b_2, None),
                        (lyr.sublayer[1].norm.a_2, None), (lyr.sublayer[1].norm.b_2, None)]
            out += [(self.encoder.norm.a_2, None), (self.encoder.norm.b_2, None)]
        out += [(self.output_layer.w_1.weight, None), (self.output_layer.w_1.bias, None)]
        if self.encoder is not None and isinstance(self.encoder.position, _LearnedPE):
            out += [(self.encoder.position.pe.weight, "align4")]
        return out

    def _view_of(self, flat, offset, p, flat_shape):
        if flat_shape is None or tuple(flat_shape) == tuple(p.shape):
            return flat[offset:offset + p.numel()].view(p.shape), p.numel()
        n = 1
        for s in flat_shape:
            n *= s
        full = flat[offset:offset + n].view(flat_shape)
        return full[..., :p.shape[-1]], n

    def _pack(self, device):
        total = int(_lib.lib().arb_scorer_param_count(ctypes.byref(self._cfg)))
        if total <= 0:
            raise NotImplementedError("unsupported scorer shape: " + _lib.lib().arb_last_error().decode())
        flat = torch.zeros(total, dtype=torch.float32, device=device)
        grad = torch.zeros(total, dtype=torch.float32, device=device)
        views, off = [], 0
        for p, shape in self._ordered():
            if shape == "align8":          # padding only
                off = (off + 7) // 8 * 8
                continue
            if shape == "align4":          # the learned positional table starts on a 16-byte boundary
                off = (off + 3) // 4 * 4
                shape = None
            v, n = self._view_of(flat, off, p, shape)
            gv, _ = self._view_of(grad, off, p, shape)
            with torch.no_grad():
                v.copy_(p.detach().to(device=device, dtype=torch.float32))
            old_grad = p.grad
            p.data = v
            if old_grad is not None:
                gv.copy_(old_grad.to(device))
                p.grad = gv
            views.append((p, v, gv))
            off += n
        assert off == total, (off, total)
        self._flat, self._flat_grad, self._views = flat, grad, views
        self._anchor = torch.zeros(1, device=device, requires_grad=True)

    def _ensure_packed(self, device):
        if self._flat is None or self._flat.device != device:
            self._pack(device)
            return
        for p, v, _ in self._views:
            if p.data_ptr() != v.data_ptr() or p.device != device:
                self._pack(device)      # e.g. after model.to(...) replaced the parameter storage
                return

    @property
    def flat_parameters(self):
        return self._flat

    @property
    def flat_gradients(self):
        return self._flat_grad

    # ---- launches -----------------------------------------------------------------------------------
    def _prep_indices(self, indices, device):
        if self._cfg.pe_mode == 0:
            return None
        if indices is None:
            raise ValueError("this model has a positional encoding: `indices` is required")
        return indices.detach().to(device=device, dtype=torch.int64).contiguous()

    def _pe_table(self, device):
        """The fixed sinusoidal table on the device of the batch (a model that was never moved with .to(device) keeps
        the buffer on the host; the parameters are moved lazily by _ensure_packed, so the table must follow)."""
        pos = self.encoder.position if self.encoder is not None else None
        if not isinstance(pos, _FixedPE):
            return None
        if pos.pe.device == device and pos.pe.dtype == torch.float32 and pos.pe.is_contiguous():
            return pos.pe
        cached = getattr(self, "_pe_dev", None)
        if cached is None or cached[0].device != device or cached[1] != pos.pe._version:
            cached = (pos.pe.detach().to(device=device, dtype=torch.float32).contiguous(), pos.pe._version)
            self._pe_dev = cached
        return cached[0]

    def _prep_inputs(self, x, mask):
        _lib.require_cuda(x, mask)
        if x.dim() != 3 or x.shape[-1] != self.n_features:
            raise ValueError(f"x must be [batch, slate, {self.n_features}]")
        if mask.shape != x.shape[:2]:
            raise ValueError("mask must be [batch, slate]")
        return mask.detach().to(torch.uint8).contiguous()

    def _pad_features(self, x):
        """The C layout of x: contiguous fp32 [B, S, _Fp] (features zero-padded to a multiple of 4)."""
        x = x.detach().float()
        if self._Fp != self.n_features:
            x = torch.nn.functional.pad(x, (0, self._Fp - self.n_features))
        return x.contiguous()

    def _input_grad(self, dx, x_meta):
        """d loss / d x in the caller's shape and dtype (the padded feature columns dropped), or None."""
        if dx is None:
            return None
        shape, dtype = x_meta
        return dx[..., :self.n_features].to(dtype).reshape(shape)

    def _draw_seed(self):
        """Per-call dropout seed from torch's global CPU generator (so torch.manual_seed makes runs repeatable)."""
        if self.training and (self.dropout_p > 0.0 or self.fc_dropout_p > 0.0):
            return int(torch.randint(0, 2 ** 62, (1,)).item())
        return 0

    @contextlib.contextmanager
    def dropout_seed_from(self, seed):
        """Inside this context, train-mode calls with dropout take their per-call dropout seed from `seed` -- a
        one-element int64 tensor on the model's CUDA device -- instead of drawing it on the host (_draw_seed).

        Each call snapshots the tensor with a device-side clone() and the kernels read that snapshot when they execute,
        so a CUDA graph captured here applies new masks whenever the tensor changes between replays (GraphedTrainStep
        does that).  The backward reads the forward's snapshot: the tensor may be advanced between a step's forward and
        its backward.  With the same seed value, the masks are bit-identical to those of a host-seeded call (the
        tensor's 64 bits are read as an unsigned integer)."""
        dev = next(self.parameters()).device
        if not (isinstance(seed, torch.Tensor) and seed.is_cuda and seed.device == dev and seed.dtype == torch.int64
                and seed.numel() == 1):
            raise ValueError("dropout_seed_from: the seed must be a one-element int64 CUDA tensor on the model's "
                             f"device ({dev})")
        prev, self._dropout_seed = self._dropout_seed, seed
        try:
            yield
        finally:
            self._dropout_seed = prev

    def _call_seed(self):
        """(seed, dropout on) for one call: an int from _draw_seed() (0 without dropout), or inside dropout_seed_from()
        with dropout on, a device-side snapshot of the seed tensor."""
        if self._dropout_seed is not None and self.training and (self.dropout_p > 0.0 or self.fc_dropout_p > 0.0):
            return self._dropout_seed.clone(), True
        seed = self._draw_seed()
        return seed, seed != 0

    def _launch_forward(self, x, mask, keep_for_backward, seed=0, indices=None, encode=False):
        """scores (encode: the encoder output [B,S,d_model]) and the workspace kept for backward (or None).
        seed: an int, or a one-element int64 device tensor read by the kernels (the *_dseed entry points)."""
        training = keep_for_backward
        B, S = x.shape[0], x.shape[1]
        dev = x.device
        cfg = ctypes.byref(self._cfg)
        # dropout is applied iff the module is in train() mode, like nn.Dropout; `training` only selects whether
        # activations are kept for backward.  (Set before the workspace query: the layout depends on it -- a call
        # without dropout may run over packed rows.)
        self._cfg.dropout = self.dropout_p if self.training else 0.0
        self._cfg.fc_dropout = self.fc_dropout_p if self.training else 0.0
        n_ws = int(_lib.lib().arb_scorer_workspace_floats(cfg, B, S, 1 if training else 0))
        ws = torch.empty(n_ws, dtype=torch.float32, device=dev)
        if encode:
            shape = (B, S, self.d_model)
        else:
            shape = (B, S) if self.d_output == 1 else (B, S, self.d_output)   # squeeze(dim=2) is a no-op for n > 1 (model.py:117)
        scores = torch.empty(shape, dtype=torch.float32, device=dev)
        name = "arb_scorer_encode" if encode else "arb_scorer_forward"
        if isinstance(seed, torch.Tensor):
            name += "_dseed"
        with torch.cuda.device(dev):
            table = self._pe_table(dev)
            rc = getattr(_lib.lib(), name)(cfg, _lib.ptr(self._flat), _lib.ptr(x), _lib.ptr(mask),
                                           _lib.ptr(indices), _lib.ptr(table), B, S,
                                           _lib.ptr(scores), _lib.ptr(ws), n_ws, 1 if training else 0,
                                           _seed_arg(seed, dev), _lib.stream_ptr(dev))
        _lib.check(rc, name)
        return scores, (ws if training else None)

    def _launch_backward(self, x, mask, scores, d_out, ws, seed=0, dropout=False, indices=None, want_params=True,
                         want_dx=False, from_hidden=False):
        """Accumulates the parameter gradients (want_params) and returns d loss / d x [B,S,_Fp] (want_dx, else None).
        d_out is d loss / d scores, or d loss / d hidden (from_hidden).  seed, dropout: what _call_seed() gave the
        forward."""
        B, S = x.shape[0], x.shape[1]
        dev = x.device
        cfg = ctypes.byref(self._cfg)
        fresh = want_params and any(p.grad is None or p.grad.data_ptr() != gv.data_ptr() for p, _, gv in self._views)
        if fresh:                      # after optimizer.zero_grad(set_to_none=True): start from zero
            self._flat_grad.zero_()
        self._cfg.dropout = self.dropout_p if dropout else 0.0          # same mask configuration as the forward call
        self._cfg.fc_dropout = self.fc_dropout_p if dropout else 0.0
        n_sc = int(_lib.lib().arb_scorer_backward_ex_scratch_floats(cfg, B, S, 1 if want_dx else 0))
        scratch = torch.empty(n_sc, dtype=torch.float32, device=dev)
        dx = torch.empty((B, S, self._Fp), dtype=torch.float32, device=dev) if want_dx else None
        name = "arb_scorer_backward_ex_dseed" if isinstance(seed, torch.Tensor) else "arb_scorer_backward_ex"
        with torch.cuda.device(dev):
            rc = getattr(_lib.lib(), name)(cfg, _lib.ptr(self._flat), _lib.ptr(x), _lib.ptr(mask),
                                           _lib.ptr(indices), B, S, _lib.ptr(scores),
                                           None if from_hidden else _lib.ptr(d_out),
                                           _lib.ptr(d_out) if from_hidden else None,
                                           _lib.ptr(self._flat_grad) if want_params else None, _lib.ptr(dx),
                                           _lib.ptr(ws), ws.numel(), _lib.ptr(scratch), n_sc,
                                           _seed_arg(seed, dev), _lib.stream_ptr(dev))
        _lib.check(rc, name)
        if fresh:
            for p, _, gv in self._views:
                if p.requires_grad:
                    p.grad = gv
        return dx

    def _replicate_for_data_parallel(self):
        raise RuntimeError(
            "allrank_b200.LTRModel cannot be replicated by nn.DataParallel (its parameters are views of one flat "
            "device buffer): run one process per GPU (torchrun) with allrank_b200.ddp.FlatDDP, or restrict "
            "CUDA_VISIBLE_DEVICES to one device; allrank_b200.integration.patch_allrank() neutralises the "
            "CustomDataParallel wrap of allrank/main.py:76-78")

    # ---- public surface (model.py:62-92) ---------------------------------------------------------------
    def _call(self, fn_cls, x, mask, indices):
        """fn_cls (_ScorerFn / _EncodeFn) through autograd when a gradient may be wanted, else a plain launch."""
        m = self._prep_inputs(x, mask)
        idx = self._prep_indices(indices, x.device)
        self._ensure_packed(x.device)
        params = any(p.requires_grad for p in self.parameters())
        if torch.is_grad_enabled() and (params or x.requires_grad):
            anchor = self._anchor if params else self._anchor.detach()
            return fn_cls.apply(anchor, x, m, self, idx)
        out, _ = self._launch_forward(self._pad_features(x), m, False, self._call_seed()[0], idx,
                                      encode=fn_cls is _EncodeFn)
        return out

    def prepare_for_output(self, x, mask, indices=None):
        """The encoder output [B, S, d_model] (model.py:62-70): the final LayerNorm's output, or with
        `transformer=None` the FC block's output.  Dropout follows train() / eval() as in forward()."""
        return self._call(_EncodeFn, x, mask, indices)

    def forward(self, x, mask, indices=None):
        return self._call(_ScorerFn, x, mask, indices)

    def score(self, x, mask, indices=None):
        out = self.forward(x, mask, indices)
        return out.sum(-1) if self.d_output > 1 else out       # model.py:119-128


def _get(cfg, name, default=None):
    if cfg is None:
        return default
    if isinstance(cfg, dict):
        return cfg.get(name, default)
    return getattr(cfg, name, default)


def make_model(fc_model, transformer, post_model, n_features, compute_dtype="tf32"):
    """Same arguments as allrank.models.model.make_model (model.py:131-151): `fc_model` dict
    {sizes, input_norm, activation, dropout}, `transformer` config object/dict {N, d_ff, h, dropout,
    positional_encoding} or None, `post_model` dict {d_output, output_activation}.
    Extension (after the reference's parameters): compute_dtype "tf32" | "bf16", see LTRModel.compute_dtype."""
    if not fc_model:
        raise NotImplementedError("allrank_b200 needs an input FC block (fc_model.sizes = [d_model])")
    sizes = [int(v) for v in _get(fc_model, "sizes")]     # (the reference mutates the caller's list, model.py:25; we do not)
    d_model = sizes[-1]
    if transformer:
        pe_cfg = _get(transformer, "positional_encoding", None)
        positional = None if pe_cfg is None else (_get(pe_cfg, "strategy"), int(_get(pe_cfg, "max_indices")))
        n_layers, heads, d_ff = int(_get(transformer, "N")), int(_get(transformer, "h")), int(_get(transformer, "d_ff"))
        dropout = float(_get(transformer, "dropout", 0.0) or 0.0)
    else:
        n_layers, heads, d_ff, dropout, positional = 0, 1, 4, 0.0, None
    return LTRModel(n_features, d_model, n_layers, heads, d_ff, dropout, _get(post_model, "output_activation", None),
                    fc_dropout=float(_get(fc_model, "dropout", 0.0) or 0.0), positional=positional,
                    d_output=int(_get(post_model, "d_output", 1)), fc_sizes=sizes,
                    fc_activation=_get(fc_model, "activation", None), input_norm=bool(_get(fc_model, "input_norm", False)),
                    compute_dtype=compute_dtype)
