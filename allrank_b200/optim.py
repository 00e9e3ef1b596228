"""FlatAdam: torch.optim.Adam semantics as ONE kernel launch over the scorer's flat parameter buffer.

The reference builds its optimiser by name from the config (allrank/main.py:82, `getattr(optim, name)`); any
torch optimiser works unchanged on allrank_b200 models because their parameters are ordinary nn.Parameters.
FlatAdam is the native alternative for the flat storage: it steps every parameter of the model with one
128-bit-vectorised launch (csrc/optim.cu), and optionally folds the 1/world_size of a sum all-reduce in.
"""
import ctypes

import torch

from . import _lib

c_p, c_i, c_f = ctypes.c_void_p, ctypes.c_int32, ctypes.c_float
_lib.register("arb_adam_step", c_i, [c_p, c_p, c_p, c_p, ctypes.c_int64, c_f, c_f, c_f, c_f, c_f, c_i, c_f, c_p])
_lib.register("arb_adam_step_dev", c_i, [c_p, c_p, c_p, c_p, ctypes.c_int64, c_f, c_f, c_f, c_f, c_f, c_p, c_f, c_p])


class FlatAdam:
    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, capturable=False):
        """capturable=True keeps the step counter on the device (like torch.optim.Adam(capturable=True)), so that a
        step can be captured into a CUDA graph and replayed (allrank_b200.graph.GraphedTrainStep)."""
        self.model = model
        self.lr, self.betas, self.eps, self.weight_decay = float(lr), tuple(betas), float(eps), float(weight_decay)
        self.capturable = bool(capturable)
        self._dev_state = None
        self.step_count = 0
        self.exp_avg = None
        self.exp_avg_sq = None

    def _state(self):
        flat = self.model.flat_parameters
        if flat is None:
            raise RuntimeError("FlatAdam: run a forward pass first (the model packs its parameters lazily)")
        if self.exp_avg is None or self.exp_avg.data_ptr() == 0 or self.exp_avg.shape != flat.shape \
                or self.exp_avg.device != flat.device:
            self.exp_avg = torch.zeros_like(flat)
            self.exp_avg_sq = torch.zeros_like(flat)
        return flat

    def step(self, grad_scale=1.0):
        flat = self._state()
        grad = self.model.flat_gradients
        self.step_count += 1
        if self.capturable:
            if self._dev_state is None or self._dev_state.device != flat.device:
                self._dev_state = torch.zeros(4, dtype=torch.float32, device=flat.device)
                self._dev_state[0] = float(self.step_count - 1)
            with torch.cuda.device(flat.device):
                rc = _lib.lib().arb_adam_step_dev(_lib.ptr(flat), _lib.ptr(grad), _lib.ptr(self.exp_avg),
                                                  _lib.ptr(self.exp_avg_sq), flat.numel(), self.lr, self.betas[0],
                                                  self.betas[1], self.eps, self.weight_decay,
                                                  _lib.ptr(self._dev_state), float(grad_scale),
                                                  _lib.stream_ptr(flat.device))
            _lib.check(rc, "arb_adam_step_dev")
            return
        with torch.cuda.device(flat.device):
            rc = _lib.lib().arb_adam_step(_lib.ptr(flat), _lib.ptr(grad), _lib.ptr(self.exp_avg),
                                          _lib.ptr(self.exp_avg_sq), flat.numel(), self.lr, self.betas[0],
                                          self.betas[1], self.eps, self.weight_decay, self.step_count,
                                          float(grad_scale), _lib.stream_ptr(flat.device))
        _lib.check(rc, "arb_adam_step")

    def zero_grad(self, set_to_none=False):
        """Zero the flat gradient buffer with one memset (the views the parameters hold stay attached)."""
        if self.model.flat_gradients is not None:
            self.model.flat_gradients.zero_()
