"""One training step -- scorer forward, loss, backward, optimiser -- captured into a CUDA graph and replayed.

At allRank's own batch size (64 slates) a step is some fifty kernels of 5-10 us each and the host, not the GPU, sets the
pace: the Python / ctypes launch path costs more than the kernels run.  The C side of allrank_b200 never synchronises
and its only allocations are stream-ordered (DESIGN.md section 2: they become memory nodes owned by the graph), so the
whole step captures into one graph; replaying it costs one launch.

    step = GraphedTrainStep(model, loss_fn, optimizer, x, y)     # x [B,S,F], y [B,S] on the device: shapes are fixed
    for xb, yb in loader:
        loss = step(xb, yb)            # copies the batch into the graph's static inputs, replays, returns the loss tensor

Restrictions (checked): the model must not use dropout in train() mode (its per-call seed is drawn on the host) and the
optimiser must keep its step counter on the device -- allrank_b200.optim.FlatAdam(capturable=True) or
torch.optim.Adam(capturable=True).  The reference's training loop (allrank/training/train_utils.py:18-29) is the
sequence captured here: loss_batch = loss_func(model(xb, mask, indices), yb); loss.backward(); opt.step(); opt.zero_grad().
"""
import torch

from .losses import PADDED_Y_VALUE


class GraphedTrainStep:
    def __init__(self, model, loss_fn, optimizer, x, y, loss_kwargs=None, indices=None, warmup=3):
        if not (x.is_cuda and y.is_cuda):
            raise ValueError("GraphedTrainStep: inputs must be CUDA tensors")
        if model.training and (getattr(model, "dropout_p", 0.0) > 0.0 or getattr(model, "fc_dropout_p", 0.0) > 0.0):
            raise ValueError("GraphedTrainStep: dropout draws its per-call seed on the host and cannot be captured")
        groups = getattr(optimizer, "param_groups", None)
        capturable = bool(getattr(optimizer, "capturable", False)) or \
            (bool(groups) and all(g.get("capturable", False) for g in groups))
        if not capturable:
            raise ValueError("GraphedTrainStep: the optimiser must be capturable (device-side step counter)")
        self.model, self.loss_fn, self.optimizer = model, loss_fn, optimizer
        self.kw = dict(loss_kwargs or {})
        self.x, self.y = x.clone(), y.clone()
        self.indices = None if indices is None else indices.clone()
        side = torch.cuda.Stream(device=x.device)
        side.wait_stream(torch.cuda.current_stream(x.device))
        with torch.cuda.stream(side):            # warm-up off the default stream (allocator pools, lazy packing)
            for _ in range(max(1, warmup)):
                self._one()
        torch.cuda.current_stream(x.device).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = self._one()

    def _one(self):
        mask = self.y == PADDED_Y_VALUE                       # train_utils.py:19
        loss = self.loss_fn(self.model(self.x, mask, self.indices), self.y, **self.kw)
        self.optimizer.zero_grad()
        loss.backward()
        self.optimizer.step()
        return loss.detach()

    def replay(self):
        """Replay on the batch the static inputs already hold (self.x / self.y); returns the loss tensor."""
        self.graph.replay()
        return self.loss

    def __call__(self, x, y, indices=None):
        self.x.copy_(x, non_blocking=True)
        self.y.copy_(y, non_blocking=True)
        if self.indices is not None and indices is not None:
            self.indices.copy_(indices, non_blocking=True)
        self.graph.replay()
        return self.loss
