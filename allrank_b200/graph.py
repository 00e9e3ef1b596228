"""One training step -- scorer forward, loss, backward, optimiser -- captured into a CUDA graph and replayed.

At allRank's own batch size (64 slates) a step is some fifty kernels of 5-10 us each and the host, not the GPU, sets the
pace: the Python / ctypes launch path costs more than the kernels run.  The C side of allrank_b200 never synchronises
and its only allocations are stream-ordered (DESIGN.md section 2: they become memory nodes owned by the graph), so the
whole step captures into one graph; replaying it costs one launch.

    step = GraphedTrainStep(model, loss_fn, optimizer, x, y)     # x [B,S,F], y [B,S] on the device: shapes are fixed
    for xb, yb in loader:
        loss = step(xb, yb)            # copies the batch into the graph's static inputs, replays, returns the loss tensor

Dropout.  A model that uses dropout in train() mode needs `dropout_seed=<int>`.  The per-call dropout seed then lives
in a device tensor, `step.dropout_seed`: the captured step first adds 1 to it and runs the model under
LTRModel.dropout_seed_from(step.dropout_seed), so the kernels read the seed when they execute.  After construction the
tensor holds `dropout_seed`, so replay k (1-based) uses the call seed dropout_seed + k and applies exactly the masks of
an eager step whose seed LTRModel._draw_seed() returned as dropout_seed + k.  Rewind or reseed it with
`step.dropout_seed.fill_(s)`.  Without `dropout_seed`, a model with dropout is refused.  What a graph still freezes:
anything else the step draws on the host -- listMLE's column permutation (torch.randperm, losses.listMLE) is drawn once
at capture and every replay reuses it.

Other restrictions (checked): the optimiser must keep its step counter on the device --
allrank_b200.optim.FlatAdam(capturable=True) or torch.optim.Adam(capturable=True).  The reference's training loop
(allrank/training/train_utils.py:18-29) is the sequence captured here: loss_batch = loss_func(model(xb, mask, indices),
yb); loss.backward(); opt.step(); opt.zero_grad().
"""
import contextlib

import torch

from .losses import PADDED_Y_VALUE


class GraphedTrainStep:
    def __init__(self, model, loss_fn, optimizer, x, y, loss_kwargs=None, indices=None, warmup=3, dropout_seed=None):
        if not (x.is_cuda and y.is_cuda):
            raise ValueError("GraphedTrainStep: inputs must be CUDA tensors")
        if dropout_seed is not None and (isinstance(dropout_seed, bool) or not isinstance(dropout_seed, int)
                                         or not -2 ** 63 <= dropout_seed < 2 ** 63):
            raise ValueError("GraphedTrainStep: dropout_seed must be an int (64-bit)")
        dropout = model.training and (getattr(model, "dropout_p", 0.0) > 0.0 or getattr(model, "fc_dropout_p", 0.0) > 0.0)
        if dropout and dropout_seed is None:
            raise ValueError("GraphedTrainStep: the model uses dropout: pass dropout_seed=<int> so that every replay "
                             "draws new masks (a host-drawn seed would be frozen into the graph)")
        groups = getattr(optimizer, "param_groups", None)
        capturable = bool(getattr(optimizer, "capturable", False)) or \
            (bool(groups) and all(g.get("capturable", False) for g in groups))
        if not capturable:
            raise ValueError("GraphedTrainStep: the optimiser must be capturable (device-side step counter)")
        self.model, self.loss_fn, self.optimizer = model, loss_fn, optimizer
        self.kw = dict(loss_kwargs or {})
        self.x, self.y = x.clone(), y.clone()
        self.indices = None if indices is None else indices.clone()
        self.dropout_seed = None if dropout_seed is None else \
            torch.tensor([dropout_seed], dtype=torch.int64, device=x.device)
        side = torch.cuda.Stream(device=x.device)
        side.wait_stream(torch.cuda.current_stream(x.device))
        with torch.cuda.stream(side):            # warm-up off the default stream (allocator pools, lazy packing)
            for _ in range(max(1, warmup)):
                self._one()
        torch.cuda.current_stream(x.device).wait_stream(side)
        if self.dropout_seed is not None:
            self.dropout_seed.fill_(dropout_seed)   # (the warm-up advanced it) replay k uses dropout_seed + k
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss = self._one()

    def _one(self):
        seeded = contextlib.nullcontext()
        if self.dropout_seed is not None:
            self.dropout_seed.add_(1)
            seeded = self.model.dropout_seed_from(self.dropout_seed)
        with seeded:
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
