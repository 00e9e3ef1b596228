"""Data-parallel training over slates: one process per GPU, ONE NCCL all-reduce of the flat gradient buffer.

The reference's only multi-GPU mechanism is single-process nn.DataParallel (allrank/main.py:76-78,
allrank/models/model_utils.py:40-53).  Slates are independent (SURVEY.md 8e), so the native equivalent
shards the batch axis across ranks and sums gradients with a single `all_reduce` over NVLink / NVSwitch:
the model's parameters are views of one flat buffer, so there is exactly one bucket (1.66 MB for the
N=2,d=128 model, 12.8 MB for N=4,d=256) -- latency-bound, no bucketing logic needed.

Semantics (parity definition, SURVEY.md 8e): W ranks x per-rank batch b reproduce the single-process gradient
of batch W*b
  * mean-over-batch losses (listNet, listMLE, approxNDCG, ...): `average=True` when every rank holds the same number
    of slates, otherwise `local_weight` = the rank's slate count (weighted mean);
  * neuralNDCG / neuralNDCG_transposed average over the slates whose ideal DCG is non-zero
    (allrank/models/losses/neuralNDCG.py:62-69): the numerator AND the count are global, so the rank's gradient is
    weighted by its own count of such slates -- `local_weight=loss_weight("neuralNDCG", y_true)`;
  * lambdaLoss(reduction="sum") and the other pair-sum losses: `average=False` (gradients add).
With `local_weight` the exchange is one scalar all-reduce of the weights followed by the usual single all-reduce of
the flat gradient.   Works with the gloo backend on CPU tensors too (tests).
"""
import torch
import torch.distributed as dist

PADDED_Y_VALUE = -1


def loss_weight(loss_name, y_true, padded_value_indicator=PADDED_Y_VALUE):
    """The number of per-slate terms the named loss averages over on this rank (a 0-dim tensor on y_true's device):
    slates with a non-zero ideal DCG for neuralNDCG* (idcg != 0 <=> some real item has a positive label, for both
    gain functions), the batch size for the mean-over-batch losses; None for sum-reduced losses."""
    if loss_name in ("neuralNDCG", "neuralNDCG_transposed"):
        real = y_true != padded_value_indicator
        return ((y_true > 0) & real).any(dim=1).sum().to(torch.float32)
    if loss_name in ("lambdaLoss",):
        return None
    return torch.tensor(float(y_true.shape[0]), device=y_true.device)


def broadcast_parameters(params_flat, src=0, group=None):
    dist.broadcast(params_flat, src=src, group=group)


def all_reduce_gradients(grad_flat, average=True, group=None, async_op=False):
    """Sum (and optionally average) one flat gradient buffer across ranks.  Returns the work handle if async."""
    work = dist.all_reduce(grad_flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
    if average and not async_op:
        grad_flat.div_(dist.get_world_size(group))
    return work


class FlatDDP:
    """Thin wrapper: keeps rank replicas in sync and reduces `model.flat_gradients` after backward.

        ddp = FlatDDP(model)            # broadcasts rank 0's parameters (after the first packing)
        loss = loss_fn(model(x, mask, idx), y); loss.backward()
        ddp.reduce_gradients()          # one NCCL all-reduce
        optimiser.step()
    """

    def __init__(self, model, average=True, group=None):
        self.model, self.average, self.group = model, average, group
        self._synced = False

    def sync_parameters(self):
        flat = self.model.flat_parameters
        if flat is None:
            raise RuntimeError("FlatDDP: run a forward pass (or model._ensure_packed(device)) first")
        broadcast_parameters(flat, 0, self.group)
        self._synced = True

    def reduce_gradients(self, fold_average_into_optimizer=False, local_weight=None):
        """All-reduce the flat gradient.  With fold_average_into_optimizer=True the 1/W is left to the optimiser
        (FlatAdam.step(grad_scale=1/W)) so the reduce is a pure sum and no extra pass over the buffer is made.
        `local_weight` (0-dim tensor, see loss_weight): global gradient = sum_r w_r g_r / sum_r w_r."""
        if not self._synced:
            self.sync_parameters()
        grad = self.model.flat_gradients
        if local_weight is not None:
            w = local_weight.detach().to(device=grad.device, dtype=torch.float32).reshape(1).clone()
            total = w.clone()
            dist.all_reduce(total, op=dist.ReduceOp.SUM, group=self.group)
            grad.mul_(w / torch.clamp(total, min=1e-30))       # a rank without any term contributes nothing
            all_reduce_gradients(grad, average=False, group=self.group)
            return 1.0
        all_reduce_gradients(grad, average=self.average and not fold_average_into_optimizer, group=self.group)
        world = dist.get_world_size(self.group)
        return (1.0 / world) if (self.average and fold_average_into_optimizer) else 1.0
