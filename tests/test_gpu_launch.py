"""A kernel whose dynamic shared memory crosses the 48 KB default limit between calls of one process: the launch helper
raises the kernel's limit the first time a launch needs more and remembers it per device, so smaller and larger
launches of the same kernel work in any order and compute what they compute alone."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# listMLE's dynamic shared memory is next_pow2(S) * 8 + S * 16 + 1088 bytes: 7 KB at S = 240 (below the default
# limit), 96 KB at S = 4000 and 190 KB at S = 8000 (the limit must be raised a second time)
SIZES = [240, 4000, 8000, 240, 4000]


def _listmle(fn, yp, yt, perm):
    p = yp.clone().requires_grad_(True)
    val = fn(p, yt, perm=perm)
    val.backward()
    return val.detach(), p.grad


def test_listmle_below_and_above_the_default_shared_memory_limit():
    from allrank_b200 import losses
    from oracle import losses_ref
    seen = {}
    for S in SIZES:
        g = torch.Generator().manual_seed(S)
        yp = torch.randn(4, S, generator=g)
        yt = torch.stack([torch.randperm(S, generator=g) for _ in range(4)]).float()   # tie-free labels
        perm = torch.randperm(S, generator=g)
        val, grad = _listmle(losses.listMLE, yp.cuda(), yt.cuda(), perm)
        ref, gref = _listmle(losses_ref.listMLE, yp.double(), yt.double(), perm)
        assert abs(val.item() - ref.item()) <= 1e-4 * abs(ref.item()), (S, val.item(), ref.item())
        err = (grad.cpu().double() - gref).abs().max().item()
        assert err <= 1e-4 * gref.abs().max().item(), (S, err)
        if S in seen:     # the same call after a larger launch of the kernel: bit-identical
            assert torch.equal(val, seen[S][0]) and torch.equal(grad, seen[S][1]), S
        seen.setdefault(S, (val, grad))
