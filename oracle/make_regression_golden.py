"""TEST INFRASTRUCTURE ONLY -- stores what the verbatim reference L1Loss / L2Loss (bm/losses.py:11-26, plain PyTorch
autograd) compute, so that tests/test_regression_loss_cpu.py can hold the drop-in losses to them wherever the tests run (the
reference tree is needed only to regenerate them).

    python oracle/make_regression_golden.py       # writes tests/golden/regression_*.npz

Each file holds one case's inputs (`est`, `out`, `mask`; `limit` > 0: the losses take est[..., limit:] and the same crop
of out and mask, as the encode task does, bm/solver.py:299-302) and, for kind in (l1, l2), `<kind>.loss`, `<kind>.d_est`
and `<kind>.d_out`: the gradients of the loss with respect to the full `est` and `out` tensors.

  regression_ragged_mask    [B, 1, T] mask with runs of False (task.mask_loss)
  regression_full_mask      a random [B, C, T] mask
  regression_all_true       the default all-True [B, 1, T] mask
  regression_all_false      no True entry: the loss is NaN and both gradients are zero
  regression_time_crop      est[..., limit:] at an odd element offset, with a ragged [B, 1, T] mask
  regression_ties           est == out on about a third of the entries (sign(0) = 0 in the L1 gradient)
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_loader  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
B, C, T = 3, 5, 13


def _ragged(gen, t):
    mask = torch.ones(B, 1, t, dtype=torch.bool)
    for b in range(B):
        start = int(torch.randint(0, t - 3, (1,), generator=gen))
        mask[b, 0, start:start + 2 + b] = False
    return mask


def cases():
    gen = torch.Generator().manual_seed(77)
    est = torch.randn(B, C, T, generator=gen)
    out = torch.randn(B, C, T, generator=gen)
    yield "ragged_mask", est, out, _ragged(gen, T), 0
    yield "full_mask", est, out, torch.rand(B, C, T, generator=gen) > 0.4, 0
    yield "all_true", est, out, torch.ones(B, 1, T, dtype=torch.bool), 0
    yield "all_false", est, out, torch.zeros(B, 1, T, dtype=torch.bool), 0
    limit = 3
    est_full = torch.randn(B, C, T + limit, generator=gen)
    out_full = torch.randn(B, C, T + limit, generator=gen)
    yield "time_crop", est_full, out_full, _ragged(gen, T + limit), limit
    ties = torch.rand(B, C, T, generator=gen) < 0.35
    yield "ties", est, torch.where(ties, est, out), torch.ones(B, 1, T, dtype=torch.bool), 0


def main():
    torch.set_num_threads(1)
    _, _, losses = ref_loader.load_reference()
    for name, est, out, mask, limit in cases():
        arrays = dict(est=est.numpy(), out=out.numpy(), mask=mask.numpy(), limit=np.int64(limit))
        for kind, cls in (("l1", losses.L1Loss), ("l2", losses.L2Loss)):
            e, o = est.clone().requires_grad_(True), out.clone().requires_grad_(True)
            loss = cls()(e[..., limit:], o[..., limit:], mask[..., limit:])
            loss.backward()
            arrays.update({f"{kind}.loss": loss.detach().numpy(), f"{kind}.d_est": e.grad.numpy(),
                           f"{kind}.d_out": o.grad.numpy()})
        path = os.path.join(OUT, f"regression_{name}.npz")
        np.savez_compressed(path, **arrays)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
