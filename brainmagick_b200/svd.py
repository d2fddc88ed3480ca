"""Drop-in `svd_penalty` (bm/svd.py): the solver's penalty on the largest singular value of every conv and linear weight,
`loss += args.optim.svd * svd_penalty(model)` (bm/solver.py:379-380), computed by grouped CUDA kernels.

The result and the random draws are the reference's: one `penalty_rng.random()` per call, and per selected weight the
`torch.randn(min(m, n), dim)` that `torch.svd_lowrank` draws, in `named_modules()` order from torch's CUDA generator.  Each
estimate is the top eigenvalue of Qᵀ A Aᵀ Q for the same randomized subspace iteration (the reference's S[0] ** 2); the
gradient is taken through the spans of the iteration rather than through QR and SVD (DESIGN §4.10).  Everything is fp32
with fp64 Gram matrices, whatever the TF32 flag or autocast.  No value is read back to the host, and the weight table is
built on the first eager call, so a step that calls it can be captured in a CUDA graph after one eager step (with
`proba == 1`: the host's coin cannot be captured)."""
from __future__ import annotations

import random

import torch

from . import functional as BF

# shared so that every distributed worker skips the penalty on the same steps (the reference's comment and seed)
penalty_rng = random.Random(1234)


def svd_penalty(model, min_size=1., dim=16, niters=2, proba=1, exact=False):
    """Penalty on the largest singular value of every `_ConvNd` / `nn.Linear` weight of `model` with at least
    `256 * min_size` elements, each viewed as `[shape[0], -1]`: Σ torch.svd_lowrank(p, dim, niters)[1][0] ** 2 / proba as a
    0-dim fp32 CUDA tensor, or the float 0. when `penalty_rng.random() > proba` (one draw per call).  `exact=True` is not
    ported."""
    coin = penalty_rng.random()
    if proba < 1 and BF.capturing():        # whichever way the coin fell, the graph would replay it on every step
        raise RuntimeError("svd_penalty with proba < 1 cannot be captured: the host's coin would be frozen into the graph")
    if coin > proba:
        return 0.
    if exact:
        raise NotImplementedError("svd_penalty(exact=True) is not ported: the CUDA path runs the randomized estimate")
    weights = []
    for _, m in model.named_modules():
        if not isinstance(m, (torch.nn.modules.conv._ConvNd, torch.nn.Linear)):
            continue
        p = m.weight
        if p.numel() / 2**8 < min_size:
            continue
        weights.append(p)
    if not weights:
        return 0 / proba
    if not (1 <= dim <= BF.SVD_MAX_DIM) or niters < 0:
        raise NotImplementedError(f"svd_penalty takes 1 <= dim <= {BF.SVD_MAX_DIM} and niters >= 0, got dim={dim}, "
                                  f"niters={niters}")
    if any(p.is_complex() for p in weights) or any(p.dtype != torch.float32 for p in weights):
        raise TypeError(f"svd_penalty kernels take fp32 weights, got {sorted({str(p.dtype) for p in weights})}")
    BF._require_cuda_svd(weights)
    if len({p.device for p in weights}) > 1:
        raise RuntimeError(f"svd_penalty: the weights are on several devices: {sorted({str(p.device) for p in weights})}")
    if not all(p.is_contiguous() for p in weights):
        raise RuntimeError("svd_penalty reads the weights in place and takes contiguous ones")
    return BF.svd_penalty(weights, dim, niters, proba)
