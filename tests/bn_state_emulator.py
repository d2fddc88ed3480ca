"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the cumulative-average BatchNorm finalize entry points of
include/bm_b200.h (`bm_bn_stats_finalize_cumulative`, `bm_bn_stats_finalize_counted_cumulative`), with the conventions of
`tests/abi_emulator.py`.  `CumulativeFinalize` is a mixin: put it first in the bases of the emulator class a test runs on.
Like the kernels, the emulation never reads the count on the host: the factor 1 / num_batches_tracked stays a tensor.
"""
from __future__ import annotations

import torch

from abi_emulator import _v


def _update(running_mean, running_var, factor, m, unb, C):
    _v(running_mean, C).mul_(1 - factor).add_(factor * m.float())
    _v(running_var, C).mul_(1 - factor).add_(factor * unb.float())


class CumulativeFinalize:
    def bm_bn_stats_finalize_cumulative(self, stats, n, eps, num_batches_tracked, running_mean, running_var, mean, invstd,
                                        C, stream):
        st = _v(stats, 2 * C)
        m = st[:C] / n
        var = (st[C:] / n - m * m).clamp_min(0)
        _v(mean, C).copy_(m.float())
        _v(invstd, C).copy_((1.0 / torch.sqrt(var + eps)).float())
        factor = (1.0 / _v(num_batches_tracked, 1).double()).float()
        _update(running_mean, running_var, factor, m, var * n / (n - 1) if n > 1 else var, C)

    def bm_bn_stats_finalize_counted_cumulative(self, stats, eps, num_batches_tracked, running_mean, running_var, mean,
                                                invstd, C, stream):
        st = _v(stats, 2 * C + 1)
        n = st[2 * C]
        m = st[:C] / n
        var = (st[C:2 * C] / n - m * m).clamp_min(0)
        _v(mean, C).copy_(m.float())
        _v(invstd, C).copy_((1.0 / torch.sqrt(var + eps)).float())
        factor = (1.0 / _v(num_batches_tracked, 1).double()).float()
        _update(running_mean, running_var, factor, m, torch.where(n > 1, var * n / (n - 1), var), C)
