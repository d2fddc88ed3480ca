"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the SyncBatchNorm entry points of include/bm_b200.h
(`bm_bn_stats_finalize_counted` and the `_reduce` / `_apply` halves of the BatchNorm backward), as an extension of
`tests/tf32_emulator.py` with the same conventions.  The row count n of the counted forms stays a tensor (slot 2C of the
sums): like the kernels, the emulation never reads it on the host.

`emulated()` is `tf32_emulator.emulated()` with these entry points added.
"""
from __future__ import annotations

import contextlib

import torch

import tf32_emulator
from abi_emulator import _act_grad, _v
from tf32_emulator import TF32Emulator


class SyncBNEmulator(TF32Emulator):
    def bm_bn_stats_finalize_counted(self, stats, eps, momentum, running_mean, running_var, mean, invstd, C, stream):
        st = _v(stats, 2 * C + 1)
        n = st[2 * C]
        m = st[:C] / n
        var = (st[C:2 * C] / n - m * m).clamp_min(0)
        _v(mean, C).copy_(m.float())
        _v(invstd, C).copy_((1.0 / torch.sqrt(var + eps)).float())
        if running_mean is not None:
            unb = torch.where(n > 1, var * n / (n - 1), var)
            _v(running_mean, C).mul_(1 - momentum).add_(momentum * m.float())
            _v(running_var, C).mul_(1 - momentum).add_(momentum * unb.float())

    @staticmethod
    def _dz(g, y, mean, invstd, gamma, beta, rows, C, act, slope):
        yh = (_v(y, rows, C) - _v(mean, C)) * _v(invstd, C)
        return _v(g, rows, C) * _act_grad(act, yh * _v(gamma, C) + _v(beta, C), slope), yh

    def bm_bn_act_skip_bwd_reduce(self, g, y, mean, invstd, gamma, beta, rows, C, act, slope, sums, dgamma, dbeta, stream):
        dz, yh = self._dz(g, y, mean, invstd, gamma, beta, rows, C, act, slope)
        s1, s2 = dz.double().sum(0), (dz * yh).double().sum(0)
        _v(sums, 2 * C).copy_(torch.cat([s1, s2]))
        _v(dbeta, C).copy_(s1.float())
        _v(dgamma, C).copy_(s2.float())

    def bm_bn_act_skip_bwd_apply(self, g, y, mean, invstd, gamma, beta, rows, C, act, slope, sums, dy, stream):
        dz, yh = self._dz(g, y, mean, invstd, gamma, beta, rows, C, act, slope)
        st = _v(sums, 2 * C + 1)
        n = st[2 * C]
        v = dz - (st[:C] / n).float() - yh * (st[C:2 * C] / n).float()
        _v(dy, rows, C).copy_(_v(gamma, C) * _v(invstd, C) * v)

    def bm_bn_gelu_skip_bwd_reduce(self, g, y, mean, invstd, gamma, beta, rows, C, sums, dgamma, dbeta, stream):
        self.bm_bn_act_skip_bwd_reduce(g, y, mean, invstd, gamma, beta, rows, C, 0, 0.0, sums, dgamma, dbeta, stream)

    def bm_bn_gelu_skip_bwd_apply(self, g, y, mean, invstd, gamma, beta, rows, C, sums, dy, stream):
        self.bm_bn_act_skip_bwd_apply(g, y, mean, invstd, gamma, beta, rows, C, 0, 0.0, sums, dy, stream)

    # deterministic forms: (workspace, workspace_floats) before the stream
    def bm_bn_act_skip_bwd_reduce_det(self, *args):
        self._inner("bm_bn_act_skip_bwd_reduce", *args[:-3], args[-1])

    def bm_bn_gelu_skip_bwd_reduce_det(self, *args):
        self._inner("bm_bn_gelu_skip_bwd_reduce", *args[:-3], args[-1])


@contextlib.contextmanager
def emulated(emulator_class=SyncBNEmulator):
    with tf32_emulator.emulated(emulator_class) as emu:
        yield emu
