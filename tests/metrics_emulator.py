"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the test-metric entry points of include/bm_b200.h
(`bm_metric_workspace`, `bm_metric_update`, `bm_metric_finalize`) as an extension of `tests/regression_emulator.py`, with
the conventions of `tests/abi_emulator.py`: each entry point's documented contract restated with torch ops on the buffers
the host code passes, interpreted through the integer arguments only.

The operands and the mask reach the C ABI through `functional._view_ptr` as the smallest flat view spanning each tensor
(encode_emulator) and are rebuilt here from that span and the stride arguments.  `emulated()` also lets CPU tensors
through the metrics' CUDA check.
"""
from __future__ import annotations

import contextlib

import torch

import regression_emulator
from abi_emulator import _v

FLAGS = dict(left_unstable=1, left_nan=2, right_unstable=4, right_nan=8, result_nan=16, counted=32)


def _nct(p, sn, sc, st, N, C, T):
    return p.as_strided((N, C, T), (sn, sc, st))


class MetricsEmulator(regression_emulator.RegressionEmulator):
    def bm_metric_workspace(self, N, C, T):
        from brainmagick_b200 import _lib
        return int(_lib.load().bm_metric_workspace(N, C, T))     # a shape query: the library answers it

    def bm_metric_update(self, kind, dtype, left, l_sn, l_sc, l_st, right, r_sn, r_sc, r_st, mask, m_sn, m_sc, m_st, m_n,
                         N, C, T, K, acc, seen, parity, ws, ws_floats, stream):
        assert kind in (0, 1, 2, 3) and dtype in (0, 1) and m_n in (1, N) and parity in (0, 1)
        assert left.dtype == right.dtype == (torch.float32, torch.float64)[dtype]
        if C * T == 0:
            return
        if kind == 3:
            assert C == 1 and K >= 1
            z = _nct(left, l_sn, l_sc, l_st, N, K, T)
            y = _nct(right, r_sn, 0, r_st, N, 1, T).double()
            m = _nct(mask, m_sn, 0, m_st, N, 1, T).bool()
            hit = m & (z.argmax(1, keepdim=True).double() == y)          # torch's argmax: first maximum, NaN maximal
            sums = [hit.double().sum(0)]
        else:
            a, b = _nct(left, l_sn, l_sc, l_st, N, C, T), _nct(right, r_sn, r_sc, r_st, N, C, T)
            m = _nct(mask, m_sn, m_sc, m_st, N, C, T).double()
            l, r = a.double(), b.double()
            if kind == 0:
                sums = [(l * r * m).sum(0), (l * m).sum(0), (r * m).sum(0), ((l * m) ** 2).sum(0), ((r * m) ** 2).sum(0)]
            else:
                d = (a - b).double() * m
                sums = [d.abs().sum(0) if kind == 1 else (d * d).sum(0)]
        count = _nct(mask, m_sn, m_sc if kind != 3 else 0, m_st, m_n, C, T).double().sum(0)
        new = torch.stack([s.reshape(-1) for s in sums] + [count.reshape(-1)])
        A = _v(acc, new.shape[0], C * T)
        s = _v(seen, 2)
        was = bool(s[parity] != 0)
        A.copy_((A if was else torch.zeros_like(A)) + new)
        if was or bool((count != 0).any()):
            s[parity ^ 1] = 1

    def bm_metric_finalize(self, kind, acc, C, T, tol, out, out_dtype, flag, stream):
        cols = C * T
        bits = 0
        if kind == 0:
            sd, sl, sr, sll, srr, cnt = _v(acc, 6, cols)
            nl2, nr2 = sll - sl * sl / cnt, srr - sr * sr / cnt
            for n2, unstable, nan in ((nl2, "left_unstable", "left_nan"), (nr2, "right_unstable", "right_nan")):
                bits |= FLAGS[unstable] if bool((n2 < -tol).any()) else 0
                bits |= FLAGS[nan] if bool(n2.isnan().any()) else 0
            res = (sd - sl * sr / cnt) / (nl2.clamp(0, float("inf")).sqrt() * nr2.clamp(0, float("inf")).sqrt()).clamp(
                tol, float("inf"))
        else:
            s, cnt = _v(acc, 2, cols)
            res = s / cnt
        bits |= FLAGS["counted"] if bool((cnt != 0).any()) else 0
        bits |= FLAGS["result_nan"] if bool(res.isnan().any()) else 0
        _v(out, cols).copy_(res)
        _v(flag, 1)[0] = bits


@contextlib.contextmanager
def emulated():
    """regression_emulator.emulated() on MetricsEmulator, with the metrics' CUDA check lifted"""
    import brainmagick_b200.functional as BF
    saved = BF._require_cuda_metric
    BF._require_cuda_metric = lambda *ts: None
    try:
        with regression_emulator.emulated(MetricsEmulator) as emu:
            yield emu
    finally:
        BF._require_cuda_metric = saved
