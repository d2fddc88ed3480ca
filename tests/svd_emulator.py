"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the spectral-norm penalty entry points of include/bm_b200.h
(`bm_svd_penalty_fwd`, `bm_svd_penalty_bwd`; `bm_svd_table` is host code and runs in the library) as an extension of
`tests/metrics_emulator.py`, with the conventions of `tests/abi_emulator.py`: each entry point's documented contract
restated with torch ops on the buffers the host code passes, interpreted through the integer arguments only.

The weights reach the entry points through the table's int64 addresses; on the CPU they are read (and only read) at those
addresses.  The value and the gradient are the fp64 restatement of oracle/svd_oracle.py on the fp32 weights and draws.
The emulated forward keeps nothing in the workspaces: the backward recomputes from the weights and the draws.  `emulated()`
also lets CPU weights through the penalty's CUDA check, and keeps every draw buffer a forward received in `emu.draws`.
"""
from __future__ import annotations

import contextlib
import ctypes

import torch

import metrics_emulator
import regression_emulator
from abi_emulator import _v
from oracle import svd_oracle

FIELDS = 12
P, M, N, TRANS, EXACT, WS, WS64, R_OFF, G_OFF = range(9)


def _weights(table, W, q):
    """per weight: (P [rows_p, cols_p] read at its address, R [n, q] offset, gradient offset)"""
    out = []
    for row in _v(table, W, FIELDS).tolist():
        m, n, trans = row[M], row[N], row[TRANS]
        rows_p, cols_p = (n, m) if trans else (m, n)
        buf = (ctypes.c_float * (rows_p * cols_p)).from_address(row[P])
        out.append((torch.frombuffer(buf, dtype=torch.float32).view(rows_p, cols_p).clone(), row[R_OFF], n, row[G_OFF]))
    return out


class SvdEmulator(metrics_emulator.MetricsEmulator):
    def __init__(self):
        super().__init__()
        self.draws = []

    def bm_svd_penalty_fwd(self, table, W, q, niter, tiles_m, tiles_n, R, ws, ws64, proba, out, stream):
        assert 1 <= q <= 32 and niter >= 0 and proba > 0
        self.draws.append(R.clone())
        total = 0.0
        for p, r_off, n, _ in _weights(table, W, q):
            total += svd_oracle.estimate(p, R.reshape(-1)[r_off:r_off + n * q].view(n, q), niter)[0]
        _v(out, 1)[0] = total / proba

    def bm_svd_penalty_bwd(self, table, W, q, niter, tiles_m, tiles_n, tiles_w, R, ws, ws64, gout, proba, grad, stream):
        s = float(_v(gout, 1)[0]) / proba
        for p, r_off, n, g_off in _weights(table, W, q):
            if g_off < 0:
                continue
            g = svd_oracle.estimate(p, R.reshape(-1)[r_off:r_off + n * q].view(n, q), niter)[1]
            grad.reshape(-1)[g_off:g_off + p.numel()].copy_((s * g).reshape(-1))


@contextlib.contextmanager
def emulated():
    """regression_emulator.emulated() on SvdEmulator, with the penalty's CUDA check lifted and no cached weight table"""
    import brainmagick_b200.functional as BF
    saved = BF._require_cuda_svd
    BF._require_cuda_svd = lambda weights: None
    BF._svd_plans.clear()
    try:
        with regression_emulator.emulated(SvdEmulator) as emu:
            yield emu
    finally:
        BF._require_cuda_svd = saved
        BF._svd_plans.clear()
