"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the masked regression loss entry points of include/bm_b200.h
(`bm_masked_loss_workspace`, `bm_masked_loss_fwd`, `bm_masked_loss_bwd`) as an extension of `tests/encode_emulator.py`,
with the conventions of `tests/abi_emulator.py`: each entry point's documented contract restated with torch ops on the
buffers the host code passes, interpreted through the integer arguments only.

The operands are strided views: they reach the C ABI through `functional._view_ptr`, which `emulated()` replaces by the
smallest flat view spanning each tensor (encode_emulator), and are rebuilt here from that span and the stride arguments.
`emulated()` also lets CPU tensors through the losses' CUDA check.
"""
from __future__ import annotations

import contextlib

import torch

import encode_emulator
from abi_emulator import _v


def _bct(p, sb, sc, st, B, C, T):
    return p.as_strided((B, C, T), (sb, sc, st))


class RegressionEmulator(encode_emulator.EncodeEmulator):
    def bm_masked_loss_workspace(self, B, C, T):
        from brainmagick_b200 import _lib
        return int(_lib.load().bm_masked_loss_workspace(B, C, T))     # a shape query: the library answers it

    def bm_masked_loss_fwd(self, kind, est, e_sb, e_sc, out, o_sb, o_sc, mask, m_sb, m_sc, m_st, B, C, T, ws, ws_floats,
                           loss, inv_n, stream):
        assert kind in (0, 1) and ws_floats >= self.bm_masked_loss_workspace(B, C, T)
        m = _bct(mask, m_sb, m_sc, m_st, B, C, T).bool()
        d = (_bct(est, e_sb, e_sc, 1, B, C, T) - _bct(out, o_sb, o_sc, 1, B, C, T))[m].double()
        n = float(m.sum())
        total = d.abs().sum() if kind == 0 else (d * d).sum()
        _v(loss, 1)[0] = float(total / n) if n else float("nan")
        _v(inv_n, 1)[0] = 1.0 / n if n else float("inf")

    def bm_masked_loss_bwd(self, kind, gout, inv_n, est, e_sb, e_sc, out, o_sb, o_sc, mask, m_sb, m_sc, m_st, B, C, T,
                           d_est, d_out, stream):
        assert kind in (0, 1)
        m = _bct(mask, m_sb, m_sc, m_st, B, C, T).bool()
        d = _bct(est, e_sb, e_sc, 1, B, C, T) - _bct(out, o_sb, o_sc, 1, B, C, T)
        scale = (1.0 if kind == 0 else 2.0) * (_v(gout, 1)[0] * _v(inv_n, 1)[0])
        g = torch.where(m, (torch.sign(d) if kind == 0 else d) * scale, torch.zeros(()))
        if d_est is not None:
            _v(d_est, B, C, T).copy_(g)
        if d_out is not None:
            _v(d_out, B, C, T).copy_(torch.where(m, -g, torch.zeros(())))


@contextlib.contextmanager
def emulated(emulator_class=RegressionEmulator):
    """encode_emulator.emulated() on `emulator_class`, with the losses' CUDA check lifted"""
    import brainmagick_b200.functional as BF
    import input_grad_emulator
    saved = BF._require_cuda_operands
    BF._require_cuda_operands = lambda *ts: None
    try:
        with input_grad_emulator.emulated(emulator_class) as emu, encode_emulator._patched_view_ptr(encode_emulator._span):
            yield emu
    finally:
        BF._require_cuda_operands = saved
