"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the input-gradient entry points of include/bm_b200.h
(`bm_sensor_mix_bwd_data`, `bm_tc_sensor_mix_bwd_data`, `bm_clip_scores_bwd`), as an extension of `tests/abi_emulator.py`
with the same conventions: each entry point's documented contract restated with torch ops on the buffers the host code
passes, interpreted through the integer arguments only (tensor-core entry points in exact fp32).

`emulated()` is `abi_emulator.emulated()` with these entry points added.
"""
from __future__ import annotations

import contextlib

import torch

import abi_emulator
from abi_emulator import _ld, _v


class InputGradEmulator(abi_emulator.Emulator):
    def bm_sensor_mix_bwd_data(self, du, ld_du, weights, rec_of_sample, mask, B, C, T, O, dmeg, stream):
        w = _v(weights, weights.numel() // (O * C), O, C)[rec_of_sample.long()[:B]]
        out = torch.einsum("bto,boc->bct", _ld(du, B * T, ld_du, O).reshape(B, T, O), w)
        if mask is not None:
            out = out * _v(mask, C)[None, :, None]
        _v(dmeg, B, C, T).copy_(out)

    def bm_tc_sensor_mix_bwd_data(self, du, w_hi, w_lo, wsel, n_sets, mask, B, T, Op, Cp, C, dmeg, status, stream):
        w = (_v(w_hi, n_sets, Cp, Op) + _v(w_lo, n_sets, Cp, Op))[wsel.long()[:B], :C]
        out = torch.einsum("bto,bco->bct", _v(du, B, T, Op), w)
        if mask is not None:
            out = out * _v(mask, C)[None, :, None]
        _v(dmeg, B, C, T).copy_(out)

    def bm_clip_scores_bwd(self, dscores, scores, inv_norm, est, cand, Bn, Bc, KT, G, coef, dest, dcand, status, stream):
        g = _v(dscores, Bn, Bc) * _v(inv_norm, Bc)
        if dest is not None:
            _v(dest, Bn, KT).copy_(g @ _v(cand, Bc, KT))
        if dcand is not None:
            norm = 1.0 / _v(inv_norm, Bc) - 1e-8
            cf = torch.where(norm > 0, (g * _v(scores, Bn, Bc)).sum(0) / norm, torch.zeros(Bc))
            _v(dcand, Bc, KT).copy_(g.t() @ _v(est, Bn, KT) - cf[:, None] * _v(cand, Bc, KT))


@contextlib.contextmanager
def emulated(emulator_class=InputGradEmulator):
    """abi_emulator.emulated() running on `emulator_class` (InputGradEmulator or a subclass of it)."""
    saved = abi_emulator.Emulator
    abi_emulator.Emulator = emulator_class
    try:
        with abi_emulator.emulated() as emu:
            yield emu
    finally:
        abi_emulator.Emulator = saved
