"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the negative-pool entry points of include/bm_b200.h
(`bm_scatter_rows`, `bm_clip_loss_fwd_pooled`, `bm_clip_loss_fwd_pooled_det`, `bm_clip_loss_bwd_pooled`), as an extension
of `tests/abi_emulator.py` with the same conventions: each entry point's documented contract restated with torch ops on the
buffers the host code passes, interpreted through the integer arguments only (tensor-core entry points in exact fp32).

The pooled forms are the contiguous forms on the candidates `[cand[:Bb]; arena[slots]]`.  `emulated()` is
`abi_emulator.emulated()` with these entry points added.
"""
from __future__ import annotations

import contextlib

import torch

import abi_emulator
from abi_emulator import _v


def _pooled(cand, Bb, arena, slots, Bc, KT):
    rows = [_v(cand, Bb, KT)]
    if Bc > Bb:
        rows.append(arena.reshape(-1, KT)[slots.long()[:Bc - Bb]])
    return torch.cat(rows).contiguous()


class NegativePoolEmulator(abi_emulator.Emulator):
    def bm_scatter_rows(self, x, rows, n_rows, row_elems, y, stream):
        r = rows.long()[:n_rows]
        assert torch.unique(r).numel() == n_rows, "bm_scatter_rows: rows must be distinct"
        y.reshape(-1, row_elems)[r] = _v(x, n_rows, row_elems)

    def bm_clip_loss_fwd_pooled(self, est, cand, Bb, arena, slots, Bn, Bc, KT, target_offset, inv_norm, scores, probs,
                                row_loss, loss, ws, ws_floats, status, stream):
        assert KT >= 32 and KT % 4 == 0 and 0 <= Bb <= Bc
        self.bm_clip_loss_fwd(est, _pooled(cand, Bb, arena, slots, Bc, KT), Bn, Bc, KT, target_offset, inv_norm, scores,
                              probs, row_loss, loss, ws, ws_floats, status, stream)

    bm_clip_loss_fwd_pooled_det = bm_clip_loss_fwd_pooled

    def bm_clip_loss_bwd_pooled(self, probs, inv_norm, cand, Bb, arena, slots, gout, Bn, Bc, KT, target_offset, G, dest,
                                status, stream):
        assert KT >= 32 and KT % 4 == 0 and G.numel() >= Bn * (-(-Bc // 4) * 4)
        self.bm_clip_loss_bwd(probs, inv_norm, _pooled(cand, Bb, arena, slots, Bc, KT), gout, Bn, Bc, KT, target_offset, G,
                              dest, status, stream)


@contextlib.contextmanager
def emulated(emulator_class=NegativePoolEmulator):
    """abi_emulator.emulated() running on `emulator_class` (NegativePoolEmulator or a subclass of it)."""
    saved = abi_emulator.Emulator
    abi_emulator.Emulator = emulator_class
    try:
        with abi_emulator.emulated() as emu:
            yield emu
    finally:
        abi_emulator.Emulator = saved
