"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the FeatureDecodingLoss entry points of include/bm_b200.h
(`bm_decoding_loss_workspace`, `bm_decoding_loss_fwd`, `bm_decoding_loss_bwd`) as an extension of
`tests/regression_emulator.py`, with the conventions of `tests/abi_emulator.py`: each entry point's documented contract
restated with torch ops on the buffers the host code passes, interpreted through the integer arguments and the feature
table only.

The operands reach the C ABI through `functional._view_ptr` as the smallest flat view spanning each tensor
(encode_emulator) and are rebuilt here from that span and the stride arguments.  `emulated()` also lets CPU tensors through
the loss's CUDA check.
"""
from __future__ import annotations

import contextlib

import torch

import regression_emulator
from abi_emulator import _v


def _rows(p, start, sb, sc, st, B, C, T):
    """[B, C, T] window of the span p from channel `start` on, through the strides"""
    return p.as_strided((B, C, T), (sb, sc, st), p.storage_offset() + start * sc)


def _targets(v, K):
    """out.long() of targets v: (class or -1 where there is none, bad >= K or NaN, bad negative, ignored)"""
    too_large = ~(v < K)
    y = torch.where(too_large, torch.zeros_like(v), v).trunc().long()
    ignored = ~too_large & (y == -100)
    negative = ~too_large & (y < 0) & ~ignored
    return torch.where(too_large | (y < 0), -1, y), too_large, negative, ignored


class DecodingLossEmulator(regression_emulator.RegressionEmulator):
    def bm_decoding_loss_workspace(self, B, T, F):
        from brainmagick_b200 import _lib
        return int(_lib.load().bm_decoding_loss_workspace(B, T, F))     # a shape query: the library answers it

    def _features(self, est, e_sb, e_sc, out, o_sb, o_sc, mask, m_sb, m_sc, m_st, B, T, table, F, weights):
        """per feature: (kind, slice of est, slice of out, mask [B, w, T] or [B, T], class weight per (b, t) or None,
        targets) as the contract reads them"""
        for f, (kind, es, w, os_, woff, slot) in enumerate(_v(table, F, 6).tolist()):
            if kind == 0:
                yield f, kind, slot, _rows(est, es, e_sb, e_sc, 1, B, w, T), _rows(out, os_, o_sb, o_sc, 1, B, w, T), \
                    _rows(mask, 0, m_sb, m_sc, m_st, B, w, T).bool(), None
            else:
                z = _rows(est, es, e_sb, e_sc, 1, B, w, T)
                v = _rows(out, os_, o_sb, o_sc, 1, B, 1, T)[:, 0]
                wt = None if woff < 0 else _v(weights, woff + w)[woff:]
                yield f, kind, slot, z, (v, wt), _rows(mask, 0, m_sb, 0, m_st, B, 1, T)[:, 0].bool(), w

    def bm_decoding_loss_fwd(self, est, e_sb, e_sc, out, o_sb, o_sc, mask, m_sb, m_sc, m_st, B, T, table, F, weights, lse,
                             ws, ws_floats, loss, scale, flag, status, stream):
        assert 1 <= F <= 15 and ws_floats >= self.bm_decoding_loss_workspace(B, T, F)
        total, seen, code = None, False, 0
        for f, kind, slot, e, o, m, K in self._features(est, e_sb, e_sc, out, o_sb, o_sc, mask, m_sb, m_sc, m_st, B, T,
                                                         table, F, weights):
            if kind == 0:
                d = (e - o)[m].double()
                s, n = (d * d).sum(), float(m.sum())
                seen |= n > 0
                sc = 2.0 / n if n else float("inf")
            else:
                v, wt = o
                lse_ = torch.logsumexp(e.double(), dim=1).float()
                _v(lse, (slot + 1) * B * T)[slot * B * T:].copy_(lse_.reshape(-1))
                y, too_large, negative, _ = _targets(v, K)
                ok = m & (y >= 0)
                zy = e.gather(1, y.clamp(min=0)[:, None])[:, 0]
                wy = torch.ones_like(v) if wt is None else wt[y.clamp(min=0)]
                s = (wy.double() * (lse_ - zy).double())[ok].sum()
                n = float(wy.double()[ok].sum())
                seen |= bool(m.any())
                sc = 1.0 / n if n else float("inf")
                if code == 0 and bool(too_large.any()):
                    code = 905 | (f << 16)
                elif code == 0 and bool((negative & m).any()):
                    code = 906 | (f << 16)
            term = torch.tensor(float(s), dtype=torch.float32) / torch.tensor(n, dtype=torch.float32)
            total = term if total is None else total + term
            _v(scale, F)[f] = sc
        code = 904 if not seen else code
        _v(loss, 1)[0] = total
        _v(flag, 1)[0] = code
        if code and status is not None and int(status[0]) == 0:
            status[0] = code & 0xFFFF

    def bm_decoding_loss_bwd(self, gout, scale, lse, est, e_sb, e_sc, out, o_sb, o_sc, mask, m_sb, m_sc, m_st, B, T, est_C,
                             out_C, table, F, weights, d_est, d_out, stream):
        g = float(_v(gout, 1)[0])
        ge, go = torch.zeros(B, est_C, T), torch.zeros(B, out_C, T)
        for f, kind, slot, e, o, m, K in self._features(est, e_sb, e_sc, out, o_sb, o_sc, mask, m_sb, m_sc, m_st, B, T,
                                                         table, F, weights):
            kind_, es, w, os_ = _v(table, F, 6)[f, :4].tolist()
            sc = float(_v(scale, F)[f])
            if kind == 0:
                grad = torch.where(m, (e - o) * sc * g, torch.zeros(()))
                ge[:, es:es + w] = grad
                go[:, os_:os_ + w] = torch.where(m, -(e - o) * sc * g, torch.zeros(()))
            else:
                v, wt = o
                y, *_ = _targets(v, K)
                ok = m & (y >= 0)
                lse_ = _v(lse, (slot + 1) * B * T)[slot * B * T:].view(B, 1, T)
                wy = torch.ones_like(v) if wt is None else wt[y.clamp(min=0)]
                onehot = torch.nn.functional.one_hot(y.clamp(min=0), K).permute(0, 2, 1).float()
                grad = (g * sc * wy)[:, None] * (torch.exp(e - lse_) - onehot)
                ge[:, es:es + K] = torch.where(ok[:, None], grad, torch.zeros(()))
        if d_est is not None:
            _v(d_est, B, est_C, T).copy_(ge)
        if d_out is not None:
            _v(d_out, B, out_C, T).copy_(go)


@contextlib.contextmanager
def emulated():
    """regression_emulator.emulated() on DecodingLossEmulator, with the decoding loss's CUDA check lifted"""
    import brainmagick_b200.functional as BF
    saved = BF._require_cuda_decoding
    BF._require_cuda_decoding = lambda *ts: None
    try:
        with regression_emulator.emulated(DecodingLossEmulator) as emu:
            yield emu
    finally:
        BF._require_cuda_decoding = saved
