"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the bf16 (`_bf16`) entry points of include/bm_b200.h, as an
extension of `tests/frozen_emulator.py` (and so of `tests/abi_emulator.py`) with the same conventions.

Each `_bf16` entry point's contract is its default form's with every operand element of the tensor-core contraction rounded
once to bf16 (round to nearest even: `x.to(torch.bfloat16)`; a weight handed over as tf32 pieces is rounded as hi + lo);
what runs outside the contraction (bias sums, the CLIP candidate norms and the candidate-gradient correction, epilogues)
reads the fp32 values.  The methods below round the contraction operands and hand them to the default form's emulation, or
restate the contraction in fp64 where its operand is formed inside the entry point (the CLIP backward's G).  Products of
bf16 values are exact, so the rounded operands carry the whole difference from the default form.  `calls` records the
entry points the host code reached.
"""
from __future__ import annotations

import contextlib

import torch

import frozen_emulator
from abi_emulator import _v
from frozen_emulator import FrozenEmulator


def rn_bf16(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> the nearest bf16 value (7 mantissa bits, ties to even), as fp32: cvt.rn.bf16x2.f32."""
    return t.detach().float().to(torch.bfloat16).float()


def _w(w_hi, w_lo):
    """The fp32 weight a form that takes tf32 pieces rounds: hi + lo (hi alone when lo is NULL)."""
    return w_hi if w_lo is None else w_hi + w_lo


def _clip_rows_loss(scores, Bn, Bc, target_offset, row_loss, loss):
    sc = _v(scores, Bn, Bc)
    rl = torch.logsumexp(sc, dim=1) - sc[torch.arange(Bn), torch.arange(Bn) + target_offset]
    _v(row_loss, Bn).copy_(rl)
    _v(loss, 1).copy_(rl.double().mean().float().reshape(1))


class BF16Emulator(FrozenEmulator):
    # ---- conv family: the default form on rounded operands (tf32 pieces: hi + lo rounded once)
    def bm_tc_conv1d_bf16(self, x, w_hi, w_lo, bias, addend, B, T, Cin, Ntot, Kw, dilation, sign, glu, act, out_tmajor, y,
                          aux, glu_out, stats, status, stream):
        self._inner("bm_tc_conv1d", rn_bf16(x), rn_bf16(_w(w_hi, w_lo)), None, bias, addend, B, T, Cin, Ntot, Kw,
                    dilation, sign, glu, act, out_tmajor, y, aux, glu_out, stats, status, stream)

    def bm_tc_conv1d_persistent_bf16(self, x, w_raw, bias, accumulate, B, T, Cin, Ntot, Kw, dilation, sign, glu, act,
                                     out_tmajor, y, aux, glu_out, stats, status, stream):
        self._inner("bm_tc_conv1d_persistent", rn_bf16(x), rn_bf16(w_raw), bias, accumulate, B, T, Cin, Ntot, Kw,
                    dilation, sign, glu, act, out_tmajor, y, aux, glu_out, stats, status, stream)

    def bm_tc_pointwise_sel_bf16(self, x, w_hi, w_lo, wsel, n_sets, B, T, Cin, Ntot, y, status, stream):
        self._inner("bm_tc_pointwise_sel", rn_bf16(x), rn_bf16(_w(w_hi, w_lo)), torch.zeros_like(w_hi), wsel, n_sets, B,
                    T, Cin, Ntot, y, status, stream)

    def bm_tc_sensor_mix_bwd_data_bf16(self, du, w_hi, w_lo, wsel, n_sets, mask, B, T, Op, Cp, C, dmeg, status, stream):
        self._inner("bm_tc_sensor_mix_bwd_data", rn_bf16(du), rn_bf16(_w(w_hi, w_lo)), torch.zeros_like(w_hi), wsel,
                    n_sets, mask, B, T, Op, Cp, C, dmeg, status, stream)

    # ---- weight gradients: the GEMM on rounded operands; the bias gradient sums the fp32 dy
    def bm_tc_wgrad_bf16(self, dy, x, B, T, M, N, Ntrue, Kw, dilation, ws, dw, dbias, status, stream):
        self._inner("bm_tc_wgrad", rn_bf16(dy), rn_bf16(x), B, T, M, N, Ntrue, Kw, dilation, ws, dw, None, status, stream)
        if dbias is not None:
            _v(dbias, M).copy_(_v(dy, B * T, M).sum(0))

    def bm_tc_wgrad_conv_bf16(self, dy, x, B, T, M, N, Ntrue, Kw, dilation, ws, dw, status, stream):
        self._inner("bm_tc_wgrad_conv", rn_bf16(dy), rn_bf16(x), B, T, M, N, Ntrue, Kw, dilation, ws, dw, status, stream)

    def bm_tc_wgrad_grouped_bf16(self, dy, x, order, seg_off, G, B, T, M, N, out, status, stream):
        self._inner("bm_tc_wgrad_grouped", rn_bf16(dy), rn_bf16(x), order, seg_off, G, B, T, M, N, out, status, stream)

    # ---- CLIP: scores on rounded operands, candidate norms from the fp32 candidates
    def bm_clip_scores_bf16(self, est, cand, Bn, Bc, KT, norms_given, inv_norm, scores, probs, ws, ws_floats, status,
                            stream):
        if not norms_given:
            self._inner("bm_candidate_inv_norms", cand, Bc, KT, torch.empty(Bc, dtype=torch.float64), inv_norm, stream)
        self._inner("bm_clip_scores", rn_bf16(est), rn_bf16(cand), Bn, Bc, KT, 1, inv_norm, scores, probs, ws, ws_floats,
                    status, stream)

    def bm_clip_loss_fwd_bf16(self, est, cand, Bn, Bc, KT, target_offset, inv_norm, scores, probs, row_loss, loss, ws,
                              ws_floats, status, stream):
        self._inner("bm_clip_scores_bf16", est, cand, Bn, Bc, KT, 0, inv_norm, scores, probs, ws, ws_floats, status, stream)
        _clip_rows_loss(scores, Bn, Bc, target_offset, row_loss, loss)

    def bm_clip_scores_det_bf16(self, *args):
        self._inner("bm_clip_scores_bf16", *args)

    def bm_clip_loss_fwd_det_bf16(self, *args):
        self._inner("bm_clip_loss_fwd_bf16", *args)

    @staticmethod
    def _clip_grads(g, scores, inv_norm, est, cand, Bn, Bc, KT, dest, dcand):
        """dest = rn(G) rn(C); dcand = rn(G)^T rn(E) - coef * C with coef from the fp32 G (see clip_cand_coef_kernel); the
        products and sums in fp64."""
        gr = rn_bf16(g).double()
        if dest is not None:
            _v(dest, Bn, KT).copy_((gr @ rn_bf16(_v(cand, Bc, KT)).double()).float())
        if dcand is not None:
            norm = 1.0 / _v(inv_norm, Bc) - 1e-8
            cf = torch.where(norm > 0, (g * _v(scores, Bn, Bc)).sum(0) / norm, torch.zeros(Bc))
            _v(dcand, Bc, KT).copy_((gr.t() @ rn_bf16(_v(est, Bn, KT)).double()).float() - cf[:, None] * _v(cand, Bc, KT))

    def bm_clip_loss_bwd_bf16(self, probs, inv_norm, cand, gout, Bn, Bc, KT, target_offset, G, dest, status, stream):
        g = self._G(probs, inv_norm, gout, Bn, Bc, target_offset)
        self._clip_grads(g, None, inv_norm, None, cand, Bn, Bc, KT, dest, None)

    def bm_clip_loss_bwd_cand_bf16(self, probs, scores, inv_norm, est, cand, gout, Bn, Bc, KT, target_offset, G, coef, dcand,
                                   status, stream):
        g = self._G(probs, inv_norm, gout, Bn, Bc, target_offset)
        self._clip_grads(g, scores, inv_norm, est, cand, Bn, Bc, KT, None, dcand)

    def bm_clip_scores_bwd_bf16(self, dscores, scores, inv_norm, est, cand, Bn, Bc, KT, G, coef, dest, dcand, status,
                                stream):
        g = _v(dscores, Bn, Bc) * _v(inv_norm, Bc)
        self._clip_grads(g, scores, inv_norm, est, cand, Bn, Bc, KT, dest, dcand)


@contextlib.contextmanager
def emulated(emulator_class=BF16Emulator):
    with frozen_emulator.emulated(emulator_class) as emu:
        yield emu
