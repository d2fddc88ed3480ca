"""TEST INFRASTRUCTURE ONLY -- the torch-CPU emulation of the NULL gradient pointers of include/bm_b200.h (a frozen
parameter's gradient, a data gradient nothing below needs), as an extension of `tests/deterministic_emulator.py` with the same
conventions.  Each method restates its entry point's contract with the NULL pointers allowed and asserts that a NULL output
is never read.  `calls` records the entry points the host code reached."""
from __future__ import annotations

import contextlib

import torch

import deterministic_emulator
from abi_emulator import _act_grad, _gelu_grad, _ld, _v
from deterministic_emulator import DeterministicEmulator


class FrozenEmulator(DeterministicEmulator):
    def bm_subject_layers_bwd(self, dx0, ld_x0, v, ld_v, subj_w, subject, subj_order, subj_off, B, T, IL, D, S, ld_dv, dv,
                              d_subj_w, stream):
        g = _ld(dx0, B * T, ld_x0, D).reshape(B, T, D)
        subj = subject.long()[:B]
        if dv is not None:
            m = _v(subj_w, S, IL, D)[subj]
            _ld(dv, B * T, ld_dv, IL).copy_(torch.einsum("btd,bpd->btp", g, m).reshape(B * T, IL))
        if d_subj_w is not None:
            order, off = subj_order.long(), subj_off.long()
            assert off[0] == 0 and off[S] == B and sorted(order.tolist()) == list(range(B))
            vv = _ld(v, B * T, ld_v, IL).reshape(B, T, IL)
            per_sample = torch.einsum("btp,btd->bpd", vv, g)
            _v(d_subj_w, S, IL, D).copy_(torch.zeros(S, IL, D).index_add_(0, subj, per_sample))

    def bm_initial_linear_bwd(self, dv, ld_dv, u, ld_u, il_w, B, T, O, IL, ld_du, du, d_il_w, d_il_b, stream):
        g = _ld(dv, B * T, ld_dv, IL)
        if du is not None:
            _ld(du, B * T, ld_du, O).copy_(g @ _v(il_w, IL, O))
        if d_il_w is not None:
            _v(d_il_w, IL, O).copy_(g.t() @ _ld(u, B * T, ld_u, O))
        if d_il_b is not None:
            _v(d_il_b, IL).copy_(g.sum(0))

    def bm_sensor_chain_bwd(self, dx0, meg, il_w, subj_w, subject, u, v, subj_order, subj_off, rec_order, rec_off, B, C, T,
                            O, IL, D, ld_x0, S, R, dv, du, d_subj_w, d_il_w, d_il_b, d_weights, stream):
        assert dv is not None or (du is None and d_il_w is None and d_il_b is None)
        assert du is not None or d_weights is None
        self._inner("bm_subject_layers_bwd", dx0, ld_x0, v, IL, subj_w, subject, subj_order, subj_off, B, T, IL, D, S, IL,
                    dv, d_subj_w, stream)
        if du is not None or d_il_w is not None or d_il_b is not None:
            self._inner("bm_initial_linear_bwd", dv, IL, u, O, il_w, B, T, O, IL, O, du, d_il_w, d_il_b, stream)
        if d_weights is not None:
            self._inner("bm_sensor_mix_bwd", du, O, meg, rec_order, rec_off, B, C, T, O, R, d_weights, stream)

    def bm_bn_act_skip_bwd(self, g, y, mean, invstd, gamma, beta, batch_stats, rows, C, act, slope, sums, dy, dgamma, dbeta,
                           stream):
        reduces = mean is not None and (batch_stats or dgamma is not None or dbeta is not None)
        if reduces:
            assert sums is not None and dgamma is not None and dbeta is not None
            return super().bm_bn_act_skip_bwd(g, y, mean, invstd, gamma, beta, batch_stats, rows, C, act, slope, sums, dy,
                                              dgamma, dbeta, stream)
        gg, yy = _v(g, rows, C).clone(), _v(y, rows, C)
        if mean is None:
            _v(dy, rows, C).copy_(gg * _act_grad(act, yy, slope))
            return
        yh = (yy - _v(mean, C)) * _v(invstd, C)
        dz = gg * _act_grad(act, yh * _v(gamma, C) + _v(beta, C), slope)
        _v(dy, rows, C).copy_(_v(gamma, C) * _v(invstd, C) * dz)

    def bm_head_bwd_params(self, dest, x, h1, q, B, T, H, F_, dq, dw0, db0, dw2, db2, stream):
        d = _v(dest, B, F_, T).transpose(1, 2).reshape(B * T, F_)
        if dw2 is not None:
            _v(dw2, 2 * H, F_).copy_(_v(q, B * T, 2 * H).t() @ d)
        if db2 is not None:
            _v(db2, F_).copy_(d.sum(0))
        dh1 = _v(dq, B * T, 2 * H).clone() * _gelu_grad(_v(h1, B * T, 2 * H))
        _v(dq, B * T, 2 * H).copy_(dh1)
        if dw0 is not None:
            _v(dw0, 2 * H, H).copy_(dh1.t() @ _v(x, B * T, H))
        if db0 is not None:
            _v(db0, 2 * H).copy_(dh1.sum(0))

    def bm_head_bwd(self, dest, x, w0, w2, h1, q, B, T, H, F_, dq, dx, dw0, db0, dw2, db2, stream):
        d = _v(dest, B, F_, T).transpose(1, 2).reshape(B * T, F_)
        if dw2 is not None:
            _v(dw2, 2 * H, F_).copy_(_v(q, B * T, 2 * H).t() @ d)
        if db2 is not None:
            _v(db2, F_).copy_(d.sum(0))
        if dx is None and dw0 is None and db0 is None:
            return
        dh1 = (d @ _v(w2, 2 * H, F_).t()) * _gelu_grad(_v(h1, B * T, 2 * H))
        _v(dq, B * T, 2 * H).copy_(dh1)
        if dw0 is not None:
            _v(dw0, 2 * H, H).copy_(dh1.t() @ _v(x, B * T, H))
        if db0 is not None:
            _v(db0, 2 * H).copy_(dh1.sum(0))
        if dx is not None:
            _v(dx, B * T, H).copy_(dh1 @ _v(w0, 2 * H, H))


@contextlib.contextmanager
def emulated(emulator_class=FrozenEmulator):
    with deterministic_emulator.emulated(emulator_class) as emu:
        yield emu

