"""A torch-CPU emulation of the FP32 entry points of include/bm_b200.h -- TEST INFRASTRUCTURE, never a product path.

Purpose: the host side (which entry points are called, with which buffers, leading dimensions, strides and in which order,
and where each gradient ends up) is Python that changes between GPU sessions.  The CUDA kernels behind the entry points
below are verified on an H100 (`-m gpu` tests) but new COMPOSITIONS of them cannot be when no GPU is at hand.  This module
implements each entry point's documented contract with torch CPU ops on the very buffers the host code passes, so the whole
drop-in can be run here against the verbatim-reference fixtures:
  * the fixtures the GPU path is known to pass must also pass on the emulator (that validates the emulator's reading of the
    contracts), and then
  * compositions that have not had a GPU run yet (ablation rows, ...) are checked numerically against their fixtures.
The tensor-core entry points are emulated with the same contracts in exact fp32 (no 3xTF32 rounding), which lets the
all-tensor-core host path (paddings, operand layouts, slices) run on the CPU as well; the shape gates (`*_supported`,
workspace sizes) are always answered by the real library.  Buffers are interpreted through the integer arguments only
(flat views), exactly like the C side.
"""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

INVALID = -0.1


def _v(t, *shape):
    """The first prod(shape) elements of buffer t as a view of that shape."""
    n = 1
    for s in shape:
        n *= s
    flat = t.reshape(-1)
    assert flat.numel() >= n, f"buffer of {flat.numel()} elements is too small for {shape}"
    return flat[:n].view(*shape)


def _ld(t, rows, ld, width):
    """rows x width window of a row-major buffer with leading dimension ld."""
    return _v(t, rows, ld)[:, :width]


def _gelu_grad(z):
    cdf = 0.5 * (1 + torch.erf(z / math.sqrt(2.0)))
    pdf = torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)
    return cdf + z * pdf


def _act(act, z, slope):
    if act == 0:
        return F.gelu(z)
    if act == 1:
        return torch.where(z > 0, z, z * slope)
    return z


def _act_grad(act, z, slope):
    if act == 0:
        return _gelu_grad(z)
    if act == 1:
        return torch.where(z > 0, torch.ones_like(z), torch.full_like(z, slope))
    return torch.ones_like(z)


def _conv(x, w_oik, dilation):
    """x [B,T,Cin] channels-last, w [Cout,Cin,Kw] -> [B,T,Cout] ('same' zero padding)."""
    kw = w_oik.shape[2]
    return F.conv1d(x.transpose(1, 2), w_oik, None, padding=(kw // 2) * dilation, dilation=dilation).transpose(1, 2)


class Emulator:
    # ---------------------------------------------------------------- K1
    def bm_attention_weights_fwd(self, positions, freq, heads, ban_centre, radius, R, C, O, P, emb, weights, stream):
        pos = _v(positions, R, C, 2)
        f = freq.reshape(-1)
        n = f.numel()
        x, y = pos[..., 0] + 0.2, pos[..., 1] + 0.2
        loc = (x[..., None, None] * f[:, None] + y[..., None, None] * f[None, :]).reshape(R, C, n * n)
        e = torch.cat([loc.cos(), loc.sin()], dim=-1)
        _v(emb, R, C, P).copy_(e)
        scores = torch.einsum("rcp,op->roc", e, _v(heads, O, P))
        masked = (pos == INVALID).all(-1)
        if ban_centre is not None:
            c = ban_centre.reshape(2)
            d = pos - c
            masked = masked | (torch.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) <= radius)
        scores = scores.masked_fill(masked[:, None, :], float("-inf"))
        _v(weights, R, O, C).copy_(torch.softmax(scores, dim=2))

    def bm_attention_weights_bwd(self, dweights, weights, emb, R, C, O, P, dscores, dheads, stream):
        w, dw = _v(weights, R, O, C), _v(dweights, R, O, C)
        ds = w * (dw - (dw * w).sum(-1, keepdim=True))
        _v(dscores, R, O, C).copy_(ds)
        _v(dheads, O, P).copy_(torch.einsum("roc,rcp->op", ds, _v(emb, R, C, P)))

    # ---------------------------------------------------------------- K2 stages
    def bm_sensor_mix_fwd(self, meg, weights, rec_of_sample, B, C, T, O, ld_u, u, stream):
        w = _v(weights, weights.numel() // (O * C), O, C)[rec_of_sample.long()[:B]]
        out = torch.einsum("bct,boc->bto", _v(meg, B, C, T), w)
        _ld(u, B * T, ld_u, O).copy_(out.reshape(B * T, O))

    def bm_initial_linear_fwd(self, u, ld_u, il_w, il_b, B, T, O, IL, ld_v, v, stream):
        _ld(v, B * T, ld_v, IL).copy_(_ld(u, B * T, ld_u, O) @ _v(il_w, IL, O).t() + _v(il_b, IL))

    def bm_subject_layers_fwd(self, v, ld_v, subj_w, subject, B, T, IL, D, ld_x0, x0, stream):
        S = subj_w.numel() // (IL * D)
        m = _v(subj_w, S, IL, D)[subject.long()[:B]]
        vv = _ld(v, B * T, ld_v, IL).reshape(B, T, IL)
        _ld(x0, B * T, ld_x0, D).copy_(torch.einsum("btp,bpd->btd", vv, m).reshape(B * T, D))

    def bm_subject_layers_bwd(self, dx0, ld_x0, v, ld_v, subj_w, subject, subj_order, subj_off, B, T, IL, D, S, ld_dv, dv,
                              d_subj_w, stream):
        g = _ld(dx0, B * T, ld_x0, D).reshape(B, T, D)
        vv = _ld(v, B * T, ld_v, IL).reshape(B, T, IL)
        subj = subject.long()[:B]
        order, off = subj_order.long(), subj_off.long()
        assert off[0] == 0 and off[S] == B and sorted(order.tolist()) == list(range(B))
        for s in range(S):
            assert (subj[order[off[s]:off[s + 1]]] == s).all(), "CSR grouping by subject is inconsistent"
        m = _v(subj_w, S, IL, D)[subj]
        _ld(dv, B * T, ld_dv, IL).copy_(torch.einsum("btd,bpd->btp", g, m).reshape(B * T, IL))
        per_sample = torch.einsum("btp,btd->bpd", vv, g)
        _v(d_subj_w, S, IL, D).copy_(torch.zeros(S, IL, D).index_add_(0, subj, per_sample))

    def bm_initial_linear_bwd(self, dv, ld_dv, u, ld_u, il_w, B, T, O, IL, ld_du, du, d_il_w, d_il_b, stream):
        g = _ld(dv, B * T, ld_dv, IL)
        uu = _ld(u, B * T, ld_u, O)
        _ld(du, B * T, ld_du, O).copy_(g @ _v(il_w, IL, O))
        _v(d_il_w, IL, O).copy_(g.t() @ uu)
        _v(d_il_b, IL).copy_(g.sum(0))

    def bm_sensor_mix_bwd(self, du, ld_du, meg, rec_order, rec_off, B, C, T, O, R, d_weights, stream):
        g = _ld(du, B * T, ld_du, O).reshape(B, T, O)
        per_sample = torch.einsum("bto,bct->boc", g, _v(meg, B, C, T))
        order, off = rec_order.long(), rec_off.long()
        out = torch.zeros(R, O, C)
        for r in range(R):
            out[r] = per_sample[order[off[r]:off[r + 1]]].sum(0)
        _v(d_weights, R, O, C).copy_(out)

    def bm_sensor_chain_fwd(self, meg, weights, rec_of_sample, il_w, il_b, subj_w, subject, B, C, T, O, IL, D, ld_x0, u, v,
                            x0, stream):
        self.bm_sensor_mix_fwd(meg, weights, rec_of_sample, B, C, T, O, O, u, stream)
        self.bm_initial_linear_fwd(u, O, il_w, il_b, B, T, O, IL, IL, v, stream)
        self.bm_subject_layers_fwd(v, IL, subj_w, subject, B, T, IL, D, ld_x0, x0, stream)

    def bm_sensor_chain_bwd(self, dx0, meg, il_w, subj_w, subject, u, v, subj_order, subj_off, rec_order, rec_off, B, C, T,
                            O, IL, D, ld_x0, S, R, dv, du, d_subj_w, d_il_w, d_il_b, d_weights, stream):
        self.bm_subject_layers_bwd(dx0, ld_x0, v, IL, subj_w, subject, subj_order, subj_off, B, T, IL, D, S, IL, dv, d_subj_w,
                                   stream)
        self.bm_initial_linear_bwd(dv, IL, u, O, il_w, B, T, O, IL, O, du, d_il_w, d_il_b, stream)
        self.bm_sensor_mix_bwd(du, O, meg, rec_order, rec_off, B, C, T, O, R, d_weights, stream)

    # ---------------------------------------------------------------- K3 / K4
    def bm_conv_weight_prep(self, w, Cout, Cin, Kw, wf, wb, stream):
        ww = _v(w, Cout, Cin, Kw)
        if wf is not None:
            _v(wf, Kw, Cin, Cout).copy_(ww.permute(2, 1, 0))
        if wb is not None:
            _v(wb, Kw, Cout, Cin).copy_(ww.permute(2, 0, 1))

    def bm_tc_weight_split(self, w, Cout, Cin, Kw, f_hi, f_lo, g_hi, g_lo, stream):
        ww = _v(w, Cout, Cin, Kw)

        def split(x):
            hi = ((x.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
            return hi, x - hi
        if f_hi is not None:
            hi, lo = split(ww.permute(2, 0, 1).contiguous())
            _v(f_hi, Kw, Cout, Cin).copy_(hi if f_lo is not None else ww.permute(2, 0, 1))
            if f_lo is not None:
                _v(f_lo, Kw, Cout, Cin).copy_(lo)
        if g_hi is not None:
            hi, lo = split(ww.permute(2, 1, 0).contiguous())
            _v(g_hi, Kw, Cin, Cout).copy_(hi if g_lo is not None else ww.permute(2, 1, 0))
            if g_lo is not None:
                _v(g_lo, Kw, Cin, Cout).copy_(lo)

    def bm_conv1d_fwd(self, x, wf, bias, B, T, Cin, Cout, Kw, dilation, y, stats, stream):
        w = _v(wf, Kw, Cin, Cout).permute(2, 1, 0)
        out = _conv(_v(x, B, T, Cin), w, dilation)
        if bias is not None:
            out = out + _v(bias, Cout)
        _v(y, B, T, Cout).copy_(out)
        if stats is not None:
            o = out.reshape(-1, Cout).double()
            _v(stats, 2 * Cout).copy_(torch.cat([o.sum(0), (o * o).sum(0)]))

    def bm_bn_stats_finalize(self, stats, n, eps, momentum, running_mean, running_var, mean, invstd, C, stream):
        st = _v(stats, 2 * C)
        m = st[:C] / n
        var = (st[C:] / n - m * m).clamp_min(0)
        _v(mean, C).copy_(m.float())
        _v(invstd, C).copy_((1.0 / torch.sqrt(var + eps)).float())
        if running_mean is not None:
            unb = var * n / (n - 1) if n > 1 else var
            _v(running_mean, C).mul_(1 - momentum).add_(momentum * m.float())
            _v(running_var, C).mul_(1 - momentum).add_(momentum * unb.float())

    def bm_bn_eval_stats(self, running_mean, running_var, eps, mean, invstd, C, stream):
        _v(mean, C).copy_(_v(running_mean, C))
        _v(invstd, C).copy_(1.0 / torch.sqrt(_v(running_var, C) + eps))

    def bm_bn_act_skip_fwd(self, y, mean, invstd, gamma, beta, x_old, x_new, rows, C, act, slope, stream):
        z = _v(y, rows, C)
        if mean is not None:
            z = (z - _v(mean, C)) * _v(invstd, C) * _v(gamma, C) + _v(beta, C)
        a = _act(act, z, slope)
        if x_old is not None:
            a = a + _v(x_old, rows, C)
        _v(x_new, rows, C).copy_(a)

    def bm_bn_gelu_skip_fwd(self, y, mean, invstd, gamma, beta, x_old, x_new, rows, C, amax_out, stream):
        self.bm_bn_act_skip_fwd(y, mean, invstd, gamma, beta, x_old, x_new, rows, C, 0, 0.0, stream)
        self._amax_out(amax_out, _v(x_new, rows * C))

    @staticmethod
    def _amax_out(cell, values):
        """The producers' `amax_out`: max |output| of what they have just written."""
        if cell is not None:
            v = values.abs()
            v = v[~torch.isnan(v)]
            _v(cell, 1).fill_(float(v.max()) if v.numel() else 0.0)

    def bm_bn_act_skip_bwd(self, g, y, mean, invstd, gamma, beta, batch_stats, rows, C, act, slope, sums, dy, dgamma, dbeta,
                           stream):
        gg, yy = _v(g, rows, C).clone(), _v(y, rows, C)
        if mean is None:
            _v(dy, rows, C).copy_(gg * _act_grad(act, yy, slope))
            return
        yh = (yy - _v(mean, C)) * _v(invstd, C)
        dz = gg * _act_grad(act, yh * _v(gamma, C) + _v(beta, C), slope)
        s1, s2 = dz.double().sum(0), (dz * yh).double().sum(0)
        _v(dbeta, C).copy_(s1.float())
        _v(dgamma, C).copy_(s2.float())
        v = dz
        if batch_stats:
            v = dz - (s1 / rows).float() - yh * (s2 / rows).float()
        _v(dy, rows, C).copy_(_v(gamma, C) * _v(invstd, C) * v)

    def bm_bn_gelu_skip_bwd(self, g, y, mean, invstd, gamma, beta, batch_stats, rows, C, sums, dy, dgamma, dbeta, amax_out,
                            stream):
        self.bm_bn_act_skip_bwd(g, y, mean, invstd, gamma, beta, batch_stats, rows, C, 0, 0.0, sums, dy, dgamma, dbeta, stream)
        self._amax_out(amax_out, _v(dy, rows * C))

    def bm_conv1d_bwd_data(self, dy, wb, addend, B, T, Cin, Cout, Kw, dilation, dx, stream):
        w = _v(wb, Kw, Cout, Cin).permute(1, 2, 0)                        # [Cout, Cin, Kw]
        g = _v(dy, B, T, Cout).transpose(1, 2)
        out = F.conv_transpose1d(g, w, None, padding=(Kw // 2) * dilation, dilation=dilation).transpose(1, 2)
        if addend is not None:
            out = out + _v(addend, B, T, Cin)
        _v(dx, B, T, Cin).copy_(out)

    def bm_conv1d_bwd_weight(self, dy, x, B, T, Cin, Cout, Kw, dilation, dw, db, stream):
        g, xx = _v(dy, B, T, Cout), _v(x, B, T, Cin)
        pad = (Kw // 2) * dilation
        xp = F.pad(xx, (0, 0, pad, pad))
        taps = [torch.einsum("bto,bti->oi", g, xp[:, j * dilation:j * dilation + T]) for j in range(Kw)]
        _v(dw, Cout, Cin, Kw).copy_(torch.stack(taps, dim=2))
        if db is not None:
            _v(db, Cout).copy_(g.reshape(-1, Cout).sum(0))

    def bm_conv1d_glu_fwd(self, x, wf, bias, B, T, Cin, H, Kw, h, out, stream):
        w = _v(wf, Kw, Cin, 2 * H).permute(2, 1, 0)
        hh = _conv(_v(x, B, T, Cin), w, 1) + _v(bias, 2 * H)
        if h is not None:
            _v(h, B, T, 2 * H).copy_(hh)
        _v(out, B, T, H).copy_(hh[..., :H] * torch.sigmoid(hh[..., H:]))

    def bm_glu_bwd(self, g, h, rows, H, dh, dbias, amax_out, stream):
        gg, hh = _v(g, rows, H), _v(h, rows, 2 * H)
        a, b = hh[:, :H], hh[:, H:]
        s = torch.sigmoid(b)
        _v(dh, rows, 2 * H).copy_(torch.cat([gg * s, gg * a * s * (1 - s)], dim=1))
        if dbias is not None:
            _v(dbias, 2 * H).copy_(_v(dh, rows, 2 * H).sum(0))
        self._amax_out(amax_out, _v(dh, rows * 2 * H))

    # ---------------------------------------------------------------- K5
    def bm_head_fwd(self, x, w0, b0, w2, b2, B, T, H, F_, h1, q, est, stream):
        pre = _v(x, B * T, H) @ _v(w0, 2 * H, H).t() + _v(b0, 2 * H)
        if h1 is not None:
            _v(h1, B * T, 2 * H).copy_(pre)
        qq = F.gelu(pre)
        _v(q, B * T, 2 * H).copy_(qq)
        out = qq @ _v(w2, 2 * H, F_) + _v(b2, F_)
        _v(est, B, F_, T).copy_(out.reshape(B, T, F_).transpose(1, 2))

    def bm_head_bwd(self, dest, x, w0, w2, h1, q, B, T, H, F_, dq, dx, dw0, db0, dw2, db2, stream):
        d = _v(dest, B, F_, T).transpose(1, 2).reshape(B * T, F_)
        qq, pre, xx = _v(q, B * T, 2 * H), _v(h1, B * T, 2 * H), _v(x, B * T, H)
        _v(dw2, 2 * H, F_).copy_(qq.t() @ d)
        _v(db2, F_).copy_(d.sum(0))
        dh1 = (d @ _v(w2, 2 * H, F_).t()) * _gelu_grad(pre)
        _v(dq, B * T, 2 * H).copy_(dh1)
        _v(dw0, 2 * H, H).copy_(dh1.t() @ xx)
        _v(db0, 2 * H).copy_(dh1.sum(0))
        _v(dx, B * T, H).copy_(dh1 @ _v(w0, 2 * H, H))

    def bm_channel_mask(self, x, mask, B, C, T, y, stream):
        _v(y, B, C, T).copy_(_v(x, B, C, T) * _v(mask, C)[None, :, None])

    def bm_transpose_nt(self, inp, Z, N, T, out, stream):
        _v(out, Z, T, N).copy_(_v(inp, Z, N, T).transpose(1, 2))

    def bm_transpose_nt_ld(self, inp, Z, N, T, ld_out, out, stream):
        o = _v(out, Z, T, ld_out)
        o[:, :, :N].copy_(_v(inp, Z, N, T).transpose(1, 2))
        o[:, :, N:].zero_()

    # ---------------------------------------------------------------- K6
    def _scores(self, est, cand, Bn, Bc, KT, inv_norm):
        c = _v(cand, Bc, KT)
        return (_v(est, Bn, KT) @ c.t()) * _v(inv_norm, Bc)

    def bm_candidate_inv_norms(self, cand, Bc, KT, ss, inv_norm, stream):
        c = _v(cand, Bc, KT).double()
        s = (c * c).sum(1)
        _v(ss, Bc).copy_(s)
        _v(inv_norm, Bc).copy_(1.0 / (1e-8 + torch.sqrt(s).float()))

    def bm_clip_scores(self, est, cand, Bn, Bc, KT, norms_given, inv_norm, scores, probs, ws, ws_floats, status, stream):
        if not norms_given:
            c = _v(cand, Bc, KT).double()
            _v(inv_norm, Bc).copy_(1.0 / (1e-8 + torch.sqrt((c * c).sum(1)).float()))
        sc = self._scores(est, cand, Bn, Bc, KT, inv_norm)
        _v(scores, Bn, Bc).copy_(sc)
        if probs is not None:
            _v(probs, Bn, Bc).copy_(torch.softmax(sc, dim=1))

    def bm_clip_loss_fwd(self, est, cand, Bn, Bc, KT, target_offset, inv_norm, scores, probs, row_loss, loss, ws, ws_floats,
                         status, stream):
        self.bm_clip_scores(est, cand, Bn, Bc, KT, 0, inv_norm, scores, probs, ws, ws_floats, status, stream)
        sc = _v(scores, Bn, Bc)
        rl = torch.logsumexp(sc, dim=1) - sc[torch.arange(Bn), torch.arange(Bn) + target_offset]
        _v(row_loss, Bn).copy_(rl)
        _v(loss, 1).copy_(rl.double().mean().float().reshape(1))

    def _G(self, probs, inv_norm, gout, Bn, Bc, target_offset):
        p = _v(probs, Bn, Bc).clone()
        p[torch.arange(Bn), torch.arange(Bn) + target_offset] -= 1
        return p * (gout.reshape(-1)[0] / Bn) * _v(inv_norm, Bc)

    def bm_clip_loss_bwd(self, probs, inv_norm, cand, gout, Bn, Bc, KT, target_offset, G, dest, status, stream):
        g = self._G(probs, inv_norm, gout, Bn, Bc, target_offset)
        _v(dest, Bn, KT).copy_(g @ _v(cand, Bc, KT))

    def bm_clip_loss_bwd_cand(self, probs, scores, inv_norm, est, cand, gout, Bn, Bc, KT, target_offset, G, coef, dcand,
                              status, stream):
        g = self._G(probs, inv_norm, gout, Bn, Bc, target_offset)
        norm = 1.0 / _v(inv_norm, Bc) - 1e-8
        cf = torch.where(norm > 0, (g * _v(scores, Bn, Bc)).sum(0) / norm, torch.zeros(Bc))
        _v(dcand, Bc, KT).copy_(g.t() @ _v(est, Bn, KT) - cf[:, None] * _v(cand, Bc, KT))


    # ---------------------------------------------------------------- tensor-core entry points (same contracts, exact fp32)
    def bm_tc_conv1d(self, x, w_hi, w_lo, bias, addend, B, T, Cin, Ntot, Kw, dilation, sign, glu, act, out_tmajor, y, aux,
                     glu_out, stats, status, stream):
        w = _v(w_hi, Kw, Ntot, Cin)
        if w_lo is not None:
            w = w + _v(w_lo, Kw, Ntot, Cin)
        xx = _v(x, B, T, Cin)
        pad = (Kw // 2) * dilation
        xp = F.pad(xx, (0, 0, pad, pad))
        out = torch.zeros(B, T, Ntot)
        for tap in range(Kw):
            shift = sign * (tap - Kw // 2) * dilation
            out += xp[:, pad + shift:pad + shift + T] @ w[tap].t()
        if bias is not None:
            out = out + _v(bias, Ntot)
        if addend is not None:
            out = out + _v(addend, B, T, Ntot)
        if stats is not None:
            o = out.reshape(-1, Ntot).double()
            _v(stats, 2 * Ntot).copy_(torch.cat([o.sum(0), (o * o).sum(0)]))
        if glu:
            H = Ntot // 2
            if y is not None:
                _v(y, B, T, Ntot).copy_(out)
            _v(glu_out, B, T, H).copy_(out[..., :H] * torch.sigmoid(out[..., H:]))
            return
        if act:
            if aux is not None:
                _v(aux, B, T, Ntot).copy_(out)
            out = F.gelu(out)
        if out_tmajor:
            _v(y, B, Ntot, T).copy_(out.transpose(1, 2))
        else:
            _v(y, B, T, Ntot).copy_(out)


    def bm_tc_conv1d_persistent(self, x, w_raw, bias, accumulate, B, T, Cin, Ntot, Kw, dilation, sign, glu, act, out_tmajor,
                                y, aux, glu_out, stats, status, stream):
        self.bm_tc_conv1d(x, w_raw, None, bias, y if accumulate else None, B, T, Cin, Ntot, Kw, dilation, sign, glu, act,
                          out_tmajor, y, aux, glu_out, stats, status, stream)

    # ---- F16 pipe (bm_tc_conv1d_f16, csrc/tc_conv.cuh): power-of-two scale from the tensor's amax, operands as fp16 hi + lo pieces ----
    @staticmethod
    def _f16_scale(amax: float) -> float:
        import math
        if not (amax > 0.0) or math.isinf(amax) or math.isnan(amax):
            return 1.0
        e = math.frexp(amax)[1] - 1                       # amax in [2^e, 2^(e+1))
        if e < -126:                                      # fp32 subnormal: exponent field 0 -> scale 1 (f16_scale_of)
            return 1.0
        return 2.0 ** max(-126, min(127, 14 - e))

    def bm_amax(self, x, n, amax, stream):
        v = _v(x, n).abs()
        v = v[~torch.isnan(v)]
        _v(amax, 1).fill_(float(v.max()) if v.numel() else 0.0)

    def bm_f16_split(self, src, n, amax, hi, lo, stream):
        v = _v(src, n) * self._f16_scale(float(_v(amax, 1)))
        h = v.to(torch.float16)
        _v(hi, n).copy_(h)
        _v(lo, n).copy_((v - h.float()).to(torch.float16))

    def bm_tc_weight_split_f16(self, w, w_amax, Cout, Cin, Kw, f_hi, f_lo, g_hi, g_lo, stream):
        v = _v(w, Cout, Cin, Kw) * self._f16_scale(float(_v(w_amax, 1)))
        h = v.to(torch.float16)
        lo = (v - h.float()).to(torch.float16)
        if f_hi is not None:
            _v(f_hi, Kw, Cout, Cin).copy_(h.permute(2, 0, 1))
            _v(f_lo, Kw, Cout, Cin).copy_(lo.permute(2, 0, 1))
        if g_hi is not None:
            _v(g_hi, Kw, Cin, Cout).copy_(h.permute(2, 1, 0))
            _v(g_lo, Kw, Cin, Cout).copy_(lo.permute(2, 1, 0))

    def bm_tc_conv1d_f16(self, x, x_amax, w_hi, w_lo, w_amax, bias, accumulate, B, T, Cin, Ntot, Kw, dilation, sign, glu, act,
                         out_tmajor, y, aux, glu_out, stats, amax_out, status, stream):
        sx, sw = self._f16_scale(float(_v(x_amax, 1))), self._f16_scale(float(_v(w_amax, 1)))
        n = Kw * Ntot * Cin
        w = (_v(w_hi, n).float() + _v(w_lo, n).float()) / sw            # what the tensor core multiplies by, unscaled
        xv = _v(x, B * T * Cin) * sx
        xh = xv.to(torch.float16)
        xq = (xh.float() + (xv - xh.float()).to(torch.float16).float()) / sx
        self.bm_tc_conv1d(xq.contiguous(), w.contiguous(), None, bias, y if accumulate else None, B, T, Cin, Ntot, Kw,
                          dilation, sign, glu, act, out_tmajor, y, aux, glu_out, stats, status, stream)
        if amax_out is not None:
            assert (glu or act) and not out_tmajor
            self._amax_out(amax_out, _v(glu_out, B * T * (Ntot // 2)) if glu else _v(y, B * T * Ntot))

    def bm_col_stats(self, y, rows, C, stats, stream):
        o = _v(y, rows, C).double()
        _v(stats, 2 * C).copy_(torch.cat([o.sum(0), (o * o).sum(0)]))

    def bm_col_sum(self, x, rows, C, out, stream):
        _v(out, C).copy_(_v(x, rows, C).sum(0))

    def bm_gelu_bwd(self, dq, h, n, dh, stream):
        _v(dh, n).copy_(_v(dq, n).clone() * _gelu_grad(_v(h, n)))

    def bm_tc_wgrad(self, dy, x, B, T, M, N, Ntrue, Kw, dilation, ws, dw, dbias, status, stream):
        g, xx = _v(dy, B, T, M), _v(x, B, T, N)
        pad = (Kw // 2) * dilation
        xp = F.pad(xx, (0, 0, pad, pad))
        taps = [torch.einsum("btm,btn->mn", g, xp[:, j * dilation:j * dilation + T])[:, :Ntrue] for j in range(Kw)]
        _v(dw, M, Ntrue, Kw).copy_(torch.stack(taps, dim=2))
        if dbias is not None:
            _v(dbias, M).copy_(g.reshape(-1, M).sum(0))

    def bm_tc_wgrad_conv(self, dy, x, B, T, M, N, Ntrue, Kw, dilation, ws, dw, status, stream):
        self.bm_tc_wgrad(dy, x, B, T, M, N, Ntrue, Kw, dilation, ws, dw, None, status, stream)

    def _f16_pieces(self, t, n, amax):
        """What the F16-pipe kernels multiply by: (hi + lo) / scale of t * scale, both pieces rounded to fp16."""
        s = self._f16_scale(float(_v(amax, 1)))
        v = _v(t, n) * s
        h = v.to(torch.float16)
        return ((h.float() + (v - h.float()).to(torch.float16).float()) / s).contiguous()

    def bm_tc_wgrad_conv_f16(self, dy, dy_amax, x, x_amax, B, T, M, N, Ntrue, Kw, dilation, ws, dw, status, stream):
        self.bm_tc_wgrad(self._f16_pieces(dy, B * T * M, dy_amax), self._f16_pieces(x, B * T * N, x_amax), B, T, M, N, Ntrue,
                         Kw, dilation, ws, dw, None, status, stream)

    def bm_tc_pointwise_sel(self, x, w_hi, w_lo, wsel, n_sets, B, T, Cin, Ntot, y, status, stream):
        w = _v(w_hi, n_sets, Ntot, Cin) + _v(w_lo, n_sets, Ntot, Cin)
        _v(y, B, T, Ntot).copy_(torch.einsum("btk,bnk->btn", _v(x, B, T, Cin), w[wsel.long()[:B]]))

    def bm_tc_wgrad_grouped(self, dy, x, order, seg_off, G, B, T, M, N, out, status, stream):
        per = torch.einsum("btm,btn->bmn", _v(dy, B, T, M), _v(x, B, T, N))
        mpad = -(-M // 128) * 128
        o = _v(out, G, mpad, N)
        o.zero_()
        order, off = order.long(), seg_off.long()
        for gi in range(G):
            o[gi, :M] = per[order[off[gi]:off[gi + 1]]].sum(0)

    def bm_fourier_emb(self, positions, freq, R, C, P, emb, stream):
        pos = _v(positions, R, C, 2)
        f = freq.reshape(-1)
        n = f.numel()
        x, y = pos[..., 0] + 0.2, pos[..., 1] + 0.2
        loc = (x[..., None, None] * f[:, None] + y[..., None, None] * f[None, :]).reshape(R, C, n * n)
        _v(emb, R, C, P).copy_(torch.cat([loc.cos(), loc.sin()], dim=-1))

    def bm_masked_softmax(self, weights, positions, ban_centre, radius, R, O, C, stream):
        pos = _v(positions, R, C, 2)
        masked = (pos == INVALID).all(-1)
        if ban_centre is not None:
            d = pos - ban_centre.reshape(2)
            masked = masked | (torch.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) <= radius)
        w = _v(weights, R, O, C)
        w.copy_(torch.softmax(w.masked_fill(masked[:, None, :], float("-inf")), dim=2))

    def bm_softmax_bwd(self, weights, dweights, rows, C, dscores, stream):
        w, dw = _v(weights, rows, C), _v(dweights, rows, C)
        _v(dscores, rows, C).copy_(w * (dw - (dw * w).sum(-1, keepdim=True)))

    def bm_head_bwd_params(self, dest, x, h1, q, B, T, H, F_, dq, dw0, db0, dw2, db2, stream):
        d = _v(dest, B, F_, T).transpose(1, 2).reshape(B * T, F_)
        _v(dw2, 2 * H, F_).copy_(_v(q, B * T, 2 * H).t() @ d)
        _v(db2, F_).copy_(d.sum(0))
        dh1 = _v(dq, B * T, 2 * H).clone() * _gelu_grad(_v(h1, B * T, 2 * H))
        _v(dq, B * T, 2 * H).copy_(dh1)
        _v(dw0, 2 * H, H).copy_(dh1.t() @ _v(x, B * T, H))
        _v(db0, 2 * H).copy_(dh1.sum(0))

    # ---------------------------------------------------------------- retrieval evaluation
    def bm_retrieval_probs(self, scores, ld, Bn, n_cols, probs, stream):
        _v(probs, Bn, n_cols).copy_(torch.softmax(_ld(scores, Bn, ld, n_cols), dim=1))

    def bm_rowdot_scaled(self, a, c, Bn, K, own, stream):
        aa, cc = _v(a, Bn, K), _v(c, Bn, K)
        _v(own, Bn).copy_((aa * cc).sum(1) / (1e-8 + cc.norm(dim=1)))

    def bm_retrieval_topk(self, vals, ld, Bn, n_cols, own_values, own_col, is_prob, k, labels, own_labels, targets, top_idx,
                          top_prob, hit, soft, row_max, row_sum, stream):
        v = _ld(vals, Bn, ld, n_cols).clone()
        if own_values is not None:
            v[:, own_col] = _v(own_values, Bn)
        if is_prob:
            p = v
            valid = v >= 0
        else:
            mx = v.max(dim=1).values
            ssum = torch.exp(v - mx[:, None]).sum(1)
            p = torch.exp(v - mx[:, None]) / ssum[:, None]
            valid = torch.ones_like(v, dtype=torch.bool)
            if row_max is not None:
                _v(row_max, Bn).copy_(mx)
            if row_sum is not None:
                _v(row_sum, Bn).copy_(ssum)
        lab = None
        if labels is not None:
            lab = _v(labels, n_cols)[None].repeat(Bn, 1)
            if own_labels is not None:
                lab[:, own_col] = _v(own_labels, Bn)
        for b in range(Bn):
            cols = [int(o) for o in torch.nonzero(valid[b]).flatten()]
            cols.sort(key=lambda o: (-float(v[b, o]), o))            # larger first, ties -> lower column
            first = -1
            for j in range(k):
                col = cols[j] if j < len(cols) else -1
                if top_idx is not None:
                    _v(top_idx, Bn, k)[b, j] = col
                if top_prob is not None:
                    _v(top_prob, Bn, k)[b, j] = float(p[b, col]) if col >= 0 else 0.0
                if col >= 0 and lab is not None and targets is not None and first < 0 and lab[b, col] == targets[b]:
                    first = j
            if hit is not None:
                _v(hit, Bn)[b] = first
            if soft is not None:
                m = (lab[b] == targets[b]) & valid[b]
                _v(soft, Bn)[b] = p[b][m].sum()

    def bm_retrieval_vocab_probs(self, scores, ld, Bn, own_scores, row_max, row_sum, perm, seg, V, own_word, vocab, stream):
        s = _v(scores, Bn, ld)
        out = _v(vocab, Bn, V + 1)
        for b in range(Bn):
            mx, inv = _v(row_max, Bn)[b], 1.0 / _v(row_sum, Bn)[b]
            p_own = torch.exp(_v(own_scores, Bn)[b] - mx) * inv if own_scores is not None else 0.0
            w_own = int(_v(own_word, Bn)[b]) if own_scores is not None else -1
            for w in range(V):
                cols = perm[int(seg[w]):int(seg[w + 1])].long()
                acc = (torch.exp(s[b, cols] - mx) * inv).sum()
                out[b, w] = acc + (p_own if w == w_own else 0.0)
            out[b, V] = p_own if w_own == V else -1.0

    # ---------------------------------------------------------------- batch preparation
    def bm_scale_clamp_crop(self, x, slot, center, scale, B, C, T, t0, T_out, limit, clip, inverse, y, peak_bits, stream):
        xx = _v(x, B, C, T)
        rows = slot.long()[:B] if slot is not None else torch.zeros(B, dtype=torch.long)
        R = center.numel() // C
        ctr, scl = _v(center, R, C), _v(scale, R, C)
        known = rows >= 0
        c = torch.where(known[:, None], ctr[rows.clamp_min(0)], torch.full((B, C), float("nan")))
        s = torch.where(known[:, None], scl[rows.clamp_min(0)], torch.ones(B, C))
        out = (xx * s[:, :, None] + c[:, :, None]) if inverse else (xx - c[:, :, None]) / s[:, :, None]
        if clip:
            out = torch.where(out < -limit, torch.full_like(out, -limit), torch.where(out > limit, torch.full_like(out, limit), out))
        _v(y, B, C, T_out).copy_(out[:, :, t0:t0 + T_out])
        if peak_bits is not None:
            window = out[:, :, t0:t0 + T_out] if clip else out
            peak = torch.nan_to_num(window.abs(), nan=0.0).reshape(B, -1).max(1).values
            _v(peak_bits, B).copy_(peak.view(torch.int32))

    def bm_reject_compact(self, peak_bits, mask, mask_elems, limit, B, keep, keep_rows, n_keep, stream):
        peak = _v(peak_bits, B).view(torch.float32)
        k = ~(peak > limit)
        if mask is not None:
            k = k & _v(mask, B, mask_elems).bool().any(1)
        _v(keep, B).copy_(k)
        rows = torch.nonzero(k).flatten().int()
        _v(keep_rows, B)[:len(rows)] = rows
        _v(n_keep, 1)[0] = len(rows)

    def bm_gather_rows(self, x, rows, n_rows, row_elems, y, stream):
        _v(y, n_rows, row_elems).copy_(x.reshape(-1, row_elems)[rows.long()[:n_rows]])


class _Stream:
    def wait_stream(self, other):
        pass


@contextlib.contextmanager
def emulated():
    """Inside this context the drop-in modules run on CPU tensors through the emulator above."""
    import brainmagick_b200.common as CM
    import brainmagick_b200.convseq as CS
    import brainmagick_b200.functional as BF
    import brainmagick_b200.simpleconv as SC
    emu = Emulator()

    def fake_ptr(t):
        if t is None:
            return None
        assert t.is_contiguous(), "non-contiguous tensor handed to the C ABI"
        return t

    def fake_call(name, *args):
        fn = getattr(emu, name, None)
        if fn is None:
            raise NotImplementedError(f"{name} is not emulated (a tensor-core entry point at fixture size?)")
        fn(*args)

    import brainmagick_b200.norm as NM
    import brainmagick_b200.retrieval as RT
    patches = [(BF, "call", fake_call), (BF, "ptr", fake_ptr), (BF, "stream", lambda: None),
               (CS, "call", fake_call), (CS, "ptr", fake_ptr), (CS, "stream", lambda: None),
               (NM, "call", fake_call), (NM, "ptr", fake_ptr), (NM, "stream", lambda: None),
               (RT, "call", fake_call), (RT, "ptr", fake_ptr), (RT, "stream", lambda: None),
               (RT, "_device", lambda: torch.device("cpu")),
               (BF, "OVERLAP_WGRAD", False), (SC, "_require_cuda", lambda meg: None),
               (CS, "_require_cuda", lambda x: None), (CM, "_require_cuda_fp32", lambda x, who: None),
               (torch.cuda, "current_stream", lambda *a, **k: _Stream())]
    saved = [(mod, name, getattr(mod, name)) for mod, name, _ in patches if hasattr(mod, name)]
    for mod, name, val in patches:
        setattr(mod, name, val)
    BF._status.setdefault(torch.device("cpu"), torch.zeros(1, dtype=torch.int32))
    BF._clip_ws.clear()
    try:
        yield emu
    finally:
        for mod, name, val in saved:
            setattr(mod, name, val)
        BF._status.pop(torch.device("cpu"), None)
        BF._clip_ws.clear()
