"""Stand-alone `ConvSequence.forward` (reference: bm/models/common.py:142-151) as ONE autograd function over the same
CUDA kernels the brain encoder uses (tensor-core implicit-GEMM convolutions with fused BatchNorm statistics / GLU, tensor-core
weight gradients, FP32-FMA kernels for shapes outside the tensor-core tiling) -- the `DeepMel` feature model
(bm/models/features.py:15-35) is exactly this.

x [B, C0, T] (channel-major, like every tensor the reference hands to a model) is transposed once to channels-last, the
first layer's input channels zero-padded to the tensor-core granularity; every layer is
    y = conv_k(x);  x = act(bn(y)) [if the layer has an activation]  (+ x_prev if skip and the shapes agree);  GLU block
and the result is transposed back to [B, C_last, T].  Backward is hand-written (no autograd through the layers).
There is no CPU path: CUDA tensors only.
"""
from __future__ import annotations

import typing as tp

import torch

from . import _lib
from ._lib import call, ptr, stream
from .functional import _Conv, _Needs, _empty, _reducing_call, _round_up, tc_status_tensor

ACT_GELU, ACT_LRELU, ACT_NONE = 0, 1, 2


class SequencePlan(tp.NamedTuple):
    dilations: tp.List[int]
    glu_after: tp.List[bool]
    has_act: tp.List[bool]            # layer k ends with (BatchNorm +) activation (activation_on_last, common.py:112)
    batch_norm: bool
    act_code: int
    act_slope: float
    skip: bool
    training: bool
    bn_eps: float
    bn_momentum: float
    bn_buffers: tp.List[tp.Optional[tp.Tuple[torch.Tensor, torch.Tensor]]]
    use_tensor_cores: bool
    keep_for_backward: bool


def _epilogue_fwd(plan: SequencePlan, y, mean, invstd, gamma, beta, x_old, x_new, rows, C, act):
    if plan.batch_norm and act == ACT_GELU:       # the encoder's tuned BatchNorm+GELU(+skip) kernel
        call("bm_bn_gelu_skip_fwd", ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(x_old), ptr(x_new), rows, C,
             None, stream())
    else:
        call("bm_bn_act_skip_fwd", ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(x_old), ptr(x_new), rows, C,
             act, float(plan.act_slope), stream())


def _sequence_needs(needs_input_grad, plan: SequencePlan) -> _Needs:
    """`_Needs` of a ConvSequence call: front = (x,), layer k = (conv_w, conv_b, gamma, beta) (False where absent)."""
    n = [bool(v) for v in needs_input_grad]
    depth = len(plan.dilations)
    layer, at = [], 2
    for k in range(depth):
        cnt = 4 if (plan.has_act[k] and plan.batch_norm) else 2
        layer.append(tuple(n[at:at + cnt]) + (False,) * (4 - cnt))
        at += cnt
    glu = {}
    for k in range(depth):
        if plan.glu_after[k]:
            glu[k] = tuple(n[at:at + 2])
            at += 2
    below = [n[1]]
    for k in range(depth):
        below.append(below[-1] or any(layer[k]) or any(glu.get(k, ())))
    return _Needs(front=(n[1],), head=(), layer=layer, glu=glu, below=below)


class _ConvSequenceFn(torch.autograd.Function):
    """inputs: plan, x, then per layer (conv_w, conv_b[, gamma, beta]) and, appended in layer order, (glu_w, glu_b).
    Only what requires grad is backpropagated, as in `functional._EncoderFn`: frozen parameters get no gradient work, the
    backward stops at the first layer that still needs a data gradient, and the forward saves only what it reads."""

    @staticmethod
    def forward(ctx, plan: SequencePlan, x_in, *params):
        depth = len(plan.dilations)
        it = iter(params)
        conv_p = []
        for k in range(depth):
            w, b = next(it), next(it)
            gamma = beta = None
            if plan.has_act[k] and plan.batch_norm:
                gamma, beta = next(it), next(it)
            conv_p.append((w, b, gamma, beta))
        glu_p = {k: (next(it), next(it)) for k in range(depth) if plan.glu_after[k]}
        nd = _sequence_needs(ctx.needs_input_grad, plan)
        st = stream()
        x_in = x_in.contiguous()
        B, C0, T = x_in.shape
        rows = B * T
        tc = plan.use_tensor_cores
        save = plan.keep_for_backward and any(ctx.needs_input_grad)
        status = tc_status_tensor(x_in.device)

        # channels-last input, zero-padded to a multiple of 64 channels when the first conv can use the tensor cores
        Cp = _round_up(C0, 64)
        if plan.skip and conv_p[0][0].shape[0] == C0:
            Cp = C0                                         # layer 0 has a residual: its input keeps the true width
        conv0 = _Conv(conv_p[0][0], T, False, tc, pad_cin_to=Cp, want_bwd=save and nd.below[0])
        if not conv0.fwd_tc and Cp != C0:
            Cp = C0
            conv0 = _Conv(conv_p[0][0], T, False, False, want_bwd=save and nd.below[0])
        x = _empty((B, T, Cp), x_in)                               # the transpose writes the pad columns as zeros
        call("bm_transpose_nt_ld", ptr(x_in), B, C0, T, Cp, ptr(x), st)

        max_c = max(w.shape[0] for w, _, _, _ in conv_p)
        stats = _empty((2 * max_c,), x_in, torch.float64)
        layers = []
        for k in range(depth):
            w, b, gamma, beta = conv_p[k]
            conv = conv0 if k == 0 else _Conv(w, T, False, tc, want_bwd=save and nd.below[k])
            keep = save and nd.below[k + 1]          # the backward reaches this layer
            cout = conv.cout
            y = _empty((B, T, cout), x_in)
            skip = plan.skip and conv.cin_true == cout
            has_bn = plan.has_act[k] and plan.batch_norm
            mean = invstd = None
            if has_bn:
                mean, invstd = _empty((cout,), x_in), _empty((cout,), x_in)
                rm, rv = plan.bn_buffers[k]
                if plan.training:
                    conv.forward(x, b.contiguous(), B, T, plan.dilations[k], y, stats, status)
                    call("bm_bn_stats_finalize", ptr(stats), rows, float(plan.bn_eps), float(plan.bn_momentum),
                         ptr(rm), ptr(rv), ptr(mean), ptr(invstd), cout, st)
                else:
                    conv.forward(x, b.contiguous(), B, T, plan.dilations[k], y, None, status)
                    call("bm_bn_eval_stats", ptr(rm), ptr(rv), float(plan.bn_eps), ptr(mean), ptr(invstd), cout, st)
            else:
                conv.forward(x, b.contiguous(), B, T, plan.dilations[k], y, None, status)
            act = plan.act_code if plan.has_act[k] else ACT_NONE
            if has_bn or act != ACT_NONE or skip:
                x_new = _empty((B, T, cout), x_in)
                _epilogue_fwd(plan, y, mean, invstd, None if gamma is None else gamma.contiguous(),
                              None if beta is None else beta.contiguous(), x if skip else None, x_new, rows, cout, act)
            else:
                x_new = y                                   # a bare convolution (DeepMel's last layer)
            # kept: the conv input for its weight gradient, y for the activation backward, x_new for the GLU weight gradient
            rec = dict(x_in=x if nd.layer[k][0] else None, y=y if nd.layer_up(k) else None, mean=mean, invstd=invstd,
                       conv=conv, skip=skip, act=act, has_bn=has_bn, x_new=x_new if nd.glu.get(k, (False,))[0] else None)
            x = x_new
            if plan.glu_after[k]:
                gw, gb = glu_p[k]
                gconv = _Conv(gw, T, True, tc, want_bwd=save and nd.layer_up(k))
                h = _empty((B, T, gconv.cout), x_in) if keep else None
                out = _empty((B, T, gconv.cout // 2), x_in)
                gconv.forward_glu(x, gb.contiguous(), B, T, h, out, status)
                rec.update(h=h, gconv=gconv)
                x = out
            layers.append(rec if keep else None)

        C_last = x.shape[2]
        out_cm = _empty((B, C_last, T), x_in)
        call("bm_transpose_nt", ptr(x), B, T, C_last, ptr(out_cm), st)       # [B, T, C] -> [B, C, T]
        if save:
            ctx.plan = plan
            ctx.needs = nd
            ctx.dims = (B, C0, Cp, T, C_last)
            ctx.saved = dict(layers=layers, conv_p=conv_p, glu_p=glu_p)
        return out_cm

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dout):
        plan: SequencePlan = ctx.plan
        s = ctx.saved
        if s is None:
            raise RuntimeError("brainmagick_b200.ConvSequence: backward through the graph a second time -- the saved "
                               "activations are released by the first backward; retain_graph is not supported")
        B, C0, Cp, T, C_last = ctx.dims
        depth = len(plan.dilations)
        rows = B * T
        st = stream()
        dout = dout.contiguous()
        status = tc_status_tensor(dout.device)
        g = _empty((B, T, C_last), dout)
        call("bm_transpose_nt", ptr(dout), B, C_last, T, ptr(g), st)          # [B, C, T] -> [B, T, C]
        nd: _Needs = ctx.needs
        need_dx = nd.front[0]
        max_c = max(w.shape[0] for w, _, _, _ in s["conv_p"])
        sums = _empty((2 * max_c,), dout, torch.float64)
        layer_grads: tp.List[tp.Any] = [None] * depth
        glu_grads = {k: (None, None) for k in nd.glu}
        for k in reversed(range(depth)):
            w, b, gamma, beta = s["conv_p"][k]
            if not nd.below[k + 1]:
                layer_grads[k] = (None,) * (4 if gamma is not None else 2)
                continue                               # nothing at or below this layer requires grad
            rec = s["layers"][k]
            conv: _Conv = rec["conv"]
            cout = conv.cout
            n_cw, n_cb, n_gamma, n_beta = nd.layer[k]
            if plan.glu_after[k]:
                gconv: _Conv = rec["gconv"]
                n_gw, n_gb = nd.glu[k]
                dh = _empty((B, T, gconv.cout), dout)
                dgb = torch.empty((gconv.cout,), device=dout.device, dtype=torch.float32) if n_gb else None
                _reducing_call("bm_glu_bwd", dout, (rows, gconv.cout // 2), ptr(g), ptr(rec["h"]), rows, gconv.cout // 2,
                               ptr(dh), ptr(dgb), None, st, reduces=n_gb)
                glu_grads[k] = gconv.backward_weight(dh, rec["x_new"], B, T, 1, dout, status, known_dbias=dgb, want_w=n_gw,
                                                     want_b=n_gb)
                if not nd.layer_up(k):
                    layer_grads[k] = (None,) * (4 if gamma is not None else 2)
                    del dh
                    continue
                g = _empty((B, T, gconv.cin), dout)
                gconv.backward_data(dh, None, B, T, 1, g, status)
                del dh
            dgamma = dbeta = None
            if rec["has_bn"]:
                # reduces in training mode; in eval mode only for trainable gamma / beta (else one elementwise pass)
                reduce = plan.training or n_gamma or n_beta
                dy = _empty((B, T, cout), dout)
                dgamma, dbeta = (_empty((cout,), dout), _empty((cout,), dout)) if reduce else (None, None)
                sums_k = sums if reduce else None
                if rec["act"] == ACT_GELU:
                    _reducing_call("bm_bn_gelu_skip_bwd", dout, (rows, cout), ptr(g), ptr(rec["y"]), ptr(rec["mean"]),
                                   ptr(rec["invstd"]), ptr(gamma.contiguous()), ptr(beta.contiguous()),
                                   1 if plan.training else 0, rows, cout, ptr(sums_k), ptr(dy), ptr(dgamma), ptr(dbeta), None,
                                   st, reduces=reduce)
                else:
                    _reducing_call("bm_bn_act_skip_bwd", dout, (rows, cout), ptr(g), ptr(rec["y"]), ptr(rec["mean"]),
                                   ptr(rec["invstd"]), ptr(gamma.contiguous()), ptr(beta.contiguous()),
                                   1 if plan.training else 0, rows, cout, rec["act"], float(plan.act_slope), ptr(sums_k),
                                   ptr(dy), ptr(dgamma), ptr(dbeta), st, reduces=reduce)
                dgamma, dbeta = (dgamma if n_gamma else None), (dbeta if n_beta else None)
            elif rec["act"] != ACT_NONE:
                dy = _empty((B, T, cout), dout)
                call("bm_bn_act_skip_bwd", ptr(g), ptr(rec["y"]), None, None, None, None, 0, rows, cout, rec["act"],
                     float(plan.act_slope), None, ptr(dy), None, None, st)
            else:
                dy = g                                       # bare convolution (+ skip): dL/dy = dL/dx_new
            # with a training-mode BatchNorm behind the conv, sum(dy) is exactly 0: skip the bias reduction
            dcw, dcb = conv.backward_weight(dy, rec["x_in"], B, T, plan.dilations[k], dout, status,
                                            bias_grad_is_zero=bool(rec["has_bn"] and plan.training), want_w=n_cw, want_b=n_cb)
            if not nd.below[k]:
                g = None
            elif rec["skip"]:
                if dy is g:                                  # the in-place reduce-add needs distinct dy and g
                    dy = g.clone()
                conv.backward_data(dy, g, B, T, plan.dilations[k], g, status)
            else:
                g_in = _empty((B, T, conv.cin), dout)
                conv.backward_data(dy, None, B, T, plan.dilations[k], g_in, status)
                g = g_in
            if gamma is not None:
                layer_grads[k] = (dcw, dcb, dgamma, dbeta)
            else:
                layer_grads[k] = (dcw, dcb)
            del dy

        dx = None
        if need_dx:
            dx_full = _empty((B, Cp, T), dout)
            call("bm_transpose_nt", ptr(g), B, T, Cp, ptr(dx_full), st)       # [B, T, Cp] -> [B, Cp, T]
            dx = dx_full[:, :C0].contiguous() if Cp != C0 else dx_full
        grads: tp.List[tp.Any] = [None, dx]
        for k in range(depth):
            grads.extend(layer_grads[k])
        for k in range(depth):
            if plan.glu_after[k]:
                grads.extend(glu_grads[k])
        ctx.saved = None
        return tuple(grads)


def _require_cuda(x: torch.Tensor) -> None:
    if not x.is_cuda:
        raise RuntimeError("brainmagick_b200.ConvSequence runs on CUDA (sm_90a) only; there is no CPU fallback")


def conv_sequence(module, x: torch.Tensor) -> torch.Tensor:
    """`ConvSequence.forward(x)` for a `brainmagick_b200.common.ConvSequence` (or `features.DeepMel`) module."""
    _require_cuda(x)
    if x.dtype != torch.float32:
        raise TypeError("brainmagick_b200.ConvSequence computes in fp32, like the reference")
    _lib.load()
    params: tp.List[torch.Tensor] = []
    bn_buffers: tp.List[tp.Any] = []
    bn0 = None
    for k, block in enumerate(module.sequence):
        conv = block[0]
        params += [conv.weight, conv.bias]
        if module.has_act[k] and module.batch_norm:
            bn = block[1]
            if bn0 is None:
                bn0 = bn
            params += [bn.weight, bn.bias]
            bn_buffers.append((bn.running_mean, bn.running_var))
        else:
            bn_buffers.append(None)
    for glu in module.glus:
        if glu is not None:
            params += [glu[0].weight, glu[0].bias]
    if bn0 is not None and bn0.momentum is None:
        raise NotImplementedError("BatchNorm cumulative-average mode (momentum=None)")
    plan = SequencePlan(
        dilations=list(module.dilations), glu_after=module.glu_after(), has_act=list(module.has_act),
        batch_norm=module.batch_norm, act_code=module.act_code, act_slope=module.act_slope, skip=module.skip,
        training=module.training, bn_eps=bn0.eps if bn0 is not None else 0.0,
        bn_momentum=bn0.momentum if bn0 is not None else 0.0, bn_buffers=bn_buffers,
        use_tensor_cores=getattr(module, "use_tensor_cores", True), keep_for_backward=torch.is_grad_enabled())
    out = _ConvSequenceFn.apply(plan, x, *params)
    if module.training and module.batch_norm:
        for k, block in enumerate(module.sequence):       # nn.BatchNorm1d bookkeeping (running stats updated on device)
            if module.has_act[k]:
                block[1].num_batches_tracked += 1
    return out
