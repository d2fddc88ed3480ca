"""Stand-alone `ConvSequence.forward` (reference: bm/models/common.py:142-151) as ONE autograd function over the same
CUDA kernels the brain encoder uses (tensor-core implicit-GEMM convolutions with fused BatchNorm statistics / GLU, tensor-core
weight gradients, FP32-FMA kernels for shapes outside the tensor-core tiling) -- the `DeepMel` feature model
(bm/models/features.py:15-35) is exactly this.

x [B, C0, T] (channel-major, like every tensor the reference hands to a model) is transposed once to channels-last, the
first layer's input channels zero-padded to the tensor-core granularity; every layer is
    y = conv_k(x);  x = act(bn(y)) [if the layer has an activation]  (+ x_prev if skip and the shapes agree);  GLU block
with, where the module has them, a rewrite conv (1x1 + LeakyReLU) after the activation and the LayerScale / post_skip gains
in front of the residual add;
and the result is transposed back to [B, C_last, T].  The layers run on the conv stack SimpleConv's encoder uses
(`functional.conv_stack_forward` / `conv_stack_backward`); backward is hand-written (no autograd through the layers).
There is no CPU path: CUDA tensors only.
"""
from __future__ import annotations

import typing as tp

import torch

from . import _lib
from ._lib import call, ptr, stream
from .functional import (SequencePlan, _Needs, _empty, bn_count_batches, bn_plan_fields, bn_sync_groups,
                         conv_stack_backward, conv_stack_forward, layer_width, replays_bf16, stack_conv0,
                         tc_status_tensor)


def _present(plan: SequencePlan, k: int) -> tp.List[bool]:
    """Which entries of layer k's parameter tuple (`functional.layer_width`) the call passes: conv_w, conv_b, then gamma,
    beta with a BatchNorm, then on a layer with a residual-branch option rewrite_w, rewrite_b, layer_scale, post_skip_w."""
    bn = plan.has_act[k] and plan.batch_norm
    out = [True, True, bn, bn]
    if layer_width(plan, k) > 4:
        rewrite, scale, post = plan.residual[k]
        out += [rewrite, rewrite, scale, post]
    return out


def _sequence_needs(needs_input_grad, plan: SequencePlan) -> _Needs:
    """`_Needs` of a ConvSequence call: front = (x,), layer k = (conv_w, conv_b, gamma, beta[, rewrite_w, rewrite_b,
    layer_scale, post_skip_w]) (False where absent)."""
    n = [bool(v) for v in needs_input_grad]
    depth = len(plan.dilations)
    layer, at = [], 2
    for k in range(depth):
        flags = []
        for present in _present(plan, k):
            flags.append(present and n[at])
            at += int(present)
        layer.append(tuple(flags))
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
    """inputs: plan, x, then per layer (conv_w, conv_b[, gamma, beta][, rewrite_w, rewrite_b][, layer_scale][, post_skip_w])
    and, appended in layer order, (glu_w, glu_b).
    Only what requires grad is backpropagated, as in `functional._EncoderFn`: frozen parameters get no gradient work, the
    backward stops at the first layer that still needs a data gradient, and the forward saves only what it reads."""

    @staticmethod
    def forward(ctx, plan: SequencePlan, x_in, *params):
        ctx.bf16 = _lib.bf16()                   # the mode the backward replays
        depth = len(plan.dilations)
        it = iter(params)
        conv_p = []
        for k in range(depth):
            conv_p.append(tuple(next(it) if present else None for present in _present(plan, k)))
        glu_p = {k: (next(it), next(it)) for k in range(depth) if plan.glu_after[k]}
        nd = _sequence_needs(ctx.needs_input_grad, plan)
        st = stream()
        x_in = x_in.contiguous()
        B, C0, T = x_in.shape
        tc = plan.use_tensor_cores
        save = plan.keep_for_backward and any(ctx.needs_input_grad)
        status = tc_status_tensor(x_in.device)

        # channels-last input, zero-padded to a multiple of 64 channels when the first conv can use the tensor cores
        conv0, Cp = stack_conv0(conv_p[0][0], T, C0, tc, plan.skip, save and nd.below[0])
        x = _empty((B, T, Cp), x_in)                               # the transpose writes the pad columns as zeros
        call("bm_transpose_nt_ld", ptr(x_in), B, C0, T, Cp, ptr(x), st)

        x, layers = conv_stack_forward(plan, x, conv0, conv_p, glu_p, nd, save, B, T, status, bare_slope=plan.act_slope)
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
    @replays_bf16
    def backward(ctx, dout):
        plan: SequencePlan = ctx.plan
        s = ctx.saved
        if s is None:
            raise RuntimeError("brainmagick_b200.ConvSequence: backward through the graph a second time -- the saved "
                               "activations are released by the first backward; retain_graph is not supported")
        B, C0, Cp, T, C_last = ctx.dims
        depth = len(plan.dilations)
        st = stream()
        dout = dout.contiguous()
        status = tc_status_tensor(dout.device)
        g = _empty((B, T, C_last), dout)
        call("bm_transpose_nt", ptr(dout), B, C_last, T, ptr(g), st)          # [B, C, T] -> [B, T, C]
        nd: _Needs = ctx.needs
        layer_grads, glu_grads, g = conv_stack_backward(plan, s["conv_p"], s["layers"], g, nd, B, T, status)
        dx = None
        if nd.front[0]:
            dx_full = _empty((B, Cp, T), dout)
            call("bm_transpose_nt", ptr(g), B, T, Cp, ptr(dx_full), st)       # [B, T, Cp] -> [B, Cp, T]
            dx = dx_full[:, :C0].contiguous() if Cp != C0 else dx_full
        grads: tp.List[tp.Any] = [None, dx]
        for k in range(depth):
            grads.extend(gk for gk, present in zip(layer_grads[k], _present(plan, k)) if present)
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
    bns: tp.List[tp.Any] = []
    for k, block in enumerate(module.sequence):
        conv = block[0]
        params += [conv.weight, conv.bias]
        if module.has_act[k] and module.batch_norm:
            bn = block[1]
            params += [bn.weight, bn.bias]
            bns.append(bn)
        else:
            bns.append(None)
        params += [t for t in module.residual_params(k) if t is not None]
    for glu in module.glus:
        if glu is not None:
            params += [glu[0].weight, glu[0].bias]
    residual = module.residual()
    plan = SequencePlan(
        dilations=list(module.dilations), glu_after=module.glu_after(), has_act=list(module.has_act),
        batch_norm=module.batch_norm, act_code=module.act_code, act_slope=module.act_slope, skip=module.skip,
        **bn_plan_fields(bns, module.training), use_tensor_cores=getattr(module, "use_tensor_cores", True),
        keep_for_backward=torch.is_grad_enabled(), residual=residual, rewrite_slope=module.rewrite_slope,
        scale_boost=module.scale_boost(), bn_groups=bn_sync_groups(bns, residual))
    bn_count_batches(bns)           # nn.BatchNorm1d bookkeeping, ahead of the finalize kernels that read it
    return _ConvSequenceFn.apply(plan, x, *params)
