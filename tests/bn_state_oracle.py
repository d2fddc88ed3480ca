"""TEST INFRASTRUCTURE ONLY -- the CPU / fp64 restatement of ConvSequence and SimpleConv in which every BatchNorm layer
follows its own module, as torch.nn.BatchNorm1d does (torch/nn/modules/batchnorm.py):

    layer in training mode      num_batches_tracked += 1; factor = momentum, or 1 / num_batches_tracked when momentum is
                                None (cumulative average); normalise with the biased batch statistics; running buffers
                                <- (1 - factor) * running + factor * (batch mean, unbiased batch variance)
    layer in eval mode          normalise with the running statistics; nothing is updated
    eps                         the layer's own

`bn` maps a layer's state_dict prefix (e.g. "encoders.meg.sequence.3.1.") to its `Layer`; `state` holds the running
buffers and counters under their state_dict names and is updated in place by a forward, like the module's buffers.  The
layer arithmetic follows `oracle.deepmel_oracle.conv_sequence`, the sensor front and the head `oracle.encode_oracle`.
Pinned against the verbatim reference by tests/golden/bn_state_*.npz (tools/make_bn_state_golden.py).
"""
from __future__ import annotations

import typing as tp

import torch
import torch.nn.functional as F

from oracle import bm_oracle, deepmel_oracle, encode_oracle


class Layer(tp.NamedTuple):
    training: bool
    eps: float
    momentum: tp.Optional[float]


def layers_of(model, prefix: str = "") -> tp.Dict[str, Layer]:
    """The `bn` argument of this module's BatchNorm layers, read from the modules themselves."""
    return {f"{prefix}{name}.": Layer(m.training, m.eps, m.momentum) for name, m in model.named_modules()
            if isinstance(m, torch.nn.BatchNorm1d)}


def batch_norm(x, p, state, pre: str, layer: Layer):
    """One BatchNorm1d layer on x [B, C, T]; p holds weight / bias, state the buffers (updated in place)."""
    if layer.training:
        state[pre + "num_batches_tracked"] = state[pre + "num_batches_tracked"] + 1
        f = layer.momentum if layer.momentum is not None else 1.0 / float(state[pre + "num_batches_tracked"])
        mean = x.mean(dim=(0, 2))
        var = x.var(dim=(0, 2), unbiased=False)
        n = x.shape[0] * x.shape[2]
        state[pre + "running_mean"] = (1 - f) * state[pre + "running_mean"] + f * mean.detach()
        state[pre + "running_var"] = (1 - f) * state[pre + "running_var"] + f * var.detach() * n / (n - 1)
    else:
        mean, var = state[pre + "running_mean"], state[pre + "running_var"]
    x = (x - mean[None, :, None]) / torch.sqrt(var[None, :, None] + layer.eps)
    return x * p[pre + "weight"][None, :, None] + p[pre + "bias"][None, :, None]


def conv_sequence(x, p, spec: deepmel_oracle.SequenceSpec, bn: tp.Dict[str, Layer], state, prefix: str = ""):
    """`deepmel_oracle.conv_sequence` with BatchNorm layer k following bn[prefix + f"sequence.{k}.1."]."""
    for k, dil in enumerate(spec.dilations()):
        old = x
        pre = f"{prefix}sequence.{k}."
        x = F.conv1d(x, p[pre + "0.weight"], p[pre + "0.bias"], padding=(spec.kernel // 2) * dil, dilation=dil)
        if spec.activation_on_last or k != spec.depth - 1:
            if spec.batch_norm:
                x = batch_norm(x, p, state, pre + "1.", bn[pre + "1."])
            x = F.gelu(x) if spec.activation == "gelu" else F.leaky_relu(x, spec.leakiness)
        if spec.skip and x.shape == old.shape:
            x = x + old
        if spec.glu and (k + 1) % spec.glu == 0:
            h = F.conv1d(x, p[f"{prefix}glus.{k}.0.weight"], p[f"{prefix}glus.{k}.0.bias"], padding=spec.glu_context)
            a, b = h.chunk(2, dim=1)
            x = a * torch.sigmoid(b)
    return x


def simpleconv(p, v: encode_oracle.EncodeVariant, inputs, rec_positions, rec_of_sample, subject_index, training: bool,
               bn: tp.Dict[str, Layer], state, ban_centre=None):
    """`encode_oracle.forward` with per-layer BatchNorm; `training` is the model's own flag (the merger's dropout)."""
    length = inputs["meg"].shape[-1]
    x = dict(inputs)
    x["meg"] = encode_oracle.front(p, v, inputs["meg"], rec_positions, rec_of_sample, subject_index, training, ban_centre)
    if v.concatenate:
        x = {"concat": torch.cat([t for _, t in sorted(x.items())], dim=1)}
    encoded = {name: conv_sequence(x[name], p, v.sequence_spec(channels), bn, state, prefix=f"encoders.{name}.")
               for name, channels in v.sizes().items()}
    y = torch.cat([t for _, t in sorted(encoded.items())], dim=1)
    if v.linear_out:
        y = F.conv_transpose1d(y, p["final.weight"], p["final.bias"])
    elif v.complex_out:
        y = bm_oracle.head(y, p)
    return y[:, :, :length]


def split_state(sd: tp.Dict[str, torch.Tensor], dtype=torch.float64):
    """state_dict -> (parameters as leaves requiring grad, buffers), floating point in `dtype`"""
    params, state = {}, {}
    for k, t in sd.items():
        if "running" in k or "num_batches" in k:
            state[k] = t.clone() if "num_batches" in k else t.to(dtype).clone()
        else:
            params[k] = t.to(dtype).clone().requires_grad_(True)
    return params, state
