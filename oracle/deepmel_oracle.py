"""TEST INFRASTRUCTURE ONLY -- CPU restatement of a stand-alone ConvSequence / the DeepMel feature model
(SURVEY.md 8(f) row 3).

    bm/models/common.py:79-151     ConvSequence: per layer Conv1d(k, dilation, pad = k//2 * dilation); BatchNorm1d and the
                                   activation unless it is the last layer with activation_on_last=False; `+ old_x` when
                                   skip and the shapes agree; a Conv1d(1 + 2*glu_context) + GLU(dim=1) block after every
                                   `glu`-th layer; default activation LeakyReLU(leakiness)
    bm/models/features.py:15-35    DeepMel = ConvSequence([n_in] + [hidden]*(layers-1) + [n_out], **kwargs)
    bm/solver.py:304-320           candidates = feature_model(features); ClipLoss back-propagates into them
Parameters use the reference's `state_dict` names (`sequence.{k}.0.weight`, `sequence.{k}.1.{weight,bias,running_*}`,
`glus.{k}.0.weight`).  Backward = torch autograd over this restatement.  Pinned against the verbatim reference classes
through `tests/golden/deepmel_small.npz` (`oracle/make_golden.py`).

Only `tests/`, `__graft_entry__.smoke()` and the CPU legs of `bench.py` may import this module.
"""
from __future__ import annotations

import typing as tp

import torch
import torch.nn.functional as F


class SequenceSpec(tp.NamedTuple):
    channels: tp.Tuple[int, ...]
    kernel: int = 3
    dilation_growth: int = 2
    dilation_period: tp.Optional[int] = 5
    batch_norm: bool = True
    skip: bool = True
    activation_on_last: bool = False
    glu: int = 2
    glu_context: int = 1
    activation: str = "lrelu"        # "lrelu" (LeakyReLU(leakiness), the ConvSequence default) or "gelu"
    leakiness: float = 0.0
    bn_eps: float = 1e-5
    bn_momentum: float = 0.1

    @property
    def depth(self) -> int:
        return len(self.channels) - 1

    def dilations(self) -> tp.List[int]:
        out, d = [], 1
        for k in range(self.depth):
            if self.dilation_period and k % self.dilation_period == 0:
                d = 1
            out.append(d)
            d *= self.dilation_growth
        return out


def deep_mel_spec(n_in_channels, n_hidden_channels, n_hidden_layers, n_out_channels, **kw) -> SequenceSpec:
    channels = (n_in_channels,) + (n_hidden_channels,) * (n_hidden_layers - 1) + (n_out_channels,)
    kw.pop("stride", None)
    return SequenceSpec(channels=channels, **kw)


def convseq_spec(channels, activation: tp.Optional[str] = None, kernel: int = 4, dilation_growth: int = 1,
                 dilation_period: tp.Optional[int] = None, batch_norm: bool = False, skip: bool = False,
                 activation_on_last: bool = True, glu: int = 0, glu_context: int = 0, leakiness: float = 0.0,
                 stride: int = 1) -> SequenceSpec:
    """SequenceSpec of `ConvSequence(channels, ...)` with the reference constructor's defaults (common.py:81-87).
    `activation`: None (LeakyReLU(leakiness)), "relu" (nn.ReLU), "leaky_relu" (nn.LeakyReLU: slope 0.01) or "gelu"."""
    assert stride == 1
    slope = {None: leakiness, "relu": 0.0, "leaky_relu": 0.01, "gelu": 0.0}[activation]
    return SequenceSpec(channels=tuple(channels), kernel=kernel, dilation_growth=dilation_growth,
                        dilation_period=dilation_period, batch_norm=batch_norm, skip=skip,
                        activation_on_last=activation_on_last, glu=glu, glu_context=glu_context,
                        activation="gelu" if activation == "gelu" else "lrelu", leakiness=slope)


def conv_sequence(x: torch.Tensor, p: tp.Dict[str, torch.Tensor], spec: SequenceSpec, training: bool,
                  new_stats: tp.Optional[dict] = None, pre_act: tp.Optional[list] = None) -> torch.Tensor:
    """x [B, C0, T] -> [B, C_last, T].  `new_stats` (optional dict) receives the BatchNorm running statistics a
    training forward would leave behind; `pre_act` (optional list) the input of every activation, detached."""
    for k, dil in enumerate(spec.dilations()):
        old = x
        pre = f"sequence.{k}."
        x = F.conv1d(x, p[pre + "0.weight"], p[pre + "0.bias"], padding=(spec.kernel // 2) * dil, dilation=dil)
        if spec.activation_on_last or k != spec.depth - 1:
            if spec.batch_norm:
                if training:
                    mean = x.mean(dim=(0, 2))
                    var = x.var(dim=(0, 2), unbiased=False)
                    if new_stats is not None:
                        n = x.shape[0] * x.shape[2]
                        m = spec.bn_momentum
                        new_stats[pre + "1.running_mean"] = (1 - m) * p[pre + "1.running_mean"] + m * mean.detach()
                        new_stats[pre + "1.running_var"] = (1 - m) * p[pre + "1.running_var"] + \
                            m * var.detach() * n / (n - 1)
                else:
                    mean, var = p[pre + "1.running_mean"], p[pre + "1.running_var"]
                x = (x - mean[None, :, None]) / torch.sqrt(var[None, :, None] + spec.bn_eps)
                x = x * p[pre + "1.weight"][None, :, None] + p[pre + "1.bias"][None, :, None]
            if pre_act is not None:
                pre_act.append(x.detach())
            x = F.gelu(x) if spec.activation == "gelu" else F.leaky_relu(x, spec.leakiness)
        if spec.skip and x.shape == old.shape:
            x = x + old
        if spec.glu and (k + 1) % spec.glu == 0:
            h = F.conv1d(x, p[f"glus.{k}.0.weight"], p[f"glus.{k}.0.bias"], padding=spec.glu_context)
            a, b = h.chunk(2, dim=1)
            x = a * torch.sigmoid(b)
    return x
