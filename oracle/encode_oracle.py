"""TEST INFRASTRUCTURE ONLY -- CPU restatement of SimpleConv over several input streams, the encoding configuration of the
reference (bm/train.py:61-67, bm/solver.py:283-294 over bm/models/simpleconv.py:150-249):

    streams          every key of in_channels; the sensor front acts on "meg", the others enter their encoder as is
    concatenate      one encoder "concat" over the streams joined in sorted key order               simpleconv.py:150-153,234-236
    join             the encoder outputs joined in sorted key order                                 simpleconv.py:242-243
    linear_out       ConvTranspose1d(final_channels, out_channels, 1) alone                         simpleconv.py:182-184
    complex_out      Conv1d -> activation -> ConvTranspose1d (bm_oracle.head)                       simpleconv.py:185-189
    neither          one encoder whose last conv maps to out_channels, without BatchNorm / act      simpleconv.py:190-193

The encoders are ConvSequence layers (`deepmel_oracle.conv_sequence`, which also covers the bare last layer that the
clip_conv restatement `bm_oracle.conv_sequence` does not have).  Pinned against the verbatim reference by
tests/golden/encode_*.npz (tools/make_encode_golden.py); the GPU tests use it at widths the fixtures cannot hold.

Only `tests/` and the profiles may import this module.
"""
from __future__ import annotations

import typing as tp

import torch
import torch.nn.functional as F

from . import bm_oracle, deepmel_oracle


class EncodeVariant(tp.NamedTuple):
    in_channels: tp.Dict[str, int]
    hidden: tp.Dict[str, int]
    out_channels: int
    n_subjects: int
    depth: int = 10
    concatenate: bool = False
    linear_out: bool = False
    complex_out: bool = True
    merger: bool = True
    merger_channels: int = 270
    merger_pos_dim: int = 2048
    merger_dropout: float = 0.2
    initial_linear: int = 270
    subject_layers: bool = True
    subject_dim: int = 0
    embedding_scale: float = 1.0
    glu: int = 2
    glu_context: int = 1
    skip: bool = True
    kernel_size: int = 3
    dilation_period: int = 5

    def kwargs(self) -> dict:
        """SimpleConv keyword arguments (the clip_conv options of conf/model/clip_conv.yaml, GELU, BatchNorm)"""
        kw = self._asdict()
        kw.update(in_channels=dict(self.in_channels), hidden=dict(self.hidden), batch_norm=True, gelu=True,
                  dilation_growth=2)
        return kw

    def front_width(self) -> int:
        c = self.in_channels["meg"]
        if self.merger:
            c = self.merger_channels
        if self.initial_linear:
            c = self.initial_linear
        return c + self.subject_dim

    def sizes(self) -> tp.Dict[str, tp.List[int]]:
        """simpleconv.py:150-159, 190-193: the channel widths of every encoder, in construction order"""
        width = dict(self.in_channels, meg=self.front_width())
        hidden = dict(self.hidden)
        if self.concatenate:
            width = {"concat": sum(width.values())}
            hidden = {"concat": sum(hidden.values())}
        sizes = {name: [width[name]] + [hidden[name]] * self.depth for name in width}
        if not (self.linear_out or self.complex_out):
            assert len(sizes) == 1
            list(sizes.values())[0][-1] = self.out_channels
        return sizes

    def sequence_spec(self, channels) -> deepmel_oracle.SequenceSpec:
        return deepmel_oracle.SequenceSpec(
            channels=tuple(channels), kernel=self.kernel_size, dilation_growth=2, dilation_period=self.dilation_period,
            batch_norm=True, skip=self.skip, activation_on_last=self.linear_out or self.complex_out, glu=self.glu,
            glu_context=self.glu_context, activation="gelu")


def front(p, v: EncodeVariant, meg, rec_positions, rec_of_sample, subject_index, training: bool, ban_centre=None):
    """simpleconv.py:207-233 on "meg": merger -> initial_linear -> subject layers -> subject embedding"""
    x = meg
    if v.merger:
        centre = ban_centre if (training and v.merger_dropout) else None
        w = bm_oracle.attention_weights(rec_positions, p["merger.heads"], centre, v.merger_dropout)
        x = torch.einsum("bct,boc->bot", x, w[rec_of_sample])
    if v.initial_linear:
        x = F.conv1d(x, p["initial_linear.0.weight"], p["initial_linear.0.bias"])
    if v.subject_layers:
        x = torch.einsum("bct,bcd->bdt", x, p["subject_layers.weights"][subject_index])
    if v.subject_dim:
        emb = p["subject_embedding.embedding.weight"][subject_index] * v.embedding_scale
        x = torch.cat([x, emb[:, :, None].expand(-1, -1, x.shape[-1])], dim=1)
    return x


def forward(p: tp.Dict[str, torch.Tensor], v: EncodeVariant, inputs: tp.Dict[str, torch.Tensor], rec_positions,
            rec_of_sample, subject_index, training: bool, ban_centre=None, new_stats=None) -> torch.Tensor:
    """simpleconv.py:198-249; parameters under the reference's state_dict names, `inputs` keyed like in_channels."""
    length = inputs["meg"].shape[-1]
    x = dict(inputs)
    x["meg"] = front(p, v, inputs["meg"], rec_positions, rec_of_sample, subject_index, training, ban_centre)
    if v.concatenate:
        x = {"concat": torch.cat([t for _, t in sorted(x.items())], dim=1)}
    encoded = {}
    for name, channels in v.sizes().items():
        pre = f"encoders.{name}."
        seq = {k[len(pre):]: t for k, t in p.items() if k.startswith(pre)}
        stats = {} if new_stats is not None else None
        encoded[name] = deepmel_oracle.conv_sequence(x[name], seq, v.sequence_spec(channels), training, new_stats=stats)
        if new_stats is not None:
            new_stats.update({pre + k: t for k, t in stats.items()})
    y = torch.cat([t for _, t in sorted(encoded.items())], dim=1)
    if v.linear_out:
        y = F.conv_transpose1d(y, p["final.weight"], p["final.bias"])
    elif v.complex_out:
        y = bm_oracle.head(y, p)
    return y[:, :, :length]
