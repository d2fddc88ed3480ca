"""Building blocks of the drop-in SimpleConv: same class names, constructor arguments, parameter names/shapes and
init distributions as bm/models/common.py, so reference checkpoints load and `model.merger.heads`,
`model.merger.position_getter.get_positions(batch)`, `model.merger.embedding(positions)` (used by the NMI
notebooks) keep working.  The modules here are *parameter containers + host logic*; the arithmetic of the
training step runs in `functional.encoder_forward` (hand-written CUDA), not in these modules' `forward`.
"""
from __future__ import annotations

import math
import typing as tp

import numpy as np
import torch
from torch import nn

from . import _lib


def _find_layout(info):
    """mne.find_layout(info) -- the only thing the hot path needs from mne (bm/models/common.py:196)."""
    if hasattr(info, "find_layout"):          # brainmagick_b200.synthetic.SyntheticInfo carries its own layout
        return info.find_layout()
    import mne
    return mne.find_layout(info)


def _require_cuda_fp32(x: torch.Tensor, who: str) -> None:
    if x.dtype != torch.float32:
        raise TypeError(f"brainmagick_b200.{who} computes in fp32, got {x.dtype}")
    if not x.is_cuda:
        raise RuntimeError(f"brainmagick_b200.{who} runs on CUDA (sm_90a) only; there is no CPU fallback")


class PositionGetter:
    """2-D sensor positions per recording, min-max normalised to [0,1]; INVALID for sensors missing from the
    layout or padded (reference: bm/models/common.py:183-236)."""
    INVALID = -0.1

    def __init__(self) -> None:
        self._cache: tp.Dict[int, torch.Tensor] = {}
        self._invalid_names: tp.Set[str] = set()

    def get_recording_layout(self, recording) -> torch.Tensor:
        key = recording.recording_index
        hit = self._cache.get(key)
        if hit is not None:
            return hit
        info = recording.mne_info
        layout = _find_layout(info)
        lookup = {name: i for i, name in reversed(list(enumerate(layout.names)))}
        in_layout, in_meg = [], []
        for meg_index, full_name in enumerate(info.ch_names):
            name = full_name.rsplit("-", 1)[0]
            pos_index = lookup.get(name)
            if pos_index is None:
                self._invalid_names.add(name)
                continue
            in_layout.append(pos_index)
            in_meg.append(meg_index)
        positions = torch.full((len(info.ch_names), 2), self.INVALID)
        xy = np.asarray(layout.pos)[in_layout, :2]
        for axis in range(2):
            col = xy[:, axis]
            col = (col - col.min()) / (col.max() - col.min())
            positions[in_meg, axis] = torch.from_numpy(col).float()
        self._cache[key] = positions
        return positions

    def get_positions(self, batch) -> torch.Tensor:
        """Per-sample positions [B, C, 2] (what the reference's notebooks read); built from one row per recording."""
        n_channels = batch.meg.shape[1]
        table, rec_of_sample, _, _ = self.batch_layout(batch, n_channels, batch.meg.device)
        return table[rec_of_sample.long()]

    def is_invalid(self, positions):
        return (positions == self.INVALID).all(dim=-1)

    # ---- fused-path helper: one row per recording present in the batch -------------------------------
    def batch_layout(self, batch, n_channels: int, device):
        """-> rec_positions [R,C,2] (device), rec_of_sample [B] int32, rec_order [B] int32, rec_off [R+1] int32."""
        rec_ids = [r.recording_index for r in batch._recordings]
        uniq = sorted(set(rec_ids))
        row_of = {rid: i for i, rid in enumerate(uniq)}
        table = torch.full((len(uniq), n_channels, 2), self.INVALID)
        first = {}
        for r in batch._recordings:
            first.setdefault(r.recording_index, r)
        for rid, row in row_of.items():
            pos = self.get_recording_layout(first[rid])
            table[row, :len(pos)] = pos
        rows = np.fromiter((row_of[r] for r in rec_ids), dtype=np.int32, count=len(rec_ids))
        order = np.argsort(rows, kind="stable").astype(np.int32)
        off = np.zeros(len(uniq) + 1, dtype=np.int32)
        np.cumsum(np.bincount(rows, minlength=len(uniq)), out=off[1:])
        to = dict(device=device, non_blocking=True)
        return (table.to(**to), torch.from_numpy(rows).to(**to), torch.from_numpy(order).to(**to),
                torch.from_numpy(off).to(**to))


class FourierEmb(nn.Module):
    """Fourier positional embedding over [-margin, 1+margin]^2 (reference: bm/models/common.py:239-271).
    Parameter-free; `forward` is kept (torch ops) only for the analysis notebooks -- the training path computes
    the same embedding inside `bm_attention_weights_fwd`."""

    def __init__(self, dimension: int = 256, margin: float = 0.2):
        super().__init__()
        n_freqs = (dimension // 2) ** 0.5
        assert int(n_freqs ** 2 * 2) == dimension
        self.dimension = dimension
        self.margin = margin

    def frequencies(self) -> torch.Tensor:
        """2*pi*k/width in the reference's fp32 op order (CPU) -- handed to the CUDA kernel as a table."""
        n = int(round((self.dimension // 2) ** 0.5))
        width = 1 + 2 * self.margin
        return 2 * math.pi * torch.arange(float(n)) / width

    def forward(self, positions):
        *lead, two = positions.shape
        assert two == 2
        f = self.frequencies().to(positions)
        shifted = positions + self.margin
        loc = (shifted[..., 0, None, None] * f[:, None] + shifted[..., 1, None, None] * f[None, :])
        loc = loc.reshape(*lead, -1)
        return torch.cat([loc.cos(), loc.sin()], dim=-1)


class ChannelMerger(nn.Module):
    """Spatial attention over sensor positions (reference: bm/models/common.py:312-362).  Holds `heads`."""

    def __init__(self, chout: int, pos_dim: int = 256, dropout: float = 0, usage_penalty: float = 0.,
                 n_subjects: int = 200, per_subject: bool = False):
        super().__init__()
        assert pos_dim % 4 == 0
        if per_subject:
            raise NotImplementedError("merger_per_subject=True is not on the accelerated path (SURVEY 8(f) row 4)")
        if usage_penalty > 0:
            raise NotImplementedError("merger_penalty>0 is not on the accelerated path (SURVEY 8(f) row 4)")
        self.position_getter = PositionGetter()
        self.per_subject = per_subject
        self.heads = nn.Parameter(torch.randn(chout, pos_dim, requires_grad=True))
        self.heads.data /= pos_dim ** 0.5
        self.dropout = dropout
        self.embedding = FourierEmb(pos_dim)
        self.usage_penalty = usage_penalty
        self._penalty = torch.tensor(0.)
        self.ban_centre_override: tp.Optional[torch.Tensor] = None   # test hook: inject the per-forward centre

    @property
    def training_penalty(self):
        # summed into the loss by bm/solver.py:376-378
        return self._penalty.to(next(self.parameters()).device)

    def draw_ban_centre(self, device) -> tp.Optional[torch.Tensor]:
        """One `torch.rand(2, device=meg.device)` per training forward, like bm/models/common.py:342-343."""
        if not (self.training and self.dropout):
            return None
        if self.ban_centre_override is not None:
            return self.ban_centre_override.to(device=device, dtype=torch.float32).contiguous()
        return torch.rand(2, device=device)

    def forward(self, meg, batch):
        """Stand-alone call (bm/models/common.py:334-362): [B, C, T] -> [B, chout, T].  Inside SimpleConv the merger is
        fused into the encoder; this runs the same stage kernels for callers that use the module on its own."""
        from . import functional as BF
        _require_cuda_fp32(meg, "ChannelMerger")
        B, C, T = meg.shape
        pos, rec_of_sample, rec_order, rec_off = self.position_getter.batch_layout(batch, C, meg.device)
        freq = self.embedding.frequencies().to(meg.device)
        return BF.channel_merger_forward(meg, self.heads, pos, rec_of_sample, rec_order, rec_off, freq,
                                         self.draw_ban_centre(meg.device), float(self.dropout))


class ScaledEmbedding(nn.Module):
    """Subject embedding stored divided by `scale` and multiplied back on use, which scales its learning rate
    (reference: bm/models/common.py:28-42).  `forward` is plain torch (a [B, E] lookup); the CUDA encoder appends the rows
    to its channels."""

    def __init__(self, num_embeddings: int, embedding_dim: int, scale: float = 10.):
        super().__init__()
        self.embedding = nn.Embedding(num_embeddings, embedding_dim)
        self.embedding.weight.data /= scale
        self.scale = scale

    @property
    def weight(self):
        return self.embedding.weight * self.scale

    def forward(self, x):
        return self.embedding(x) * self.scale


class SubjectLayers(nn.Module):
    """Per-subject 1x1 linear layer (reference: bm/models/common.py:45-62).  Holds `weights` [S, Cin, Cout]."""

    def __init__(self, in_channels: int, out_channels: int, n_subjects: int, init_id: bool = False):
        super().__init__()
        self.weights = nn.Parameter(torch.randn(n_subjects, in_channels, out_channels))
        if init_id:
            assert in_channels == out_channels
            self.weights.data[:] = torch.eye(in_channels)[None]
        self.weights.data *= 1 / in_channels ** 0.5

    def forward(self, x, subjects):
        """Stand-alone call (bm/models/common.py:55-58): einsum("bct,bcd->bdt", x, weights[subjects]); inside SimpleConv the
        layer is fused into the encoder."""
        from . import functional as BF
        _require_cuda_fp32(x, "SubjectLayers")
        n_subjects = self.weights.shape[0]
        if subjects.numel() and (int(subjects.max()) >= n_subjects or int(subjects.min()) < 0):
            raise IndexError(f"subject index out of range for {n_subjects} subjects")      # the reference's gather raises too
        return BF.subject_layers_forward(x, self.weights, subjects.to(device=x.device, dtype=torch.int32).contiguous())

    def __repr__(self):
        S, C, D = self.weights.shape
        return f"SubjectLayers({C}, {D}, {S})"


class LayerScale(nn.Module):
    """Learnt per-channel gain on a residual branch, `(boost * scale)[:, None] * x` with `scale` initialised to
    init / boost (reference: bm/models/common.py:65-76).  Inside a ConvSequence the gain is applied by the layer's
    CUDA epilogue; `forward` is kept for callers that use the module on its own."""

    def __init__(self, channels: int, init: float = 0.1, boost: float = 5.):
        super().__init__()
        self.scale = nn.Parameter(torch.zeros(channels, requires_grad=True))
        self.scale.data[:] = init / boost
        self.boost = boost

    def forward(self, x):
        return (self.boost * self.scale[:, None]) * x


class ConvSequence(nn.Module):
    """Dilated Conv1d (+ BatchNorm) + activation stack with residual skips and GLU blocks (reference:
    bm/models/common.py:79-151).  Submodule names (`sequence.{k}.{i}`, `glus.{k}.0`) and construction order match the
    reference, so `state_dict()` keys and seeded initialisation are interchangeable.

    Two users: `SimpleConv` fuses the `clip_conv` family (batch_norm, skip, GELU, GLU) into its own forward/backward;
    a stand-alone sequence (the `DeepMel` feature model) runs through `forward(x)` -> `convseq.conv_sequence`.
    Accelerated: stride 1, odd kernel <= 3, GELU / LeakyReLU / ReLU, with or without BatchNorm, skip,
    activation_on_last, GLU every `glu` layers with context <= 1, and the residual-branch options: `rewrite` (a 1x1 conv +
    LeakyReLU(leakiness) after the activation), `scale` (LayerScale) and `post_skip` (a depthwise 1x1 gain), the last two on
    layers that keep their width when `skip` is set.  Everything else raises NotImplementedError.

    Per layer k: `has_act[k]`, `has_rewrite[k]`, `has_scale[k]`, `has_post_skip[k]`, and `index[k]`, the position of each
    submodule in `sequence[k]` ('conv', 'bn', 'rewrite', 'scale', 'post_skip'; absent keys: no such module)."""

    def __init__(self, channels: tp.Sequence[int], kernel: int = 4, dilation_growth: int = 1,
                 dilation_period: tp.Optional[int] = None, stride: int = 2, dropout: float = 0.0,
                 leakiness: float = 0.0, groups: int = 1, decode: bool = False, batch_norm: bool = False,
                 dropout_input: float = 0, skip: bool = False, scale: tp.Optional[float] = None,
                 rewrite: bool = False, activation_on_last: bool = True, post_skip: bool = False, glu: int = 0,
                 glu_context: int = 0, glu_glu: bool = True, activation: tp.Any = None) -> None:
        super().__init__()
        unsupported = dict(stride=stride != 1, dropout=bool(dropout), groups=groups != 1, decode=decode,
                           dropout_input=bool(dropout_input), glu_glu=not glu_glu, kernel=kernel % 2 != 1 or kernel > 3,
                           activation=activation not in (None, nn.GELU, nn.ReLU, nn.LeakyReLU),
                           glu_context=bool(glu) and glu_context > 1)
        bad = [k for k, v in unsupported.items() if v]
        if bad:
            raise NotImplementedError(f"ConvSequence options without a CUDA implementation: {bad} (SURVEY 8(f) row 4)")
        channels = tuple(channels)
        self.skip = skip
        self.kernel = kernel
        self.glu_kernel = 1 + 2 * glu_context
        self.batch_norm = batch_norm
        # activation code / slope understood by the kernels: 0 = GELU, 1 = LeakyReLU(slope) (ReLU = slope 0)
        self.act_code = 0 if activation is nn.GELU else 1
        self.act_slope = 0.0 if activation is nn.ReLU else (0.01 if activation is nn.LeakyReLU else float(leakiness))
        make_act = (lambda: nn.LeakyReLU(leakiness)) if activation is None else activation
        # what SimpleConv's fused forward/backward covers: BatchNorm wherever there is an activation (skip, glu, the
        # activation kind and a bare last layer are free there)
        self.clip_conv_family = bool(batch_norm)
        self.sequence = nn.ModuleList()
        self.glus = nn.ModuleList()
        # the LeakyReLU after a rewrite conv is LeakyReLU(leakiness) whatever the stack's activation (common.py:124)
        self.rewrite_slope = float(leakiness)
        self.dilations: tp.List[int] = []
        self.has_act: tp.List[bool] = []
        self.has_rewrite: tp.List[bool] = []
        self.has_scale: tp.List[bool] = []
        self.has_post_skip: tp.List[bool] = []
        self.index: tp.List[tp.Dict[str, int]] = []
        dilation = 1
        for k, (chin, chout) in enumerate(zip(channels[:-1], channels[1:])):
            if dilation_period and (k % dilation_period) == 0:
                dilation = 1
            self.dilations.append(dilation)
            layers: tp.List[nn.Module] = [nn.Conv1d(chin, chout, kernel, 1, (kernel // 2) * dilation, dilation=dilation)]
            index = dict(conv=0)
            dilation *= dilation_growth
            is_last = k == len(channels) - 2
            self.has_act.append(activation_on_last or not is_last)
            if self.has_act[-1]:
                if batch_norm:
                    index["bn"] = len(layers)
                    layers.append(nn.BatchNorm1d(num_features=chout))
                layers.append(make_act())
                if rewrite:
                    index["rewrite"] = len(layers)
                    layers += [nn.Conv1d(chout, chout, 1), nn.LeakyReLU(leakiness)]
            self.has_rewrite.append(self.has_act[-1] and rewrite)
            gains = chin == chout and skip
            if gains and scale is not None:
                index["scale"] = len(layers)
                layers.append(LayerScale(chout, scale))
            if gains and post_skip:
                index["post_skip"] = len(layers)
                layers.append(nn.Conv1d(chout, chout, 1, groups=chout, bias=False))
            self.has_scale.append(gains and scale is not None)
            self.has_post_skip.append(gains and post_skip)
            self.index.append(index)
            self.sequence.append(nn.Sequential(*layers))
            if glu and (k + 1) % glu == 0:
                self.glus.append(nn.Sequential(
                    nn.Conv1d(chout, 2 * chout, self.glu_kernel, padding=glu_context), nn.GLU(dim=1)))
            else:
                self.glus.append(None)

    def glu_after(self) -> tp.List[bool]:
        return [g is not None for g in self.glus]

    def residual(self) -> tp.Optional[tp.List[tp.Tuple[bool, bool, bool]]]:
        """Per layer (rewrite, scale, post_skip) for `functional.SequencePlan.residual`; None when no layer has one."""
        flags = list(zip(self.has_rewrite, self.has_scale, self.has_post_skip))
        return flags if any(any(f) for f in flags) else None

    def scale_boost(self) -> float:
        return next((m.boost for m in self.modules() if isinstance(m, LayerScale)), 5.0)

    def residual_params(self, k: int) -> tp.List[tp.Optional[torch.Tensor]]:
        """[rewrite_w, rewrite_b, layer_scale, post_skip_w] of layer k, None where absent."""
        block, at = self.sequence[k], self.index[k]
        rw = block[at["rewrite"]] if "rewrite" in at else None
        return [None if rw is None else rw.weight, None if rw is None else rw.bias,
                block[at["scale"]].scale if "scale" in at else None,
                block[at["post_skip"]].weight if "post_skip" in at else None]

    def forward(self, x):
        from . import convseq
        return convseq.conv_sequence(self, x)


def require_library():
    """Fail loudly (no fallback) when the CUDA extension is missing."""
    _lib.load()
