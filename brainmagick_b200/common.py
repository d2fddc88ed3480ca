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
        table, rows, order, off = self.batch_layout_host(batch, n_channels)
        to = dict(device=device, non_blocking=True)
        return (table.to(**to), torch.from_numpy(rows).to(**to), torch.from_numpy(order).to(**to),
                torch.from_numpy(off).to(**to))

    def batch_layout_host(self, batch, n_channels: int):
        """`batch_layout` on the host: (rec_positions [R,C,2] fp32 tensor, rec_of_sample [B], rec_order [B] and
        rec_off [R+1] int32 numpy arrays); rows are the recordings in ascending recording_index."""
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
        return table, rows, order, off


class StaticBatch:
    """A batch of fixed shape whose sensor layout lives in device buffers, for training / evaluation steps captured in a CUDA
    graph (torch.cuda.graph): the graph reads these buffers, and the caller refills them with `fill_` before each replay.
    `SimpleConv.forward` and `ChannelMerger.forward` take it in place of a reference batch, in eager mode too.

    Buffers (on `device`, fixed addresses): subject_index [B] int32, rec_positions [R_max, C, 2] fp32 (one row per recording
    slot), rec_of_sample [B] and rec_order [B] int32, rec_off [R_max + 1] int32 (CSR offsets of the samples of each slot).
    A batch with R < R_max recordings fills slots 0..R-1 exactly as `PositionGetter.batch_layout` lays out a reference batch;
    slots R..R_max-1 repeat slot 0's positions and own empty segments (rec_off[r] = B).  Their attention weights are
    therefore finite (an all-INVALID row would be a softmax over -inf only: NaN, and NaN * 0 poisons the heads' gradient)
    and their weight gradients are exact zeros."""

    def __init__(self, batch_size: int, n_channels: int, max_recordings: int, device):
        if min(batch_size, n_channels, max_recordings) < 1:
            raise ValueError(f"StaticBatch needs batch_size, n_channels and max_recordings >= 1, got "
                             f"{batch_size}, {n_channels}, {max_recordings}")
        self.batch_size, self.n_channels, self.max_recordings = int(batch_size), int(n_channels), int(max_recordings)
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        B, C, R = self.batch_size, self.n_channels, self.max_recordings
        sizes = dict(rec_positions=R * C * 2, subject_index=B, rec_of_sample=B, rec_order=B, rec_off=R + 1)
        cuda = self.device.type == "cuda"
        # every field is 4 bytes wide: one int32 staging buffer (pinned) and one device buffer, sent with one copy
        total = sum(sizes.values())
        self._stage = torch.zeros(total, dtype=torch.int32, pin_memory=cuda)
        self._buffer = torch.zeros(total, dtype=torch.int32, device=self.device)
        self._staged, at = {}, 0
        for name, n in sizes.items():
            host, dev = self._stage[at:at + n], self._buffer[at:at + n]
            if name == "rec_positions":
                host, dev = host.view(torch.float32).view(R, C, 2), dev.view(torch.float32).view(R, C, 2)
            self._staged[name] = host
            setattr(self, name, dev)
            at += n
        self._copied = torch.cuda.Event() if cuda else None   # recorded after the last copy out of the staging buffer
        self._copy_pending = False
        self._position_getter = PositionGetter()

    def layout(self):
        """(rec_positions, rec_of_sample, rec_order, rec_off): the device buffers, as `PositionGetter.batch_layout` returns."""
        return self.rec_positions, self.rec_of_sample, self.rec_order, self.rec_off

    def check(self, meg: torch.Tensor) -> None:
        """Raises ValueError unless meg [B, C, T] has this batch's B and C and lives on its device."""
        if meg.shape[0] != self.batch_size or meg.shape[1] != self.n_channels or meg.device != self.device:
            raise ValueError(f"input of shape {tuple(meg.shape)} on {meg.device} for a StaticBatch of batch_size "
                             f"{self.batch_size}, n_channels {self.n_channels} on {self.device}")

    def fill_(self, batch) -> "StaticBatch":
        """Refill the buffers from a reference-style batch (`subject_index`, `_recordings`, `meg`): the layout is computed on
        the host by `PositionGetter.batch_layout_host`, then everything goes to the device in one non-blocking copy from the
        pinned staging buffer, on the current stream (a CUDA subject_index is copied device to device on the same stream).
        Waits first for the previous copy out of the staging buffer.  Not allowed while a CUDA graph is being captured.

        In eager use the autograd graph of a step keeps references to these buffers until its backward has run: call
        `fill_` for the next batch only after the backward of the step that read the previous contents (not ahead of it
        to prefetch, nor between the forwards of accumulated steps), or that backward reads the new layout."""
        from . import functional as BF
        if BF.capturing():
            raise RuntimeError("StaticBatch.fill_ copies from host memory: call it before a replay, not inside the capture")
        B, C, R_max = self.batch_size, self.n_channels, self.max_recordings
        subject = batch.subject_index.reshape(-1)
        meg = getattr(batch, "meg", None)
        if len(batch._recordings) != B or subject.numel() != B or (meg is not None and meg.shape[0] != B):
            raise ValueError(f"a batch of {len(batch._recordings)} samples for a StaticBatch of batch_size {B}")
        if meg is not None and meg.shape[1] != C:
            raise ValueError(f"a batch of {meg.shape[1]} channels for a StaticBatch of n_channels {C}")
        table, rows, order, off = self._position_getter.batch_layout_host(batch, C)
        R = table.shape[0]
        if R > R_max:
            raise ValueError(f"a batch of {R} distinct recordings for a StaticBatch of max_recordings {R_max}")
        if self._copy_pending:
            self._copied.synchronize()          # the previous copy may still be reading the staging buffer
        st = self._staged
        st["rec_positions"][:R] = table
        st["rec_positions"][R:] = table[0]
        st["rec_of_sample"].numpy()[:] = rows
        st["rec_order"].numpy()[:] = order
        st["rec_off"].numpy()[:R + 1] = off
        st["rec_off"][R + 1:] = B
        if not subject.is_cuda:
            st["subject_index"].copy_(subject)
        self._buffer.copy_(self._stage, non_blocking=True)
        if subject.is_cuda:
            self.subject_index.copy_(subject)
        if self._copied is not None:
            self._copied.record(torch.cuda.current_stream(self.device))    # the stream the copies above ran on
            self._copy_pending = True
        return self


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
        self._freq: tp.Optional[torch.Tensor] = None                 # `frequencies(device)`'s copy

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

    def frequencies(self, device) -> torch.Tensor:
        """The embedding's frequency table (`FourierEmb.frequencies`) on `device`, copied there once: a step captured in a
        CUDA graph copies nothing from the host."""
        if self._freq is None or self._freq.device != torch.device(device):
            self._freq = self.embedding.frequencies().to(device)
        return self._freq

    def batch_layout(self, batch, meg: torch.Tensor):
        """(rec_positions, rec_of_sample, rec_order, rec_off) of `batch` for the input meg [B, C, T]: a StaticBatch's device
        buffers as they are, else the reference batch's layout built on the host and copied to meg's device."""
        from . import functional as BF
        if isinstance(batch, StaticBatch):
            batch.check(meg)
            return batch.layout()
        if BF.capturing():
            raise RuntimeError("a reference batch's sensor layout is built on the host and copied to the device on every "
                               "forward, which a CUDA graph capture cannot hold: pass a brainmagick_b200.StaticBatch")
        return self.position_getter.batch_layout(batch, meg.shape[1], meg.device)

    def forward(self, meg, batch):
        """Stand-alone call (bm/models/common.py:334-362): [B, C, T] -> [B, chout, T].  Inside SimpleConv the merger is
        fused into the encoder; this runs the same stage kernels for callers that use the module on its own."""
        from . import functional as BF
        _require_cuda_fp32(meg, "ChannelMerger")
        pos, rec_of_sample, rec_order, rec_off = self.batch_layout(batch, meg)
        return BF.channel_merger_forward(meg, self.heads, pos, rec_of_sample, rec_order, rec_off, self.frequencies(meg.device),
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
