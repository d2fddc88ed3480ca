"""Drop-in `SimpleConv` brain encoder (reference: bm/models/simpleconv.py:22-249).

Same constructor signature, submodule/parameter names (=> interchangeable `state_dict`), construction order
(=> identical parameters for a given `torch.manual_seed`), `forward(inputs, batch) -> [B, F, T]`, train/eval
semantics (BatchNorm running statistics, one spatial-dropout centre per training forward), and the same autograd
behaviour: gradients reach every parameter and, when it requires grad, the tensor passed as `inputs["meg"]`.
The arithmetic runs in hand-written sm_90a CUDA through the C ABI (`functional.encoder_forward`); there is no PyTorch/CPU fallback.

Accelerated configuration = the `clip_conv` family of conf/model/clip_conv.yaml (merger + initial_linear +
subject_layers + ConvSequence(batch_norm) + head), with or without `skip`, with any `glu` period, with GELU or
(Leaky)ReLU, with or without the `complex_out` head, and with merger / initial_linear / subject_layers each optional
or replaced by a subject embedding -- every row of the paper's ablation table (grids/nmi/ablation_final.py:42-52).
The un-ablated configuration takes the fused tensor-core path; a missing sensor stage switches the sensor chain to
its stage-by-stage form.  Options outside that family are accepted by the
signature but raise NotImplementedError (SURVEY.md 8(f) row 4).

Encoding models (bm/train.py:61-67) take more input streams than "meg", e.g. in_channels=dict(meg=C, features=F): the
sensor front acts on "meg" (always required), every other stream enters its own encoder as is, and the encoder outputs
are joined in sorted key order before the head -- `linear_out` (one 1x1 ConvTranspose) or `complex_out`; with
`concatenate` one encoder "concat" reads the streams joined in sorted key order (simpleconv.py:150-196, 234-243).
"""
from __future__ import annotations

import random
import typing as tp

import torch
from torch import nn

from . import functional as BF
from .common import ChannelMerger, ConvSequence, ScaledEmbedding, StaticBatch, SubjectLayers, require_library


def _require_cuda(meg: torch.Tensor) -> None:
    if not meg.is_cuda:
        raise RuntimeError("brainmagick_b200.SimpleConv runs on CUDA (sm_90a) only; there is no CPU fallback")


class SimpleConv(nn.Module):
    def __init__(self,
                 # Channels
                 in_channels: tp.Dict[str, int],
                 out_channels: int,
                 hidden: tp.Dict[str, int],
                 # Overall structure
                 depth: int = 4,
                 concatenate: bool = False,
                 linear_out: bool = False,
                 complex_out: bool = False,
                 # Conv layer
                 kernel_size: int = 5,
                 growth: float = 1.,
                 dilation_growth: int = 2,
                 dilation_period: tp.Optional[int] = None,
                 skip: bool = False,
                 post_skip: bool = False,
                 scale: tp.Optional[float] = None,
                 rewrite: bool = False,
                 groups: int = 1,
                 glu: int = 0,
                 glu_context: int = 0,
                 glu_glu: bool = True,
                 gelu: bool = False,
                 # Dual path RNN
                 dual_path: int = 0,
                 # Dropouts, BN, activations
                 conv_dropout: float = 0.0,
                 dropout_input: float = 0.0,
                 batch_norm: bool = False,
                 relu_leakiness: float = 0.0,
                 # Subject specific settings
                 n_subjects: int = 200,
                 subject_dim: int = 64,
                 subject_layers: bool = False,
                 subject_layers_dim: str = "input",
                 subject_layers_id: bool = False,
                 embedding_scale: float = 1.0,
                 # stft transform
                 n_fft: tp.Optional[int] = None,
                 fft_complex: bool = True,
                 # Attention multi-dataset support
                 merger: bool = False,
                 merger_pos_dim: int = 256,
                 merger_channels: int = 270,
                 merger_dropout: float = 0.2,
                 merger_penalty: float = 0.,
                 merger_per_subject: bool = False,
                 dropout: float = 0.,
                 dropout_rescale: bool = True,
                 initial_linear: int = 0,
                 initial_depth: int = 1,
                 initial_nonlin: bool = False,
                 subsample_meg_channels: int = 0,
                 ):
        super().__init__()
        if set(in_channels.keys()) != set(hidden.keys()):
            raise ValueError("Channels and hidden keys must match "
                             f"({set(in_channels.keys())} and {set(hidden.keys())})")
        assert kernel_size % 2 == 1, "For padding to work, this must be verified"
        if "meg" not in in_channels:
            raise NotImplementedError("SimpleConv's sensor front is built around the 'meg' stream: in_channels needs it")
        if len(in_channels) > 4:
            raise NotImplementedError("SimpleConv joins at most 4 input streams (the channel-join kernel takes 4 sources); "
                                      f"got {sorted(in_channels)}")
        self._stream_channels = {name: c for name, c in in_channels.items() if name != "meg"}
        off_path = dict(
            growth=growth != 1., dual_path=bool(dual_path), n_fft=n_fft is not None, dropout=dropout > 0.,
            initial_depth=initial_depth != 1, initial_nonlin=initial_nonlin)
        bad = [k for k, v in off_path.items() if v]
        if bad:
            raise NotImplementedError(
                f"SimpleConv options outside the accelerated clip_conv family: {bad}; see SURVEY.md 8(f) row 4")
        require_library()

        self._concatenate = concatenate
        self.out_channels = out_channels
        self.subsampled_meg_channels: tp.Optional[list] = None
        if subsample_meg_channels:               # simpleconv.py:97-102: the same draw as the reference
            indexes = list(range(in_channels["meg"]))
            random.Random(1234).shuffle(indexes)
            self.subsampled_meg_channels = indexes[:subsample_meg_channels]
        self._channel_mask: tp.Optional[torch.Tensor] = None
        self.dropout = None
        self.stft = None
        self.subject_embedding = None
        self.dual_path = None
        self.n_input_channels = in_channels["meg"]

        # construction order == the reference's (simpleconv.py:104-196), so a seeded constructor is RNG-identical.
        # merger / initial_linear / subject_layers are each optional and a subject embedding may be appended (the
        # sensor-side rows of the ablation table, grids/nmi/ablation_final.py:44,46,50,51)
        self.merger = self.initial_linear = self.subject_layers = None
        if merger:
            self.merger = ChannelMerger(merger_channels, pos_dim=merger_pos_dim, dropout=merger_dropout,
                                        usage_penalty=merger_penalty, n_subjects=n_subjects,
                                        per_subject=merger_per_subject)
            in_channels["meg"] = merger_channels
        if initial_linear:
            self.initial_linear = nn.Sequential(nn.Conv1d(in_channels["meg"], initial_linear, 1))
            in_channels["meg"] = initial_linear
        if subject_layers:
            meg_dim = in_channels["meg"]
            dim = {"hidden": hidden["meg"], "input": meg_dim}[subject_layers_dim]
            self.subject_layers = SubjectLayers(meg_dim, dim, n_subjects, subject_layers_id)
            in_channels["meg"] = dim
        if subject_dim:
            self.subject_embedding = ScaledEmbedding(n_subjects, subject_dim, embedding_scale)
            in_channels["meg"] += subject_dim

        # simpleconv.py:85-90: GELU, else LeakyReLU(relu_leakiness), else ReLU -- in the ConvSequence and in the head
        if gelu:
            activation, make_act = nn.GELU, nn.GELU
        elif relu_leakiness:
            activation, make_act = None, (lambda: nn.LeakyReLU(relu_leakiness))    # ConvSequence builds the same module
        else:
            activation, make_act = nn.ReLU, nn.ReLU
        self._streams = [name for name in in_channels if name != "meg"]      # the streams that enter their encoder as is
        if concatenate:                          # simpleconv.py:150-153: one encoder over the streams joined by sorted key
            in_channels = {"concat": sum(in_channels.values())}
            hidden = {"concat": sum(hidden.values())}
        sizes = {name: [in_channels[name]] + [int(round(hidden[name] * growth ** k)) for k in range(depth)]
                 for name in in_channels}
        final_channels = sum(s[-1] for s in sizes.values())
        seq_kw = {}
        if linear_out:                           # simpleconv.py:182-184
            assert not complex_out
            self.final = nn.ConvTranspose1d(final_channels, out_channels, 1, 1, 0)
        elif complex_out:
            self.final = nn.Sequential(
                nn.Conv1d(final_channels, 2 * final_channels, 1),
                make_act(),
                nn.ConvTranspose1d(2 * final_channels, out_channels, 1, 1, 0))
        else:
            # simpleconv.py:190-193: no head; the last convolution maps to out_channels, without BatchNorm / activation
            assert len(sizes) == 1, "if no linear_out, there must be a single branch."
            self.final = None
            seq_kw["activation_on_last"] = False
            list(sizes.values())[0][-1] = out_channels
        self.encoders = nn.ModuleDict({name: ConvSequence(
            channels, kernel=kernel_size, stride=1, leakiness=relu_leakiness, dropout=conv_dropout,
            dropout_input=dropout_input, batch_norm=batch_norm, dilation_growth=dilation_growth, groups=groups,
            dilation_period=dilation_period, skip=skip, post_skip=post_skip, scale=scale, rewrite=rewrite, glu=glu,
            glu_context=glu_context, glu_glu=glu_glu, activation=activation, **seq_kw) for name, channels in sizes.items()})
        if not all(seq.clip_conv_family for seq in self.encoders.values()):
            raise NotImplementedError("SimpleConv's fused encoder needs batch_norm=True; "
                                      "see SURVEY.md 8(f) row 4")
        self._unused_layout: tp.Dict[tuple, tuple] = {}     # merger=False: placeholder layout tables per (device, B, C)
        self.use_tensor_cores = True     # False forces the FP32-FMA kernels everywhere (debugging / A-B timing)

    # ------------------------------------------------------------------------------------------------
    def _encoder0(self) -> str:
        """The encoder that follows the sensor front: "meg", or "concat" over every stream"""
        return "concat" if self._concatenate else "meg"

    @staticmethod
    def _layer_params(seq: ConvSequence):
        out = []
        for k, block in enumerate(seq.sequence):
            conv = block[0]
            if seq.has_act[k]:
                out += [conv.weight, conv.bias, block[1].weight, block[1].bias]
            else:
                out += [conv.weight, conv.bias, None, None]          # the bare last layer of complex_out=False
            if any((seq.has_rewrite[k], seq.has_scale[k], seq.has_post_skip[k])):
                out += seq.residual_params(k)                        # rewrite_w, rewrite_b, layer_scale, post_skip_w
        for glu in seq.glus:
            if glu is not None:
                out += [glu[0].weight, glu[0].bias]
        return out

    @staticmethod
    def _bns(seq: ConvSequence) -> list:
        """layer k's BatchNorm module, None on the bare last layer"""
        return [blk[1] if seq.has_act[k] else None for k, blk in enumerate(seq.sequence)]

    def _sequence_fields(self, seq: ConvSequence) -> dict:
        """The `functional.SequencePlan` fields of one encoder"""
        residual = seq.residual()
        bns = self._bns(seq)
        return dict(
            dilations=list(seq.dilations), glu_after=seq.glu_after(), **BF.bn_plan_fields(bns, self.training),
            keep_for_backward=torch.is_grad_enabled(), use_tensor_cores=self.use_tensor_cores, skip=seq.skip,
            act_code=seq.act_code, act_slope=seq.act_slope, has_act=list(seq.has_act), batch_norm=True, residual=residual,
            rewrite_slope=seq.rewrite_slope, scale_boost=seq.scale_boost(), bn_groups=BF.bn_sync_groups(bns, residual))

    def _plan(self, meg: torch.Tensor, batch) -> BF.EncoderPlan:
        seq: ConvSequence = self.encoders[self._encoder0()]
        device = meg.device
        B, C, _ = meg.shape
        if self.merger is None:                 # no spatial attention: the layout tables are never read
            if isinstance(batch, StaticBatch):
                batch.check(meg)
            key = (device, B, C)
            if key not in self._unused_layout:  # made once: a captured step copies nothing from the host
                zeros = torch.zeros(B, dtype=torch.int32, device=device)
                self._unused_layout[key] = (torch.zeros(1, C, 2, device=device), zeros, zeros,
                                            torch.tensor([0, B], dtype=torch.int32, device=device))
            pos, rec_of_sample, rec_order, rec_off = self._unused_layout[key]
        else:
            pos, rec_of_sample, rec_order, rec_off = self.merger.batch_layout(batch, meg)
        if not isinstance(batch, StaticBatch) and not batch.subject_index.is_cuda and BF.capturing():
            raise RuntimeError("the batch's subject_index is on the host, and a CUDA graph capture cannot copy it: pass a "
                               "brainmagick_b200.StaticBatch or a batch whose subject_index is a CUDA tensor")
        fields = self._sequence_fields(seq)
        encoders = tuple((name, BF.SequencePlan(**self._sequence_fields(self.encoders[name])))
                         for name in self.encoders if name != self._encoder0())
        return BF.EncoderPlan(
            **fields, kernel_size=seq.kernel, glu_kernel=seq.glu_kernel,
            rec_positions=pos, rec_of_sample=rec_of_sample, rec_order=rec_order, rec_off=rec_off,
            subject=batch.subject_index.to(device=device, dtype=torch.int32).contiguous(),
            freq=None if self.merger is None else self.merger.frequencies(device),
            ban_centre=None if self.merger is None else self.merger.draw_ban_centre(device),
            ban_radius=0.0 if self.merger is None else float(self.merger.dropout),
            has_sub_emb=self.subject_embedding is not None, streams=tuple(self._streams), encoders=encoders,
            concatenate=self._concatenate)

    def forward(self, inputs, batch):
        """inputs: {"meg": [B, C, T], and every other stream of in_channels: [B, C_s, T]}, CUDA fp32 tensors (a stream may
        be a view, e.g. cropped in time); the sensor front (merger, initial_linear, subject layers / embedding) acts on
        "meg", which is always required.  Gradients reach every parameter and each input tensor that requires grad.
        batch: a reference-style batch (`subject_index`, `_recordings`), or a `StaticBatch` whose device buffers are used as
        they are -- what a step captured in a CUDA graph needs (DESIGN.md, "CUDA graph capture")."""
        meg = inputs["meg"]
        _require_cuda(meg)
        if meg.dtype != torch.float32:
            raise TypeError("brainmagick_b200.SimpleConv computes in fp32, like the reference")
        assert meg.shape[1] == self.n_input_channels, "number of MEG channels differs from in_channels['meg']"
        length = meg.shape[-1]
        streams = []
        for name in self._streams:
            x = inputs[name]
            _require_cuda(x)
            if x.dtype != torch.float32 or x.dim() != 3:
                raise TypeError(f"brainmagick_b200.SimpleConv: inputs[{name!r}] must be an fp32 [B, C, T] tensor")
            if x.shape[0] != meg.shape[0] or x.shape[2] != length:
                raise ValueError(f"inputs[{name!r}] has shape {tuple(x.shape)}; every stream needs meg's B and T")
            if x.shape[1] != self._stream_channels[name]:
                raise ValueError(f"inputs[{name!r}] has {x.shape[1]} channels; in_channels[{name!r}] is "
                                 f"{self._stream_channels[name]}")
            streams.append(x)
        plan = self._plan(meg, batch)
        for seq in self.encoders.values():      # nn.BatchNorm1d bookkeeping, ahead of the finalize kernels that read it
            BF.bn_count_batches(self._bns(seq))
        if self.subsampled_meg_channels is not None:         # simpleconv.py:200-203, applied inside the encoder node
            if self._channel_mask is None or self._channel_mask.device != meg.device:
                mask = torch.zeros(self.n_input_channels)
                mask[self.subsampled_meg_channels] = 1.
                self._channel_mask = mask.to(meg.device)
            plan.channel_mask = self._channel_mask
            plan.masked_meg = inputs["meg"] = torch.empty(meg.shape, device=meg.device)
        heads = None if self.merger is None else self.merger.heads
        il_w, il_b = (None, None) if self.initial_linear is None else \
            (self.initial_linear[0].weight, self.initial_linear[0].bias)
        subj_w = None if self.subject_layers is None else self.subject_layers.weights
        sub_emb = None
        if self.subject_embedding is not None:           # [B, E]; its gradient returns through torch's embedding backward
            sub_emb = self.subject_embedding(batch.subject_index.to(meg.device).long())
        if self.final is None:
            head = [None] * 4
        elif isinstance(self.final, nn.ConvTranspose1d):    # linear_out
            head = [None, None, self.final.weight, self.final.bias]
        else:
            head = [self.final[0].weight, self.final[0].bias, self.final[2].weight, self.final[2].bias]
        est = BF.encoder_forward(plan, meg, heads, il_w, il_b, subj_w, *head,
                                 self._layer_params(self.encoders[self._encoder0()]), sub_emb=sub_emb, streams=streams,
                                 encoder_params=[self._layer_params(self.encoders[name]) for name, _ in plan.encoders])
        return est[:, :, :length]
