"""autograd.Functions that run the hot path through the C ABI (libbm_b200.so).

`encoder_forward` is SimpleConv.forward at the clip_conv configuration (bm/models/simpleconv.py:198-249) as ONE
autograd node: its backward launches the hand-written gradient kernels in reverse order, so `loss.backward()`
leaves ordinary dense `.grad` tensors on every parameter (what bm/solver.py:384-387 and
flashy.distrib.sync_model expect), and on `meg` when it requires grad (gradient-based attribution).  `clip_loss` /
`clip_scores` / `clip_scores_grad` are ClipLoss (bm/losses.py:77-114).

Kernel selection is by shape only: contractions whose channel counts fit the tensor-core tiling (K % 32 == 0 and an
N tile of 64..160 dividing N -- every layer of the real clip_conv model) run on the tensor-core kernels
(3xTF32, `bm_tc_*`; single-pass TF32 when PyTorch's float32 matmul precision allows TF32, bf16 operands under bf16
autocast, see `_tc_call`); other shapes
(the tiny unit-test models) run on the FP32-FMA kernels of the same library.
"""
from __future__ import annotations

import dataclasses
import functools
import typing as tp
import weakref

import torch
import torch.distributed as dist

from . import _lib
from ._lib import call, ptr, stream


ACT_GELU, ACT_LRELU, ACT_NONE = 0, 1, 2      # activation codes of the epilogue kernels


@dataclasses.dataclass
class SequencePlan:
    """The layers of a ConvSequence (bm/models/common.py:79-151) as `conv_stack_forward` / `conv_stack_backward` run them:
    layer k is conv (+ BatchNorm if `batch_norm` and has_act[k]) (+ activation if has_act[k]) (+ the layer input if `skip`
    and the conv keeps the width), then a GLU block if glu_after[k].

    `residual[k]` = (rewrite, scale, post_skip) of layer k (None: no layer has one): a 1x1 conv + LeakyReLU(rewrite_slope)
    after the activation, then the LayerScale gain (its factor `scale_boost`) and the depthwise post_skip gain, in front of
    the residual add (common.py:123-130).  A layer with any of them takes `layer_width(plan, k)` = 8 parameters.

    `bn_groups[k]`: the process group layer k's BatchNorm takes its statistics over (an nn.SyncBatchNorm, see
    `bn_sync_groups`), None where the layer uses its own rows (None: no layer syncs).

    `training`, `bn_eps`, `bn_momentum` hold for every BatchNorm layer unless `bn_layers` is set: then `bn_layers[k]` is
    layer k's own mode and settings (None where the layer has no BatchNorm); see `bn_plan_fields` and `bn_layer`."""
    dilations: tp.List[int]
    glu_after: tp.List[bool]
    has_act: tp.List[bool]            # layer k ends with (BatchNorm +) activation (activation_on_last, common.py:112)
    batch_norm: bool
    act_code: int                     # ACT_GELU, or ACT_LRELU with slope act_slope (ReLU: slope 0)
    act_slope: float
    skip: bool
    training: bool
    bn_eps: float
    bn_momentum: float
    bn_buffers: tp.List[tp.Optional[tp.Tuple[torch.Tensor, torch.Tensor]]]   # (running_mean, running_var) per layer
    use_tensor_cores: bool
    keep_for_backward: bool
    residual: tp.Optional[tp.List[tp.Tuple[bool, bool, bool]]] = dataclasses.field(default=None, kw_only=True)
    rewrite_slope: float = dataclasses.field(default=0.0, kw_only=True)
    scale_boost: float = dataclasses.field(default=5.0, kw_only=True)
    bn_groups: tp.Optional[tp.List[tp.Any]] = dataclasses.field(default=None, kw_only=True)
    bn_layers: tp.Optional[tp.List[tp.Optional["BnLayer"]]] = dataclasses.field(default=None, kw_only=True)


class BnLayer(tp.NamedTuple):
    """One BatchNorm layer's mode and settings, as torch.nn.BatchNorm1d reads them from its own module."""
    training: bool                    # batch statistics; running buffers and num_batches_tracked updated
    eps: float
    momentum: tp.Optional[float]      # None: cumulative average, factor 1 / num_batches_tracked computed on the device
    num_batches_tracked: tp.Optional[torch.Tensor]   # the counter a cumulative-average layer's finalize reads


def bn_plan_fields(bns, training: bool) -> dict:
    """The SequencePlan fields `training`, `bn_eps`, `bn_momentum`, `bn_buffers` and `bn_layers` from layer k's BatchNorm
    module bns[k] (None: the layer has none) in a module whose own mode is `training`.  Each layer follows its own module,
    as torch does: batch statistics exactly when bn.training, and its own eps and momentum.  `bn_layers` stays None when
    every layer has the module's mode and the first layer's eps and a numeric momentum: such a plan is the uniform one."""
    present = [bn for bn in bns if bn is not None]
    for bn in present:
        if not bn.track_running_stats or bn.running_mean is None or bn.running_var is None:
            raise NotImplementedError("BatchNorm without running statistics (track_running_stats=False)")
    eps, momentum = (present[0].eps, present[0].momentum) if present else (0.0, 0.0)
    layers = [None if bn is None else
              BnLayer(bool(bn.training), float(bn.eps), None if bn.momentum is None else float(bn.momentum),
                      bn.num_batches_tracked if bn.momentum is None and bn.training else None) for bn in bns]
    uniform = momentum is not None and all(
        layer is None or (layer.training == training and layer.eps == eps and layer.momentum == momentum)
        for layer in layers)
    return dict(training=training, bn_eps=eps, bn_momentum=0.0 if momentum is None else momentum,
                bn_buffers=[None if bn is None else (bn.running_mean, bn.running_var) for bn in bns],
                bn_layers=None if uniform else layers)


def bn_layer(plan: SequencePlan, k: int) -> BnLayer:
    """Layer k's BatchNorm mode and settings (the layer has a BatchNorm)."""
    if plan.bn_layers is not None:
        return plan.bn_layers[k]
    return BnLayer(plan.training, plan.bn_eps, plan.bn_momentum, None)


def bn_count_batches(bns) -> None:
    """nn.BatchNorm1d's bookkeeping on the device: num_batches_tracked += 1 on every layer in training mode.  Called before
    the layers run, as torch does, so that a cumulative-average finalize reads the incremented count on the same stream."""
    for bn in bns:
        if bn is not None and bn.training:
            bn.num_batches_tracked.add_(1)


def bn_sync_groups(bns, residual=None):
    """The plan's `bn_groups` from layer k's BatchNorm module bns[k] (None: the layer has none): torch's SyncBatchNorm rule
    (`need_sync` in torch/nn/modules/batchnorm.py) -- an nn.SyncBatchNorm in training mode, torch.distributed initialised
    and more than one rank in its process_group (None: WORLD) takes the group's statistics; every other layer its own.
    -> the per-layer groups, or None when no layer syncs.  `residual`: the plan's residual-branch flags; a syncing layer
    with a LayerScale or post_skip gain raises (its BatchNorm backward runs inside bm_bn_act_gain_skip_bwd)."""
    if not (dist.is_available() and dist.is_initialized()):
        return None
    groups = []
    for k, bn in enumerate(bns):
        group = None
        if isinstance(bn, torch.nn.SyncBatchNorm) and bn.training:
            pg = bn.process_group if bn.process_group else dist.group.WORLD
            if dist.get_world_size(pg) > 1:
                group = pg
        if group is not None and residual is not None and (residual[k][1] or residual[k][2]):
            raise NotImplementedError("SyncBatchNorm on a ConvSequence layer with a LayerScale (scale) or post_skip gain")
        groups.append(group)
    if any(g is not None for g in groups) and capturing():
        raise RuntimeError("a SyncBatchNorm layer with more than one rank all-reduces its statistics, which a CUDA graph "
                           "capture of the step cannot hold; capture on one rank or use nn.BatchNorm1d")
    return groups if any(g is not None for g in groups) else None


def _bn_finalize(stats, rows, group, layer: BnLayer, rm, rv, mean, invstd, C, st):
    """Batch statistics -> mean, invstd and the running-buffer update of one training-mode BatchNorm layer: the `_counted`
    forms for a syncing layer (its row count is in stats[2C]), the `_cumulative` forms for momentum=None."""
    if group is not None and layer.momentum is None:
        call("bm_bn_stats_finalize_counted_cumulative", ptr(stats), float(layer.eps), ptr(layer.num_batches_tracked),
             ptr(rm), ptr(rv), ptr(mean), ptr(invstd), C, st)
    elif group is not None:
        call("bm_bn_stats_finalize_counted", ptr(stats), float(layer.eps), float(layer.momentum), ptr(rm), ptr(rv),
             ptr(mean), ptr(invstd), C, st)
    elif layer.momentum is None:
        call("bm_bn_stats_finalize_cumulative", ptr(stats), rows, float(layer.eps), ptr(layer.num_batches_tracked),
             ptr(rm), ptr(rv), ptr(mean), ptr(invstd), C, st)
    else:
        call("bm_bn_stats_finalize", ptr(stats), rows, float(layer.eps), float(layer.momentum), ptr(rm), ptr(rv),
             ptr(mean), ptr(invstd), C, st)


def _sync_bn_sums(buf, C, rows, group):
    """All-reduce (sum) over `group` of a SyncBatchNorm layer's fp64 column sums buf[:2C], with this rank's row count in
    buf[2C]: the group's count (per-rank batches may be ragged) travels in the same collective, and the `_counted` /
    `_apply` kernels read it on the device, so the host never waits for it."""
    head = buf[:2 * C + 1]
    head[2 * C].fill_(float(rows))
    dist.all_reduce(head, group=group)


def layer_width(plan: SequencePlan, k: int) -> int:
    """Entries of layer k's parameter tuple: (conv_w, conv_b, gamma, beta), then on a layer with a residual-branch option
    (rewrite_w, rewrite_b, layer_scale, post_skip_w); None where a parameter is absent."""
    return 8 if plan.residual is not None and any(plan.residual[k]) else 4


@dataclasses.dataclass
class EncoderPlan(SequencePlan):
    """Everything `encoder_forward` needs that is not a differentiable tensor.  SimpleConv's ConvSequence has BatchNorm and
    an activation on every layer, except a bare last layer when complex_out=False (simpleconv.py:190-193)."""
    kernel_size: int
    glu_kernel: int
    rec_positions: torch.Tensor            # [R,C,2] fp32, rows = recordings present in the batch
    rec_of_sample: torch.Tensor            # [B] int32 -> row of rec_positions
    rec_order: torch.Tensor                # [B] int32 samples sorted by recording
    rec_off: torch.Tensor                  # [R+1] int32 CSR offsets
    subject: torch.Tensor                  # [B] int32
    freq: torch.Tensor                     # [sqrt(P/2)] fp32 Fourier frequencies
    ban_centre: tp.Optional[torch.Tensor]  # [2] fp32 or None
    ban_radius: float
    has_sub_emb: bool = False              # the last tensor argument is the [B, E] subject-embedding rows
    channel_mask: tp.Optional[torch.Tensor] = None   # [C] subsample_meg_channels mask (simpleconv.py:200-203), or None
    masked_meg: tp.Optional[torch.Tensor] = None     # [B,C,T] buffer that receives meg * channel_mask
    # several input streams (simpleconv.py:150-196, 234-243).  This plan's own layers are encoder 0: "meg", or "concat"
    # over every stream; `encoders` are the others, each with its own layer plan
    streams: tp.Tuple[str, ...] = ()                 # the input streams other than "meg", in argument order
    encoders: tp.Tuple[tp.Tuple[str, SequencePlan], ...] = ()
    concatenate: bool = False


def _empty(shape, like, dtype=torch.float32):
    return torch.empty(shape, device=like.device, dtype=dtype)


_status: tp.Dict[torch.device, torch.Tensor] = {}


def tc_status_tensor(device) -> torch.Tensor:
    """Device int32 word the tensor-core kernels set if their bounded pipeline waits ever time out."""
    device = torch.device(device)
    if device not in _status:
        _status[device] = torch.zeros(1, dtype=torch.int32, device=device)
    return _status[device]


MASK_NOT_ALL_TRUE = 903   # status code of bm_check_all_true: a ClipLoss mask with a False entry (900-902: the kernels' own)
# status codes of bm_decoding_loss_fwd (FeatureDecodingLoss): no mask entry set, a class target >= K, a bad negative target
DECODING_NO_MASK, DECODING_TARGET_TOO_LARGE, DECODING_TARGET_NEGATIVE = 904, 905, 906


def check_tc_status(device=None) -> None:
    """Synchronising check (tests, bench, end of epoch): raises if a kernel reported a bad subject index, a ClipLoss mask that
    is not all true or a FeatureDecodingLoss data error (both checked on the device in a captured step), or a tensor-core
    pipeline timeout."""
    for dev, t in _status.items():
        if device is None or torch.device(device) == dev:
            code = int(t.item())
            if code == 900:
                t.zero_()
                raise IndexError(f"a subject / recording index is outside the weight sets of the per-sample 1x1 layer on {dev} "
                                 "(bm/models/common.py:57 raises there too)")
            if code == MASK_NOT_ALL_TRUE:
                t.zero_()
                raise AssertionError(f"mask is not supported for now (a ClipLoss mask with a False entry on {dev})")
            if code in (DECODING_NO_MASK, DECODING_TARGET_TOO_LARGE, DECODING_TARGET_NEGATIVE):
                t.zero_()
                raise _decoding_error(code, f"on {dev}")
            if code != 0:
                raise _lib.BmB200Error(f"a tensor-core kernel reported a pipeline timeout (barrier code {code}) on {dev}")


def capturing() -> bool:
    """True while the current CUDA stream is being captured into a CUDA graph (torch.cuda.graph): then no step may read
    device memory on the host, copy from host memory or run a collective.  The one place the host code asks."""
    return torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing()


def check_all_true(mask: torch.Tensor, code: int = MASK_NOT_ALL_TRUE) -> None:
    """Enqueue `assert mask.all()` on the device (bm_check_all_true): a False entry sets the status word to `code`, which
    the next check_tc_status() raises."""
    m = mask.detach()
    if m.dtype not in (torch.bool, torch.uint8):
        m = m != 0
    m = m.contiguous()
    call("bm_check_all_true", ptr(m), m.numel(), int(code), ptr(tc_status_tensor(m.device)), stream())


OVERLAP_WGRAD = True   # weight-gradient kernels on a side stream, concurrent with the data-gradient kernels of the layer


_side_streams: tp.Dict[torch.device, torch.cuda.Stream] = {}


def _side_stream(device) -> torch.cuda.Stream:
    device = torch.device(device)
    if device not in _side_streams:
        _side_streams[device] = torch.cuda.Stream(device=device)
    return _side_streams[device]


def _on_side(side, keep_alive, fn, *operands):
    """fn() on the weight-gradient stream `side`, after everything queued so far on the current (main) stream; side None:
    inline.  The operands the side kernels read go to `keep_alive`, which the caller keeps until the main stream has waited
    on `side` (no record_stream on them: with the host running steps ahead it would block the allocator from reusing ~3 GB
    of blocks and force cudaMallocs in the timed loop); fn's output tensors are recorded on the main stream."""
    if side is None:
        return fn()
    main = torch.cuda.current_stream()
    side.wait_stream(main)
    with torch.cuda.stream(side):
        out = fn()
    keep_alive.append(operands)
    for o in out if isinstance(out, tuple) else (out,):
        if o is not None:
            o.record_stream(main)
    return out


def _round_up(n, m):
    return (n + m - 1) // m * m


# ---- deterministic forms ------------------------------------------------------------------------------------------
# Under torch.use_deterministic_algorithms(True) (`_lib.deterministic()`) every entry point whose default form finishes a
# floating-point reduction with atomics is replaced by its `_det` form (include/bm_b200.h), which reduces in a fixed order
# through a workspace allocated here.  With the flag off the call stream is exactly the default one.
def _det_workspace(name, like, *dims) -> torch.Tensor:
    n = int(getattr(_lib.load(), name + "_workspace")(*dims))
    return torch.empty((max(n, 2),), device=like.device, dtype=torch.float32)


def _reducing_call(name, like, ws_dims, *args, reduces=True):
    """call(name, *args) -- or, under the determinism flag, `name`_det with the workspace of `name`_det_workspace(*ws_dims)
    inserted before the stream argument (ws_dims None: a _det form without workspace, same arguments).  `reduces=False`:
    the NULL gradient pointers of this call leave nothing to reduce, so the _det form gets no workspace (NULL, 0)."""
    if not _lib.deterministic():
        return call(name, *args)
    if ws_dims is not None and not reduces:
        return call(name + "_det", *args[:-1], None, 0, args[-1])
    if ws_dims is None:
        return call(name + "_det", *args)
    ws = _det_workspace(name + "_det", like, *ws_dims)
    return call(name + "_det", *args[:-1], ptr(ws), ws.numel(), args[-1])


# ---- TF32 and bf16 forms ---------------------------------------------------------------------------------------------
# Under TF32 matmul precision (`_lib.tf32()`: torch.set_float32_matmul_precision("high"), matmul.allow_tf32 = True, ...) every
# tensor-core contraction takes its single-pass `_tf32` form (include/bm_b200.h), with the same arguments.  Under
# torch.autocast("cuda", dtype=torch.bfloat16) (`_lib.bf16()`, recorded by each autograd node's forward for its backward)
# it takes its `_bf16` form instead, whatever the TF32 flag says.  The FP32-FMA kernels stay exact (TF32 and bf16 are
# permitted, not required) and the fp16-piece entry points keep their one form.
# tensor-core entry points with a `_det` form of the same arguments
_DET_SAME_ARGS = ("bm_clip_scores", "bm_clip_loss_fwd", "bm_clip_loss_fwd_pooled")


def replays_bf16(backward):
    """An autograd node's backward, run with the bf16 mode its forward recorded in `ctx.bf16` (`_lib.recorded_bf16`)."""
    @functools.wraps(backward)
    def run(ctx, *grads):
        with _lib.recorded_bf16(ctx.bf16):
            return backward(ctx, *grads)
    return run


def _tc_call(name, *args):
    """call(name[_det][_bf16 | _tf32], *args) for a tensor-core entry point: its `_det` form under the determinism flag where
    it has one, then the `_bf16` form under bf16 autocast, else the `_tf32` form under TF32 matmul precision."""
    if name in _DET_SAME_ARGS and _lib.deterministic():
        name += "_det"
    if _lib.bf16():
        name += "_bf16"
    elif _lib.tf32():
        name += "_tf32"
    return call(name, *args)


def col_sum(x, rows, C, out, st):
    """out[c] = sum_r x[r, c] (bm_col_sum, or bm_col_sum_det under the determinism flag)."""
    if _lib.deterministic():
        ws = _det_workspace("bm_col_sum_det", x, rows, C)
        call("bm_col_sum_det", ptr(x), rows, C, ptr(ws), ws.numel(), ptr(out), st)
    else:
        call("bm_col_sum", ptr(x), rows, C, ptr(out), st)


def col_stats(y, rows, C, stats, st):
    """BatchNorm batch statistics of channels-last y (bm_col_stats, or bm_col_stats_det under the determinism flag)."""
    if _lib.deterministic():
        ws = _det_workspace("bm_col_stats_det", y, rows, C)
        call("bm_col_stats_det", ptr(y), rows, C, ptr(ws), ws.numel(), ptr(stats), st)
    else:
        call("bm_col_stats", ptr(y), rows, C, ptr(stats), st)


def tc_wgrad(dy, x, B, T, M, N, Ntrue, kw, dilation, status, dbias=None):
    """dw[m][n][tap] = sum_{b,t} dy[b,t,m] x[b,t+(tap-kw//2)*dilation,n] on the tensor cores -> [M, Ntrue, kw];
    `dbias` [M] (optional) receives sum_{b,t} dy[b,t,m]."""
    lib = _lib.load()
    dw = _empty((M, Ntrue, kw), dy)
    rows = kw * N                                       # output rows of bm_tc_wgrad_conv's GEMM, tiled in blocks of 256
    pair_ok = bool(lib.bm_tc_wgrad_conv_supported(T, M, N, kw)) and \
        rows / (-(-rows // 256) * 256) >= 0.9            # else the single-CTA kernel wastes less on padding rows
    if pair_ok:
        ws = _empty((int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, kw)),), dy)
        _tc_call("bm_tc_wgrad_conv", ptr(dy), ptr(x), B, T, M, N, Ntrue, kw, dilation, ptr(ws), ptr(dw), ptr(status),
                 stream())
        if dbias is not None:
            col_sum(dy, B * T, M, dbias, stream())
        return dw
    ws = _empty((int(lib.bm_tc_wgrad_workspace(B, M, N, kw)),), dy)
    det = _lib.deterministic()                # the kernel's own bias reduction is atomic: a fixed-order column sum instead
    _tc_call("bm_tc_wgrad", ptr(dy), ptr(x), B, T, M, N, Ntrue, kw, dilation, ptr(ws), ptr(dw), None if det else ptr(dbias),
             ptr(status), stream())
    if det and dbias is not None:
        col_sum(dy, B * T, M, dbias, stream())
    return dw


def group_layout(index: torch.Tensor, n_groups: int):
    """CSR grouping of the samples by `index` (values 0..n_groups-1): (order [B] int32, offsets [n_groups+1] int32), computed
    on the device WITHOUT a device->host synchronisation -- torch.bincount sizes its output from the data and stalls the host
    until everything queued before it has run (8.6 ms of a 17.6 ms step, measured with profiles/host_profile.py)."""
    order = torch.argsort(index, stable=True).to(torch.int32)
    groups = torch.arange(n_groups, device=index.device, dtype=index.dtype)
    counts = (index.reshape(-1, 1) == groups.reshape(1, -1)).sum(0)
    off = torch.zeros(n_groups + 1, dtype=torch.int32, device=index.device)
    off[1:] = torch.cumsum(counts, 0).to(torch.int32)
    return order, off


class _Conv:
    """One conv layer's prepared operands + the kernel choice (tensor-core or FP32-FMA)."""

    def __init__(self, w: torch.Tensor, T: int, glu: bool, allow_tc: bool, pad_cin_to: int = 0, want_bwd=True):
        self.cout, self.cin_true, self.kw = w.shape
        self.glu = glu
        w = w.contiguous()
        if pad_cin_to and pad_cin_to != self.cin_true:
            wp = torch.zeros(self.cout, pad_cin_to, self.kw, device=w.device, dtype=w.dtype)
            wp[:, :self.cin_true] = w
            w = wp
        self.cin = w.shape[1]
        st = stream()
        lib = _lib.load()
        g = 1 if glu else 0
        # raw-weight entry point (bm_tc_conv1d_persistent) where its shape gate fits, else the pre-split one
        # (bm_tc_conv1d), else FP32 FMA
        self.fwd_pp = allow_tc and bool(lib.bm_tc_conv1d_persistent_supported(T, self.cin, self.cout, self.kw, g))
        self.bwd_pp = allow_tc and bool(lib.bm_tc_conv1d_persistent_supported(T, self.cout, self.cin, self.kw, 0))
        fwd_tc = self.fwd_pp or (allow_tc and bool(lib.bm_tc_conv_supported(T, self.cin, self.cout, self.kw, g)))
        bwd_tc = self.bwd_pp or (allow_tc and bool(lib.bm_tc_conv_supported(T, self.cout, self.cin, self.kw, 0)))
        self.fwd_tc, self.bwd_tc = fwd_tc, bwd_tc
        self.wgrad_tc = allow_tc and bool(lib.bm_tc_wgrad_supported(self.cout, self.cin))
        self.f_hi = self.f_lo = self.g_hi = self.g_lo = self.wf = self.wb = None
        need_f = fwd_tc                                            # fp32 K-major operands for the tensor-core kernels
        need_g = bwd_tc and want_bwd
        if need_f or need_g:
            # RAW fp32 for the persistent kernel (it derives the tf32 lo part itself), a pre-split tf32 hi/lo pair for the
            # single-CTA kernel
            if need_f:
                self.f_hi = _empty((self.kw, self.cout, self.cin), w)
                self.f_lo = None if self.fwd_pp else _empty((self.kw, self.cout, self.cin), w)
            if need_g:
                self.g_hi = _empty((self.kw, self.cin, self.cout), w)
                self.g_lo = None if self.bwd_pp else _empty((self.kw, self.cin, self.cout), w)
            call("bm_tc_weight_split", ptr(w), self.cout, self.cin, self.kw, ptr(self.f_hi), ptr(self.f_lo),
                 ptr(self.g_hi), ptr(self.g_lo), st)
        if (not fwd_tc) or (want_bwd and not bwd_tc):
            self.wf = _empty((self.kw, self.cin, self.cout), w) if not fwd_tc else None
            self.wb = _empty((self.kw, self.cout, self.cin), w) if (want_bwd and not bwd_tc) else None
            call("bm_conv_weight_prep", ptr(w), self.cout, self.cin, self.kw, ptr(self.wf), ptr(self.wb), st)

    def run_tc(self, fwd: bool, x, bias, addend, B, T, dilation, glu, act, tmajor, y, aux, glu_out, stats, status):
        """One tensor-core conv launch: forward taps (fwd) or the data gradient; `addend` must be None or `y` itself
        (in-place accumulation) on the persistent kernel."""
        st = stream()
        if fwd:
            pp, hi, lo, cin, ntot, sign = self.fwd_pp, self.f_hi, self.f_lo, self.cin, self.cout, 1
        else:
            pp, hi, lo, cin, ntot, sign = self.bwd_pp, self.g_hi, self.g_lo, self.cout, self.cin, -1
        if pp:
            assert addend is None or addend.data_ptr() == y.data_ptr(), "the persistent kernel accumulates in place only"
            _tc_call("bm_tc_conv1d_persistent", ptr(x), ptr(hi), ptr(bias), 0 if addend is None else 1, B, T, cin, ntot,
                     self.kw, dilation, sign, glu, act, tmajor, ptr(y), ptr(aux), ptr(glu_out), ptr(stats), ptr(status), st)
        else:
            assert stats is None
            _tc_call("bm_tc_conv1d", ptr(x), ptr(hi), ptr(lo), ptr(bias), ptr(addend), B, T, cin, ntot, self.kw, dilation,
                     sign, glu, act, tmajor, ptr(y), ptr(aux), ptr(glu_out), None, ptr(status), st)

    # y = conv(x) (+bias); optionally BatchNorm statistics into `stats`
    def forward(self, x, bias, B, T, dilation, y, stats, status):
        st = stream()
        if self.fwd_tc:
            fused = stats is not None and self.fwd_pp          # BatchNorm statistics out of the conv epilogue
            if self.cout > 320 or _lib.deterministic():
                fused = False                                   # the kernel keeps the statistics of ONE N tile in smem, and
                                                                # commits them with atomics
            self.run_tc(True, x, bias, None, B, T, dilation, 0, 0, 0, y, None, None, stats if fused else None, status)
            if stats is not None and not fused:
                col_stats(y, B * T, self.cout, stats, st)
        elif stats is not None and _lib.deterministic():
            call("bm_conv1d_fwd", ptr(x), ptr(self.wf), ptr(bias), B, T, self.cin, self.cout, self.kw, dilation,
                 ptr(y), None, st)
            col_stats(y, B * T, self.cout, stats, st)
        else:
            call("bm_conv1d_fwd", ptr(x), ptr(self.wf), ptr(bias), B, T, self.cin, self.cout, self.kw, dilation,
                 ptr(y), ptr(stats), st)

    def forward_glu(self, x, bias, B, T, h, out, status):
        st = stream()
        if self.fwd_tc:
            self.run_tc(True, x, bias, None, B, T, 1, 1, 0, 0, h, None, out, None, status)
        else:
            call("bm_conv1d_glu_fwd", ptr(x), ptr(self.wf), ptr(bias), B, T, self.cin, self.cout // 2, self.kw,
                 ptr(h), ptr(out), st)

    def backward_data(self, dy, addend, B, T, dilation, dx, status):
        st = stream()
        if self.bwd_tc:
            self.run_tc(False, dy, None, addend, B, T, dilation, 0, 0, 0, dx, None, None, None, status)
        else:
            call("bm_conv1d_bwd_data", ptr(dy), ptr(self.wb), ptr(addend), B, T, self.cin, self.cout, self.kw,
                 dilation, ptr(dx), st)

    def backward_weight(self, dy, x, B, T, dilation, like, status, bias_grad_is_zero=False, known_dbias=None, want_w=True,
                        want_b=True):
        """`bias_grad_is_zero`: the conv feeds a training-mode BatchNorm, whose backward makes sum(dy) == 0 exactly
        (the reference's value there is rounding noise around 0); skip the reduction.  `known_dbias`: the producer of dy
        already summed it over the rows.  `want_w` / `want_b` False: that parameter is frozen; its gradient is neither
        computed nor returned (None)."""
        if not want_w:
            if not want_b:
                return None, None
            if known_dbias is not None:
                return None, known_dbias
            db = torch.zeros((self.cout,), device=like.device) if bias_grad_is_zero else _empty((self.cout,), like)
            if not bias_grad_is_zero:
                col_sum(dy, B * T, self.cout, db, stream())
            return None, db
        if not want_b:
            if self.wgrad_tc:
                return tc_wgrad(dy, x, B, T, self.cout, self.cin, self.cin_true, self.kw, dilation, status), None
            dw = _empty((self.cout, self.cin, self.kw), like)
            _reducing_call("bm_conv1d_bwd_weight", like, (B, T, self.cin, self.cout, self.kw), ptr(dy), ptr(x), B, T,
                           self.cin, self.cout, self.kw, dilation, ptr(dw), None, stream())
            return (dw[:, :self.cin_true].contiguous() if self.cin != self.cin_true else dw), None
        if self.wgrad_tc:
            if known_dbias is not None:
                return tc_wgrad(dy, x, B, T, self.cout, self.cin, self.cin_true, self.kw, dilation, status), known_dbias
            if bias_grad_is_zero:
                dw = tc_wgrad(dy, x, B, T, self.cout, self.cin, self.cin_true, self.kw, dilation, status)
                return dw, torch.zeros((self.cout,), device=like.device)
            db = _empty((self.cout,), like)
            dw = tc_wgrad(dy, x, B, T, self.cout, self.cin, self.cin_true, self.kw, dilation, status, dbias=db)
            return dw, db
        db = _empty((self.cout,), like)
        dw = _empty((self.cout, self.cin, self.kw), like)
        _reducing_call("bm_conv1d_bwd_weight", like, (B, T, self.cin, self.cout, self.kw), ptr(dy), ptr(x), B, T, self.cin, self.cout, self.kw,
                       dilation, ptr(dw), ptr(db), stream())
        if self.cin != self.cin_true:
            dw = dw[:, :self.cin_true].contiguous()
        return dw, db


def _epilogue(kind, has_bn, act, slope, head, tail=()):
    """(entry point, arguments before the stream) of a ConvSequence layer epilogue without gains, `kind` "fwd", "bwd",
    "bwd_reduce" or "bwd_apply": bm_bn_gelu_skip_* (amax_out NULL) for a BatchNorm + GELU layer, else bm_bn_act_skip_* with
    the activation code and slope.  head: the arguments up to C; tail: the ones after the activation's."""
    if has_bn and act == ACT_GELU:
        return "bm_bn_gelu_skip_" + kind, head + tail + ((None,) if kind in ("fwd", "bwd") else ())
    return "bm_bn_act_skip_" + kind, head + (act, float(slope)) + tail


# ----------------------------------------------------------------------------------------------------
# The ConvSequence layers (bm/models/common.py:142-151) on channels-last activations: SimpleConv's encoder and the
# stand-alone ConvSequence / DeepMel both run them through these two functions.
# ----------------------------------------------------------------------------------------------------
def _residual_branch_forward(plan: SequencePlan, k, p, x, y, mean, invstd, skip, act, save, nd: "_Needs", B, T, status,
                             bare_slope):
    """Epilogue of layer k with its residual-branch options (common.py:117-130): a = act(bn(y)); with `rewrite`
    r = LeakyReLU(conv1x1(a)) (else r = a); x_new = post * ((boost * scale) * r) (+ x).  The gains and the residual add run
    in `bm_bn_act_gain_skip_fwd` (without a gain, the rewrite's LeakyReLU and the add in `bm_bn_act_skip_fwd`).
    -> (x_new, the record entries `_residual_branch_backward` reads)"""
    st = stream()
    rows, cout = B * T, y.shape[2]
    _, _, gamma, beta, rw, rb, ls, ps = p
    if mean is not None:
        gamma, beta = gamma.contiguous(), beta.contiguous()
    ls = None if ls is None else ls.contiguous()
    ps = None if ps is None else ps.contiguous()            # [C, 1, 1]: one weight per channel
    gain = ls is not None or ps is not None
    slope = float(plan.act_slope if plan.has_act[k] else bare_slope)
    x_old = x if skip else None
    x_new = _empty((B, T, cout), x)
    rec = dict(gain=gain, ls=ls, ps=ps, rconv=None, a=None, y2=None)
    src = y
    if rw is not None:
        a = _empty((B, T, cout), x)
        name, args = _epilogue("fwd", mean is not None, act, slope,
                               (ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), None, ptr(a), rows, cout))
        call(name, *args, st)
        need_dy = nd.below[k] or any(nd.layer[k][:4])
        rconv = _Conv(rw, T, False, plan.use_tensor_cores, want_bwd=save and need_dy)
        y2 = _empty((B, T, cout), x)
        rconv.forward(a, rb.contiguous(), B, T, 1, y2, None, status)
        rec.update(rconv=rconv, a=a if nd.layer[k][4] else None, y2=y2 if nd.layer_up(k) else None)
        src, mean, invstd, gamma, beta, act, slope = y2, None, None, None, None, ACT_LRELU, plan.rewrite_slope
    if gain:
        call("bm_bn_act_gain_skip_fwd", ptr(src), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(x_old), ptr(x_new),
             rows, cout, act, float(slope), ptr(ls), float(plan.scale_boost), ptr(ps), st)
    else:
        call("bm_bn_act_skip_fwd", ptr(src), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(x_old), ptr(x_new), rows,
             cout, act, float(slope), st)
    return x_new, rec


def _residual_branch_backward(plan: SequencePlan, k, p, rec, g, nd: "_Needs", B, T, status, sums3, weight_grad):
    """Backward of `_residual_branch_forward` given g = dL/dx_new -> (dy, g_act, (d rewrite_w, d rewrite_b, d scale,
    d post_skip_w), dgamma, dbeta).  Without a rewrite conv the gain kernel also runs the BatchNorm / activation backward:
    dy = dL/dy and g_act None.  With one, dy is None and g_act = dL/da, the gradient the caller hands to the BatchNorm /
    activation backward.  Frozen gains are not reduced, a frozen rewrite conv gets no weight gradient, and nothing below
    the options is computed when no layer parameter or earlier stage needs it (dy and g_act None)."""
    st = stream()
    rows = B * T
    like = status
    cout = rec["conv"].cout
    _, _, gamma, beta, rw, rb, _, _ = p
    n_rw, n_rb, n_ls, n_ps = nd.layer[k][4:8]
    _, _, n_gamma, n_beta = nd.layer[k][:4]
    need_dy = nd.below[k] or any(nd.layer[k][:4])
    ls, ps = rec["ls"], rec["ps"]
    if rw is not None:
        src, mean, invstd, gm, bt = rec["y2"], None, None, None, None
        act, slope = ACT_LRELU, plan.rewrite_slope
        want_dsrc = need_dy or n_rw or n_rb
    else:
        src, mean, invstd = rec["y"], rec["mean"], rec["invstd"]
        gm, bt = (gamma.contiguous(), beta.contiguous()) if mean is not None else (None, None)
        act, slope = rec["act"], (plan.act_slope if plan.has_act[k] else 0.0)
        want_dsrc = need_dy
    dsrc = dgamma = dbeta = dls = dps = None
    batch_stats = mean is not None and bn_layer(plan, k).training
    if rec["gain"] and (want_dsrc or n_ls or n_ps):
        bn_reduce = mean is not None and (batch_stats or n_gamma or n_beta)
        if bn_reduce:
            dgamma, dbeta = _empty((cout,), like), _empty((cout,), like)
        dls = _empty((cout,), like) if n_ls else None
        dps = _empty((cout, 1, 1), like) if n_ps else None
        dsrc = _empty((B, T, cout), like)
        reduce = bool(bn_reduce or n_ls or n_ps)
        _reducing_call("bm_bn_act_gain_skip_bwd", like, (rows, cout), ptr(g), ptr(src), ptr(mean), ptr(invstd), ptr(gm),
                       ptr(bt), 1 if batch_stats else 0, rows, cout, act, float(slope), ptr(ls), float(plan.scale_boost),
                       ptr(ps), ptr(sums3 if reduce else None), ptr(dsrc), ptr(dgamma), ptr(dbeta), ptr(dls), ptr(dps), st,
                       reduces=reduce)
    elif not rec["gain"] and want_dsrc:                     # a rewrite without gain: the LeakyReLU backward alone
        dsrc = _empty((B, T, cout), like)
        call("bm_bn_act_skip_bwd", ptr(g), ptr(src), None, None, None, None, 0, rows, cout, ACT_LRELU, float(slope), None,
             ptr(dsrc), None, None, st)
    if rw is None:
        return (dsrc if need_dy else None), None, (None, None, dls, dps), dgamma, dbeta
    drw, drb = weight_grad(rec["rconv"], dsrc, rec["a"], 1, False, want=(n_rw, n_rb))
    g_act = None
    if need_dy:
        g_act = _empty((B, T, cout), like)
        rec["rconv"].backward_data(dsrc, None, B, T, 1, g_act, status)
    return None, g_act, (drw, drb, dls, dps), None, None

def conv_stack_forward(plan: SequencePlan, x, conv0: _Conv, conv_p, glu_p, nd: "_Needs", save: bool, B, T, status,
                       bare_slope: float):
    """x [B,T,C] -> (output [B,T,C_last], per-layer records for `conv_stack_backward`, None where the backward does not
    reach).  conv_p[k] = (conv_w, conv_b, gamma, beta), gamma / beta None without BatchNorm; glu_p[k] = (glu_w, glu_b).
    `conv0`: layer 0's prepared `_Conv`, its input padding chosen by the caller.  `save`: a backward will run.
    `bare_slope`: the slope handed to the epilogue kernel of a bare conv with a residual (act = none: the kernel ignores it)."""
    st = stream()
    rows = B * T
    tc = plan.use_tensor_cores
    # a syncing layer's count goes into slot 2C of its sums (`_sync_bn_sums`)
    stats = _empty((2 * max(p[0].shape[0] for p in conv_p) + (1 if plan.bn_groups else 0),), x, torch.float64)
    layers = []
    for k, p in enumerate(conv_p):
        w, b, gamma, beta = p[:4]
        conv = conv0 if k == 0 else _Conv(w, T, False, tc, want_bwd=save and nd.below[k])
        cout = conv.cout
        y = _empty((B, T, cout), x)
        keep = save and nd.below[k + 1]          # the backward reaches this layer
        has_bn = plan.has_act[k] and plan.batch_norm
        act = plan.act_code if plan.has_act[k] else ACT_NONE
        mean = invstd = None
        if has_bn:
            mean, invstd = _empty((cout,), x), _empty((cout,), x)
            rm, rv = plan.bn_buffers[k]
            group = plan.bn_groups[k] if plan.bn_groups else None
            layer = bn_layer(plan, k)
            if layer.training:
                conv.forward(x, b.contiguous(), B, T, plan.dilations[k], y, stats, status)
                if group is not None:
                    # SyncBatchNorm: one all-reduce per layer, issued whatever the data, so every rank issues the same ones
                    _sync_bn_sums(stats, cout, rows, group)
                _bn_finalize(stats, rows, group, layer, rm, rv, mean, invstd, cout, st)
            else:
                # eval mode (the module's, or this layer's alone): the running statistics, no statistics epilogue
                conv.forward(x, b.contiguous(), B, T, plan.dilations[k], y, None, status)
                call("bm_bn_eval_stats", ptr(rm), ptr(rv), float(layer.eps), ptr(mean), ptr(invstd), cout, st)
        else:
            conv.forward(x, b.contiguous(), B, T, plan.dilations[k], y, None, status)
        skip = plan.skip and conv.cin_true == cout
        x_new = y                                   # a bare convolution
        if len(p) > 4:
            x_new, extra = _residual_branch_forward(plan, k, p, x, y, mean, invstd, skip, act, save, nd, B, T, status,
                                                    bare_slope)
            rec = dict(x_in=x if nd.layer[k][0] else None,
                       y=y if (plan.has_act[k] or extra["gain"]) and nd.layer_up(k) else None, mean=mean, invstd=invstd,
                       conv=conv, skip=skip, act=act, has_bn=has_bn, x_new=x_new if nd.glu.get(k, (False,))[0] else None,
                       **extra)
        elif has_bn or act != ACT_NONE or skip:
            x_new = _empty((B, T, cout), x)
            gamma, beta = (gamma.contiguous(), beta.contiguous()) if has_bn else (None, None)
            name, args = _epilogue("fwd", has_bn, act, plan.act_slope if plan.has_act[k] else bare_slope,
                                   (ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(x) if skip else None, ptr(x_new),
                                    rows, cout))
            call(name, *args, st)
        if len(p) == 4:
            # kept: the conv input for its weight gradient, y for the activation backward, x_new for the GLU weight gradient
            rec = dict(x_in=x if nd.layer[k][0] else None, y=y if plan.has_act[k] and nd.layer_up(k) else None, mean=mean,
                       invstd=invstd, conv=conv, skip=skip, act=act, has_bn=has_bn,
                       x_new=x_new if nd.glu.get(k, (False,))[0] else None)
        x = x_new
        if plan.glu_after[k]:
            gw, gb = glu_p[k]
            gconv = _Conv(gw, T, True, tc, want_bwd=save and nd.layer_up(k))
            h = _empty((B, T, gconv.cout), x) if keep else None
            out = _empty((B, T, gconv.cout // 2), x)
            gconv.forward_glu(x, gb.contiguous(), B, T, h, out, status)
            rec.update(h=h, gconv=gconv)
            x = out
        layers.append(rec if keep else None)
    return x, layers


def conv_stack_backward(plan: SequencePlan, conv_p, layers, g, nd: "_Needs", B, T, status, side=None, keep_alive=None):
    """g = dL/d(output of conv_stack_forward) [B,T,C_last] -> (per layer (d conv_w, d conv_b, d gamma, d beta),
    {k: (d glu_w, d glu_b)}, dL/dx); None for every gradient not asked for, and dL/dx only if nd.below[0].  The backward
    stops at the deepest layer that needs a gradient.  `side`, `keep_alive`: the weight-gradient kernels run through
    `_on_side`, concurrent with the data-gradient kernels (side None: inline)."""
    st = stream()
    rows = B * T
    like = status                                   # allocations only read the device off it
    sums = _empty((2 * max(p[0].shape[0] for p in conv_p) + (1 if plan.bn_groups else 0),), like, torch.float64)
    sums3 = _empty((3 * max(p[0].shape[0] for p in conv_p),), like, torch.float64) if plan.residual else None
    layer_grads: tp.List[tp.Any] = [(None,) * len(p) for p in conv_p]
    glu_grads = {k: (None, None) for k in nd.glu}

    def weight_grad(conv: _Conv, dy, x, dilation, bias_zero, known_dbias=None, want=(True, True)):
        if not any(want):
            return None, None
        return _on_side(side, keep_alive, lambda: conv.backward_weight(
            dy, x, B, T, dilation, like, status, bias_grad_is_zero=bias_zero, known_dbias=known_dbias, want_w=want[0],
            want_b=want[1]), dy, x)

    for k in reversed(range(len(conv_p))):
        if not nd.below[k + 1]:
            break                                  # nothing at or below this layer requires grad
        rec = layers[k]
        _, _, gamma, beta = conv_p[k][:4]
        conv: _Conv = rec["conv"]
        cout = conv.cout
        n_cw, n_cb, n_gamma, n_beta = nd.layer[k][:4]
        if plan.glu_after[k]:
            gconv: _Conv = rec["gconv"]
            n_gw, n_gb = nd.glu[k]
            dh = _empty((B, T, gconv.cout), like)
            dgb = _empty((gconv.cout,), like) if n_gb else None    # the GLU conv's bias gradient, summed while dh is made
            _reducing_call("bm_glu_bwd", like, (rows, gconv.cout // 2), ptr(g), ptr(rec["h"]), rows, gconv.cout // 2,
                           ptr(dh), ptr(dgb), None, st, reduces=n_gb)
            glu_grads[k] = weight_grad(gconv, dh, rec["x_new"], 1, False, dgb, want=(n_gw, n_gb))
            if not nd.layer_up(k):
                del dh
                break
            g = _empty((B, T, gconv.cin), like)
            gconv.backward_data(dh, None, B, T, 1, g, status)
            del dh
        dgamma = dbeta = dy = None
        g_act, opt_grads = g, ()                    # the gradient at the activation's output; the options' gradients
        if len(conv_p[k]) > 4:
            dy, g_act, opt_grads, dgamma, dbeta = _residual_branch_backward(plan, k, conv_p[k], rec, g, nd, B, T, status,
                                                                            sums3, weight_grad)
            if dy is None and g_act is None:        # nothing below the residual-branch options needs a gradient
                layer_grads[k] = (None, None, None, None) + opt_grads
                continue
        group = plan.bn_groups[k] if plan.bn_groups else None
        batch_stats = rec["has_bn"] and bn_layer(plan, k).training
        if dy is not None:
            pass                                    # the gain kernel ran the BatchNorm / activation backward
        elif rec["has_bn"] and group is not None:
            # SyncBatchNorm (torch's SyncBatchNorm backward): dgamma / dbeta from the local sums; the data gradient, when
            # the layer's input needs one (torch's needs_input_grad[0]), from the group's sums after their all-reduce.
            # Whether that all-reduce is issued depends on requires_grad flags only, never on data, so every rank issues
            # the same collectives in the same order (DESIGN 4.1).
            dgamma, dbeta = _empty((cout,), like), _empty((cout,), like)
            gm, bt = gamma.contiguous(), beta.contiguous()
            head = (ptr(g_act), ptr(rec["y"]), ptr(rec["mean"]), ptr(rec["invstd"]), ptr(gm), ptr(bt), rows, cout)
            name, args = _epilogue("bwd_reduce", True, rec["act"], plan.act_slope, head, (ptr(sums), ptr(dgamma), ptr(dbeta)))
            _reducing_call(name, like, (rows, cout), *args, st)
            if n_cw or n_cb or nd.below[k]:
                _sync_bn_sums(sums, cout, rows, group)
                dy = _empty((B, T, cout), like)
                name, args = _epilogue("bwd_apply", True, rec["act"], plan.act_slope, head, (ptr(sums), ptr(dy)))
                call(name, *args, st)
        elif rec["has_bn"]:
            # the batch statistics' backward reduces in training mode; in eval mode only for trainable gamma / beta (else
            # the BatchNorm + activation backward is one elementwise pass)
            reduce = batch_stats or n_gamma or n_beta
            dy = _empty((B, T, cout), like)
            dgamma, dbeta = (_empty((cout,), like), _empty((cout,), like)) if reduce else (None, None)
            name, args = _epilogue("bwd", True, rec["act"], plan.act_slope,
                                   (ptr(g_act), ptr(rec["y"]), ptr(rec["mean"]), ptr(rec["invstd"]), ptr(gamma.contiguous()),
                                    ptr(beta.contiguous()), 1 if batch_stats else 0, rows, cout),
                                   (ptr(sums if reduce else None), ptr(dy), ptr(dgamma), ptr(dbeta)))
            _reducing_call(name, like, (rows, cout), *args, st, reduces=reduce)
        elif rec["act"] != ACT_NONE:
            dy = _empty((B, T, cout), like)
            call("bm_bn_act_skip_bwd", ptr(g_act), ptr(rec["y"]), None, None, None, None, 0, rows, cout, rec["act"],
                 float(plan.act_slope), None, ptr(dy), None, None, st)
        else:
            # bare convolution: dL/dy = dL/dx_new.  With a residual, g is accumulated in place below while the weight
            # gradient may still read dy: dy is then a copy
            dy = g.clone() if (rec["skip"] and nd.below[k]) else g
        # with a training-mode BatchNorm behind the conv, sum(dy) is exactly 0: no bias reduction (a SyncBatchNorm's is 0
        # summed over the group only)
        dcw, dcb = weight_grad(conv, dy, rec["x_in"], plan.dilations[k], batch_stats and group is None,
                               want=(n_cw, n_cb))
        if not nd.below[k]:
            pass
        elif rec["skip"]:
            # in place: g += conv_transpose(dy) (addend == output: the conv epilogue adds g and stores the sum over it)
            conv.backward_data(dy, g, B, T, plan.dilations[k], g, status)
        else:
            g_in = _empty((B, T, conv.cin), like)
            conv.backward_data(dy, None, B, T, plan.dilations[k], g_in, status)
            g = g_in
        layer_grads[k] = (dcw, dcb, dgamma if n_gamma else None, dbeta if n_beta else None) + opt_grads
        del dy, g_act
    return layer_grads, glu_grads, g


# ----------------------------------------------------------------------------------------------------
# The sensor-side front (simpleconv.py:104-151, 207-233): ChannelMerger attention -> sensor mix -> initial_linear ->
# SubjectLayers -> subject embedding, on channels-last activations.  A stage whose parameters are None is absent (the
# ablation rows merger=False / initial_linear=0 / subject_layers=False / subject_dim, grids/nmi/ablation_final.py:44,46,50,51).
# SimpleConv's encoder runs it through `front_forward` / `front_backward`; the stand-alone ChannelMerger and SubjectLayers
# call its FP32-FMA stage helpers.
# ----------------------------------------------------------------------------------------------------
def _attention_fwd(heads, positions, freq, ban_centre, radius, C):
    """ChannelMerger attention weights of every recording on the FP32-FMA kernel -> (emb [R,C,P], att [R,O,C])."""
    R, (O, P) = positions.shape[0], heads.shape
    emb, att = _empty((R, C, P), heads), _empty((R, O, C), heads)
    call("bm_attention_weights_fwd", ptr(positions), ptr(freq), ptr(heads.contiguous()), ptr(ban_centre), float(radius), R,
         C, O, P, ptr(emb), ptr(att), stream())
    return emb, att


def _attention_bwd(d_att, att, emb):
    """dheads [O,P] from the attention weights' gradient d_att [R,O,C], on the FP32-FMA kernel."""
    R, O, C = att.shape
    P = emb.shape[2]
    dscores, dheads = _empty((R, O, C), att), _empty((O, P), att)
    _reducing_call("bm_attention_weights_bwd", att, None, ptr(d_att), ptr(att), ptr(emb), R, C, O, P, ptr(dscores),
                   ptr(dheads), stream())
    return dheads


def _mix_fwd(meg, att, rec_of_sample, u):
    """u[b,t,o] = sum_c att[rec_b][o][c] meg[b,c,t] on the FP32-FMA kernel, into the first O columns of u [B,T,ld]."""
    B, C, T = meg.shape
    call("bm_sensor_mix_fwd", ptr(meg), ptr(att), ptr(rec_of_sample), B, C, T, att.shape[1], u.shape[2], ptr(u), stream())


def _mix_bwd(du, meg, att, rec_order, rec_off):
    """The mix's weight gradient d_att [R,O,C] from du [B,T,ld], samples grouped by recording, on the FP32-FMA kernel."""
    B, C, T = meg.shape
    R, O, _ = att.shape
    d_att = _empty((R, O, C), meg)
    call("bm_sensor_mix_bwd", ptr(du), du.shape[2], ptr(meg), ptr(rec_order), ptr(rec_off), B, C, T, O, R, ptr(d_att),
         stream())
    return d_att


def _mix_bwd_data(du, att, rec_of_sample, mask):
    """dmeg [B,C,T] = mask[c] * sum_o att[rec_b][o][c] du[b,t,o] (mask None: no mask) on the FP32-FMA kernel."""
    B, T = du.shape[:2]
    _, O, C = att.shape
    dmeg = _empty((B, C, T), du)
    call("bm_sensor_mix_bwd_data", ptr(du), du.shape[2], ptr(att), ptr(rec_of_sample), ptr(mask), B, C, T, O, ptr(dmeg),
         stream())
    return dmeg


def _subject_fwd(x, subj_w, subject, out):
    """out[b,t,:D] = x[b,t,:IL] @ subj_w[subject_b] on the FP32-FMA kernel; x [B,T,ld_x], out [B,T,ld_out]."""
    B, T = x.shape[:2]
    _, IL, D = subj_w.shape
    call("bm_subject_layers_fwd", ptr(x), x.shape[2], ptr(subj_w.contiguous()), ptr(subject), B, T, IL, D, out.shape[2],
         ptr(out), stream())


def _subject_bwd(g, x, subj_w, subject, shape, ld, want_dx, want_dw):
    """g [B,T,ld_g] (first D columns) -> (dx [B,T,ld], d_subj_w [S,IL,D]) on the FP32-FMA kernel, None where not wanted.
    shape = (S, IL, D); x [B,T,ld], the forward input, is read for d_subj_w only, subj_w for dx only.  The pad columns of dx
    are zero: a tensor-core contraction reads them."""
    S, IL, D = shape
    B, T = g.shape[:2]
    order, off = group_layout(subject, S) if want_dw else (None, None)
    dx = None
    if want_dx:
        dx = torch.zeros((B, T, ld), device=g.device) if ld != IL else _empty((B, T, ld), g)
    dw = _empty((S, IL, D), g) if want_dw else None
    call("bm_subject_layers_bwd", ptr(g), g.shape[2], ptr(x), ld, ptr(subj_w), ptr(subject), ptr(order), ptr(off), B, T, IL,
         D, S, ld, ptr(dx), ptr(dw), stream())
    return dx, dw


def front_forward(plan: "EncoderPlan", meg, heads, il_w, il_b, subj_w, sub_emb, w0, nd: "_Needs", save: bool, status):
    """meg [B,C,T] -> (x [B,T,Dp] channels-last input of conv layer 0, conv0 = layer 0's prepared `_Conv` of weight w0 with
    its input padded to Dp, the record `front_backward` reads).  heads, (il_w, il_b), subj_w, sub_emb [B,E]: the stages'
    parameters, None where a stage is absent.  `save`: a backward will run.  w0 None (concatenate: layer 0 reads the
    joined streams, whose width the caller pads): conv0 is None; x is still zero-padded to a multiple of 64 channels in
    the complete chain on the tensor cores (rec["width"]: its valid columns, rec["pad_width"]: its row length).

    Kernel choice: the tensor-core stages run only in the complete chain (merger, initial_linear and subject layers, no
    subject embedding), each where its padded widths pass the shape gates; a complete chain whose initial_linear is not on
    the tensor cores is the fused FP32-FMA `bm_sensor_chain_fwd`; everything else runs the FP32-FMA stage kernels one by one,
    with layer 0 unpadded."""
    st = stream()
    lib = _lib.load()
    B, C, T = meg.shape
    R = plan.rec_positions.shape[0]
    n_meg, n_heads, n_il_w, _, n_subj, _ = nd.front
    want_bwd0 = save and nd.below[0]
    chain = heads is not None and il_w is not None and subj_w is not None and sub_emb is None
    tc = chain and plan.use_tensor_cores
    O = heads.shape[0] if heads is not None else C          # the mix, initial_linear and subject-layer output widths
    IL = il_w.shape[0] if il_w is not None else O
    D = subj_w.shape[2] if subj_w is not None else IL
    Op, ILp, Dp = O, IL, D                                  # ... and their widths in the buffers, zero-padded
    rec = dict(meg=meg, chain=chain, emb=None, att=None, heads_tc=False, megT=None, subj_pad=None)

    def _padded(width_pad, width, written_in_full):
        """[B,T,width_pad]; the pad columns need a fill only where an FP32-FMA kernel (valid columns only) writes it"""
        if width_pad == width or written_in_full:
            return _empty((B, T, width_pad), meg)
        return torch.zeros((B, T, width_pad), device=meg.device)

    if heads is not None:
        # K1 attention weights per recording (the score contraction on the tensor cores when the widths fit)
        P = heads.shape[1]
        Opad = _round_up(O, 64)
        if tc and bool(lib.bm_tc_conv1d_persistent_supported(C, P, Opad, 1, 0)) and bool(lib.bm_tc_wgrad_supported(Opad, P)):
            hpad = torch.zeros((Opad, P, 1), device=meg.device)
            hpad[:O, :, 0] = heads
            heads_conv = _Conv(hpad, C, False, True, want_bwd=False)
            emb = _empty((R, C, P), meg)
            call("bm_fourier_emb", ptr(plan.rec_positions), ptr(plan.freq), R, C, P, ptr(emb), st)
            att_full = _empty((R, Opad, C), meg)          # scores[r][o][c] = <emb[r][c], heads[o]> written channel-major
            heads_conv.run_tc(True, emb, None, None, R, C, 1, 0, 0, 1, att_full, None, None, None, status)
            call("bm_masked_softmax", ptr(att_full), ptr(plan.rec_positions), ptr(plan.ban_centre), float(plan.ban_radius),
                 R, Opad, C, st)
            att = att_full[:, :O].contiguous()
            rec["heads_tc"] = True
        else:
            emb, att = _attention_fwd(heads, plan.rec_positions, plan.freq, plan.ban_centre, plan.ban_radius, C)
        rec.update(emb=emb, att=att)

    conv0 = il_conv = None
    if chain and w0 is None and plan.use_tensor_cores:
        Dp = _round_up(D, 64)        # concatenate: x0 padded as for layer 0, so the subject layers keep their tensor-core form
    elif chain and w0 is not None:
        # x0 kept zero-padded to a multiple of 64 channels when the tensor-core conv follows
        Dp = _round_up(D, 64)
        conv0 = _Conv(w0, T, False, plan.use_tensor_cores, pad_cin_to=Dp, want_bwd=want_bwd0)
        if not conv0.fwd_tc:
            Dp = D
            conv0 = _Conv(w0, T, False, False, want_bwd=want_bwd0)
    if tc:
        # `initial_linear` on the tensor cores when the (64-padded) widths fit: u and v are then kept zero-padded
        Op, ILp = _round_up(O, 64), _round_up(IL, 64)
        wpad = torch.zeros((ILp, Op, 1), device=meg.device)
        wpad[:IL, :O, 0] = il_w.reshape(IL, O)
        il_conv = _Conv(wpad, T, False, True, want_bwd=save and (n_meg or n_heads))
        if not (il_conv.fwd_tc and il_conv.bwd_tc and il_conv.wgrad_tc):
            il_conv = None
            Op, ILp = O, IL
    Cp = _round_up(C, 128)
    mix_tc = il_conv is not None and bool(lib.bm_tc_conv_supported(T, Cp, Op, 1, 0)) and \
        bool(lib.bm_tc_wgrad_supported(Op, Cp))
    subj_tc = il_conv is not None and (Dp != D or D % 64 == 0) and bool(lib.bm_tc_conv_supported(T, ILp, Dp, 1, 0)) and \
        bool(lib.bm_tc_conv_supported(T, Dp, ILp, 1, 0)) and bool(lib.bm_tc_wgrad_supported(ILp, Dp))

    if chain and il_conv is None:
        # One call: the library's own composition of the three FP32-FMA stage kernels, which the pinned call streams hold.
        u, v, x = _empty((B, T, O), meg), _empty((B, T, IL), meg), _padded(Dp, D, False)
        call("bm_sensor_chain_fwd", ptr(meg), ptr(att), ptr(plan.rec_of_sample), ptr(il_w.reshape(IL, O).contiguous()),
             ptr(il_b.contiguous()), ptr(subj_w.contiguous()), ptr(plan.subject), B, C, T, O, IL, D, Dp, ptr(u), ptr(v),
             ptr(x), st)
    else:
        # K2 sensor mix (without a merger: the raw sensors, channels-last)
        if heads is None:
            u = _empty((B, T, C), meg)
            call("bm_transpose_nt", ptr(meg), B, C, T, ptr(u), st)
        elif mix_tc:
            # meg transposed once to channels-last (sensor count padded to 128), then u = megT @ att[rec]^T is a pointwise
            # contraction with a per-sample weight set (one per recording)
            u = _padded(Op, O, True)
            megT = _empty((B, T, Cp), meg)                 # the transpose writes the pad columns as zeros
            call("bm_transpose_nt_ld", ptr(meg), B, C, T, Cp, ptr(megT), st)
            att_pad = torch.zeros((R, Op, Cp), device=meg.device)
            att_pad[:, :O, :C] = att
            aw_hi, aw_lo = _empty((R * Op, Cp), meg), _empty((R * Op, Cp), meg)
            call("bm_tc_weight_split", ptr(att_pad), R * Op, Cp, 1, ptr(aw_hi), ptr(aw_lo), None, None, st)
            _tc_call("bm_tc_pointwise_sel", ptr(megT), ptr(aw_hi), ptr(aw_lo), ptr(plan.rec_of_sample), R, B, T, Cp, Op,
                     ptr(u), ptr(status), st)
            rec["megT"] = megT
        else:
            u = _padded(Op, O, False)
            _mix_fwd(meg, att, plan.rec_of_sample, u)
        # initial_linear (simpleconv.py:112-120)
        v = u
        if il_conv is not None:
            v = _empty((B, T, ILp), meg)
            bpad = torch.zeros((ILp,), device=meg.device)
            bpad[:IL] = il_b
            il_conv.forward(u, bpad, B, T, 1, v, None, status)
        elif il_w is not None:
            v = _empty((B, T, IL), meg)
            call("bm_initial_linear_fwd", ptr(u), O, ptr(il_w.reshape(IL, O).contiguous()), ptr(il_b.contiguous()), B, T, O,
                 IL, IL, ptr(v), st)
        # SubjectLayers (common.py:45-62)
        x = v
        if subj_tc:
            # per-subject weights, zero-padded; forward operand [s][d][p] (K-major in p), tf32-split
            S = subj_w.shape[0]
            x = _padded(Dp, D, True)
            subj_pad = torch.zeros((S, ILp, Dp), device=meg.device)
            subj_pad[:, :IL, :D] = subj_w
            mt = subj_pad.transpose(1, 2).contiguous()
            sf_hi, sf_lo = _empty((S * Dp, ILp), meg), _empty((S * Dp, ILp), meg)
            call("bm_tc_weight_split", ptr(mt), S * Dp, ILp, 1, ptr(sf_hi), ptr(sf_lo), None, None, st)
            _tc_call("bm_tc_pointwise_sel", ptr(v), ptr(sf_hi), ptr(sf_lo), ptr(plan.subject), S, B, T, ILp, Dp, ptr(x),
                     ptr(status), st)
            rec["subj_pad"] = subj_pad
        elif subj_w is not None:
            x = _padded(Dp, D, False)
            _subject_fwd(v, subj_w, plan.subject, x)
    if sub_emb is not None:                                    # ScaledEmbedding appended as channels (simpleconv.py:231-233)
        x = torch.cat([x, sub_emb[:, None, :].expand(B, T, sub_emb.shape[1])], dim=2).contiguous()
    if conv0 is None and w0 is not None:
        conv0 = _Conv(w0, T, False, plan.use_tensor_cores, want_bwd=want_bwd0)
    # u and v (the initial_linear and subject-layer inputs) are read by those stages' weight gradients only
    rec.update(u=u if n_il_w else None, v=v if n_subj else None, il_conv=il_conv, widths=(O, IL, D), pads=(Op, ILp, Dp),
               width=D + (0 if sub_emb is None else sub_emb.shape[1]), pad_width=x.shape[2])
    return x, conv0, rec


def front_backward(plan: "EncoderPlan", rec, g, heads, il_w, subj_w, sub_emb, need, status):
    """g = dL/dx [B,T,Dp] (x of `front_forward`) -> (dheads, d_il_w, d_il_b, d_subj, d_sub_emb, dmeg); None where a stage is
    absent or its gradient is not asked for.  need = requires-grad of (meg, heads, il_w, il_b, subj_w, sub_emb): each stage
    computes the gradients asked of it, and its data gradient only while a stage below it still needs one."""
    st = stream()
    meg, att, il_conv, megT = rec["meg"], rec["att"], rec["il_conv"], rec["megT"]
    B, C, T = meg.shape
    R = plan.rec_positions.shape[0]
    O, IL, D = rec["widths"]
    Op, ILp, Dp = rec["pads"]
    n_meg, n_heads, n_il_w, n_il_b, n_subj, n_emb = need
    want_dv = n_meg or n_heads or n_il_w or n_il_b          # the gradient at the subject layers' input
    want_du = n_meg or n_heads                              # ... and at initial_linear's input
    dheads = d_il_w = d_il_b = d_subj = d_sub_emb = dmeg = d_att = None
    if sub_emb is not None:
        if n_emb:
            d_sub_emb = g[:, :, D:].sum(dim=1)               # the embedding is constant over time
        g = g[:, :, :D].contiguous() if any(need[:5]) else None

    if rec["chain"] and il_conv is None:
        S = subj_w.shape[0]
        subj_order, subj_off = group_layout(plan.subject, S) if n_subj else (None, None)
        dv = _empty((B, T, IL), meg) if want_dv else None
        du = _empty((B, T, O), meg) if want_du else None
        d_subj = _empty((S, IL, D), meg) if n_subj else None
        d_il_w = _empty((IL, O), meg) if n_il_w else None
        d_il_b = _empty((IL,), meg) if n_il_b else None
        d_att = _empty((R, O, C), meg) if n_heads else None
        _reducing_call("bm_sensor_chain_bwd", meg, (B, T, O, IL), ptr(g), ptr(meg), ptr(il_w.reshape(IL, O).contiguous()),
                       ptr(subj_w.contiguous()), ptr(plan.subject), ptr(rec["u"]), ptr(rec["v"]), ptr(subj_order),
                       ptr(subj_off), ptr(plan.rec_order), ptr(plan.rec_off), B, C, T, O, IL, D, Dp, S, R, ptr(dv), ptr(du),
                       ptr(d_subj), ptr(d_il_w), ptr(d_il_b), ptr(d_att), st, reduces=n_il_w or n_il_b)
    else:
        # SubjectLayers
        dv = g
        if rec["subj_pad"] is not None:
            S = subj_w.shape[0]
            dv = None
            if want_dv:
                subj_pad = rec["subj_pad"]                               # [S][ILp][Dp]: data-gradient operand as is
                sb_hi, sb_lo = _empty((S * ILp, Dp), meg), _empty((S * ILp, Dp), meg)
                call("bm_tc_weight_split", ptr(subj_pad), S * ILp, Dp, 1, ptr(sb_hi), ptr(sb_lo), None, None, st)
                dv = _empty((B, T, ILp), meg)
                _tc_call("bm_tc_pointwise_sel", ptr(g), ptr(sb_hi), ptr(sb_lo), ptr(plan.subject), S, B, T, Dp, ILp,
                         ptr(dv), ptr(status), st)
            if n_subj:
                subj_order, subj_off = group_layout(plan.subject, S)
                dm = _empty((S, _round_up(ILp, 128), Dp), meg)
                _tc_call("bm_tc_wgrad_grouped", ptr(rec["v"]), ptr(g), ptr(subj_order), ptr(subj_off), S, B, T, ILp, Dp,
                         ptr(dm), ptr(status), st)
                d_subj = dm[:, :IL, :D].contiguous()
        elif subj_w is not None and (want_dv or n_subj):
            dv, d_subj = _subject_bwd(g, rec["v"], subj_w.contiguous(), plan.subject, subj_w.shape, ILp, want_dv, n_subj)
        # initial_linear
        du = dv if il_w is None else None
        if il_conv is not None:
            if want_du:
                du = _empty((B, T, Op), meg)
                il_conv.backward_data(dv, None, B, T, 1, du, status)
            if n_il_w:
                dbp = _empty((ILp,), meg) if n_il_b else None
                d_il_w = tc_wgrad(dv, rec["u"], B, T, ILp, Op, O, 1, 1, status, dbias=dbp)[:IL, :, 0].contiguous()
                d_il_b = dbp[:IL].contiguous() if n_il_b else None
            elif n_il_b:
                dbp = _empty((ILp,), meg)
                col_sum(dv, B * T, ILp, dbp, st)
                d_il_b = dbp[:IL].contiguous()
        elif il_w is not None and want_dv:
            # du feeds the merger's and meg's gradients.  Without a merger it is kept whenever this stage runs: one GEMM
            # onto the raw sensors, and a trainable step keeps the call stream it has always had
            du = _empty((B, T, O), meg) if (want_du or heads is None) else None
            d_il_w = _empty((IL, O), meg) if n_il_w else None
            d_il_b = _empty((IL,), meg) if n_il_b else None
            _reducing_call("bm_initial_linear_bwd", meg, (B, T, O, IL), ptr(dv), IL, ptr(rec["u"]), O,
                           ptr(il_w.reshape(IL, O).contiguous()), B, T, O, IL, O, ptr(du), ptr(d_il_w), ptr(d_il_b), st,
                           reduces=bool(n_il_w or n_il_b))
        # the sensor mix's weight gradient
        if not n_heads:
            pass
        elif megT is not None:
            Cp = megT.shape[2]
            dwp = _empty((R, _round_up(Op, 128), Cp), meg)
            _tc_call("bm_tc_wgrad_grouped", ptr(du), ptr(megT), ptr(plan.rec_order), ptr(plan.rec_off), R, B, T, Op, Cp,
                     ptr(dwp), ptr(status), st)
            d_att = dwp[:, :O, :C].contiguous()
        else:
            d_att = _mix_bwd(du, meg, att, plan.rec_order, plan.rec_off)

    def meg_grad():
        """dmeg [B,C,T] from du, the gradient at the mix output (without a merger: at the raw sensors, channels-last)"""
        if heads is None:
            dmeg = _empty((B, C, T), meg)
            call("bm_transpose_nt", ptr(du), B, T, C, ptr(dmeg), st)
            if plan.channel_mask is not None:
                call("bm_channel_mask", ptr(dmeg), ptr(plan.channel_mask), B, C, T, ptr(dmeg), st)
            return dmeg
        if megT is None or not bool(_lib.load().bm_tc_conv_supported(T, Op, megT.shape[2], 1, 0)):
            return _mix_bwd_data(du, att, plan.rec_of_sample, plan.channel_mask)
        # on the tensor cores when the mix ran there and the transposed contraction fits their shape gate
        Cp = megT.shape[2]
        dmeg = _empty((B, C, T), meg)
        att_t = torch.zeros((R, Cp, Op), device=meg.device)           # weight set r: [c][o], zero-padded
        att_t[:, :C, :O] = att.transpose(1, 2)
        w_hi, w_lo = _empty((R * Cp, Op), meg), _empty((R * Cp, Op), meg)
        call("bm_tc_weight_split", ptr(att_t), R * Cp, Op, 1, ptr(w_hi), ptr(w_lo), None, None, st)
        _tc_call("bm_tc_sensor_mix_bwd_data", ptr(du), ptr(w_hi), ptr(w_lo), ptr(plan.rec_of_sample), R,
                 ptr(plan.channel_mask), B, T, Op, Cp, C, ptr(dmeg), ptr(status), st)
        return dmeg

    # the complete chain forms dmeg before the attention backward, the stage-by-stage front after it (the pinned call order)
    if n_meg and rec["chain"]:
        dmeg = meg_grad()
    if n_heads and rec["heads_tc"]:
        emb, P = rec["emb"], heads.shape[1]
        Opad = _round_up(O, 64)
        dscores = _empty((R, O, C), meg)
        call("bm_softmax_bwd", ptr(att), ptr(d_att), R * O, C, ptr(dscores), st)
        ds_t = _empty((R, C, Opad), meg)                   # pad columns zeroed by the transpose
        call("bm_transpose_nt_ld", ptr(dscores), R, O, C, Opad, ptr(ds_t), st)
        dheads = tc_wgrad(ds_t, emb, R, C, Opad, P, P, 1, 1, status)[:O, :, 0].contiguous()
    elif n_heads:
        dheads = _attention_bwd(d_att, att, rec["emb"])
    if n_meg and not rec["chain"]:
        dmeg = meg_grad()
    if d_il_w is not None:
        d_il_w = d_il_w.reshape(il_w.shape)
    return dheads, d_il_w, d_il_b, d_subj, d_sub_emb, dmeg


# ----------------------------------------------------------------------------------------------------
# The output head (simpleconv.py:185-193, 245): `final` = 1x1 Conv1d [2H,H] -> activation -> 1x1 ConvTranspose1d [2H,F] on
# the channels-last output of the conv stack, handed out channel-major; with complex_out=False only the transpose.
# ----------------------------------------------------------------------------------------------------
def head_forward(plan: "EncoderPlan", x, w0, b0, w2, b2, nd: "_Needs", save: bool, B, T, status, want_g=None):
    """x [B,T,H] (the conv stack's output) -> (estimate [B,F,T], the record `head_backward` reads).  w0, b0, w2, b2: the
    Conv1d and ConvTranspose1d parameters, all None without a head, w0 and b0 None with linear_out.  `save`: a backward
    will run.  `want_g`: the gradient at x is needed (None: nd.below[-1]).  The form is chosen here:
      bare       no head: the stack already ends on out_channels, the estimate is its transpose;
      linear     linear_out (simpleconv.py:182-184): the 1x1 ConvTranspose alone as a `_Conv`, storing channel-major from
                 the tensor-core epilogue where the gates pass, else on FP32 FMA followed by a transpose;
      generic    an activation other than GELU: the two convs as `_Conv`s with the activation kernel between them, then a
                 transpose to channel-major;
      tc         GELU, and both convs pass the tensor-core gates both ways: the GELU and the channel-major store fused into
                 the conv epilogues, and the weight gradients on the tensor cores (on the side stream);
      tc_params  the same where the weight gradients' shapes do not fit the tensor cores: they come from
                 `bm_head_bwd_params`;
      fma        GELU, a conv gate fails: the FP32-FMA `bm_head_fwd` / `bm_head_bwd`."""
    st = stream()
    if w2 is None:
        F = x.shape[2]
        est = _empty((B, F, T), x)
        call("bm_transpose_nt", ptr(x), B, T, F, ptr(est), st)
        return est, dict(form="bare", F=F)
    n_w0, n_b0, n_w2, _ = nd.head
    if want_g is None:
        want_g = nd.below[-1]                        # the gradient at the head's input (the stack's output)
    tc = plan.use_tensor_cores
    if w0 is None:
        H, F = w2.shape[0], w2.shape[1]
        lin = _Conv(w2.permute(1, 0, 2).contiguous(), T, False, tc, want_bwd=save and want_g)    # as a conv: [F, H, 1]
        est = _empty((B, F, T), x)
        if lin.fwd_tc:
            lin.run_tc(True, x, b2.contiguous(), None, B, T, 1, 0, 0, 1, est, None, None, None, status)
        else:
            est_cl = _empty((B, T, F), x)
            lin.forward(x, b2.contiguous(), B, T, 1, est_cl, None, status)
            call("bm_transpose_nt", ptr(est_cl), B, T, F, ptr(est), st)
        return est, dict(form="linear", H=H, F=F, want_g=want_g, lin=lin, x_last=x if n_w2 else None)
    H, F = w0.shape[1], w2.shape[1]
    H2 = 2 * H
    want_dh1 = want_g or n_w0 or n_b0                # ... and below the head's activation
    head0 = _Conv(w0, T, False, tc, want_bwd=save and want_g)                                    # [2H, H, 1]
    head2 = _Conv(w2.permute(1, 0, 2).contiguous(), T, False, tc, want_bwd=save and want_dh1)    # as a conv: [F, 2H, 1]
    h1, q, est = _empty((B, T, H2), x), _empty((B, T, H2), x), _empty((B, F, T), x)
    if plan.act_code != ACT_GELU:
        form = "generic"
    elif head0.fwd_tc and head2.fwd_tc and head0.bwd_tc and head2.bwd_tc:
        form = "tc" if head0.wgrad_tc and bool(_lib.load().bm_tc_wgrad_supported(H2, F)) else "tc_params"
    else:
        form = "fma"
    w0_2, w2_2 = w0.reshape(H2, H).contiguous(), w2.reshape(H2, F).contiguous()
    if form == "fma":
        call("bm_head_fwd", ptr(x), ptr(w0_2), ptr(b0.contiguous()), ptr(w2_2), ptr(b2.contiguous()), B, T, H, F, ptr(h1),
             ptr(q), ptr(est), st)
    elif form == "generic":
        head0.forward(x, b0.contiguous(), B, T, 1, h1, None, status)
        call("bm_bn_act_skip_fwd", ptr(h1), None, None, None, None, None, ptr(q), B * T, H2, plan.act_code,
             float(plan.act_slope), st)
        est_cl = _empty((B, T, F), x)
        head2.forward(q, b2.contiguous(), B, T, 1, est_cl, None, status)
        call("bm_transpose_nt", ptr(est_cl), B, T, F, ptr(est), st)
    else:
        head0.run_tc(True, x, b0.contiguous(), None, B, T, 1, 0, 1, 0, q, h1 if save else None, None, None, status)
        head2.run_tc(True, q, b2.contiguous(), None, B, T, 1, 0, 0, 1, est, None, None, None, status)
    return est, dict(form=form, H=H, F=F, want_g=want_g, want_dh1=want_dh1, head0=head0, head2=head2, w0_2=w0_2, w2_2=w2_2,
                     h1=h1, x_last=x if n_w0 else None, q=q if n_w2 else None)


def head_backward(plan: "EncoderPlan", rec, dest, need, B, T, status, side, keep_alive):
    """dest = dL/d(estimate) [B,F,T] -> (g = dL/dx [B,T,H] of `head_forward`'s x, d w0, d b0, d w2, d b2); None for every
    gradient not asked for, and g only if the forward's `nd.below` asked for it.  need = requires-grad of (w0, b0, w2, b2).
    `side`, `keep_alive`: the tensor-core weight gradients run through `_on_side`."""
    st = stream()
    dest = dest.contiguous()
    form = rec["form"]
    if form == "bare":
        g = _empty((B, T, rec["F"]), dest)   # the gradient of the estimate IS the stack's output gradient
        call("bm_transpose_nt", ptr(dest), B, rec["F"], T, ptr(g), st)
        return g, None, None, None, None
    H, F = rec["H"], rec["F"]
    if form == "linear":
        lin: _Conv = rec["lin"]
        _, _, n_w2, n_b2 = need
        dest_t = _empty((B, T, F), dest)
        call("bm_transpose_nt", ptr(dest), B, F, T, ptr(dest_t), st)
        dw2 = db2 = g = None
        if n_w2 or n_b2:                              # the weight contraction on the side stream, in the ConvTranspose layout

            def lin_wgrad():
                dw, db = lin.backward_weight(dest_t, rec["x_last"], B, T, 1, dest, status, want_w=n_w2, want_b=n_b2)
                return (None if dw is None else dw.permute(1, 0, 2).contiguous()), db
            dw2, db2 = _on_side(side if n_w2 else None, keep_alive, lin_wgrad, dest_t, rec["x_last"])
        if rec["want_g"]:
            g = _empty((B, T, H), dest)
            lin.backward_data(dest_t, None, B, T, 1, g, status)
        return g, None, None, dw2, db2
    H2, rows = 2 * H, B * T
    n_w0, n_b0, n_w2, n_b2 = need
    want_g, want_dh1 = rec["want_g"], rec["want_dh1"]
    x_last, h1, q = rec["x_last"], rec["h1"], rec["q"]
    g = _empty((B, T, H), dest) if want_g else None
    dw0 = dw2 = db0 = db2 = None
    if form in ("tc_params", "fma"):                   # the fused kernels write the gradients asked of them
        dw0 = _empty((H2, H, 1), dest) if n_w0 else None
        db0 = _empty((H2,), dest) if n_b0 else None
        dw2 = _empty((H2, F, 1), dest) if n_w2 else None
        db2 = _empty((F,), dest) if n_b2 else None
    if form == "fma":
        dq = _empty((B, T, H2), dest) if want_dh1 else None
        _reducing_call("bm_head_bwd", dest, (B, T, H, F), ptr(dest), ptr(x_last), ptr(rec["w0_2"]), ptr(rec["w2_2"]),
                       ptr(h1), ptr(q), B, T, H, F, ptr(dq), ptr(g), ptr(dw0), ptr(db0), ptr(dw2), ptr(db2), st,
                       reduces=any(need))
        return g, dw0, db0, dw2, db2

    head0: _Conv = rec["head0"]
    head2: _Conv = rec["head2"]
    dest_t = _empty((B, T, F), dest)
    call("bm_transpose_nt", ptr(dest), B, F, T, ptr(dest_t), st)
    dq = None                                         # dL/dq, q = act(h1) the ConvTranspose's input
    if want_dh1 or (form == "tc_params" and (n_w2 or n_b2)):     # bm_head_bwd_params reads dq in any case
        dq = _empty((B, T, H2), dest)
        head2.backward_data(dest_t, None, B, T, 1, dq, status)
    # dW2 / db2, and dh1 = dL/dh1 (in place of dq where the activation backward allows it)
    dh1 = dq
    if form == "generic":
        dw2c, db2 = head2.backward_weight(dest_t, q, B, T, 1, dest, status, want_w=n_w2, want_b=n_b2)   # [F, 2H, 1]
        dw2 = None if dw2c is None else dw2c.permute(1, 0, 2).contiguous()
        if want_dh1:
            dh1 = _empty((B, T, H2), dest)
            call("bm_bn_act_skip_bwd", ptr(dq), ptr(h1), None, None, None, None, 0, rows, H2, plan.act_code,
                 float(plan.act_slope), None, ptr(dh1), None, None, st)
    elif form == "tc":
        if n_w2:    # in the ConvTranspose layout [2H, F, 1]; overlaps the dq contraction queued just before
            dw2 = _on_side(side, keep_alive, lambda: tc_wgrad(q, dest_t, B, T, H2, F, F, 1, 1, status), q, dest_t)
        if n_b2:
            db2 = _empty((F,), dest)
            col_sum(dest_t, rows, F, db2, st)
        if want_dh1:
            call("bm_gelu_bwd", ptr(dq), ptr(h1), rows * H2, ptr(dq), st)
    elif any(need):
        _reducing_call("bm_head_bwd_params", dest, (B, T, H, F), ptr(dest), ptr(x_last), ptr(h1), ptr(q), B, T, H, F,
                       ptr(dq), ptr(dw0), ptr(db0), ptr(dw2), ptr(db2), st)
    elif want_g:
        call("bm_gelu_bwd", ptr(dq), ptr(h1), rows * H2, ptr(dq), st)
    if form != "tc_params" and (n_w0 or n_b0):
        # on the side stream only the weight contraction (a lone bias sum stays on the main stream)
        dw0, db0 = _on_side(side if form == "tc" and n_w0 else None, keep_alive, lambda: head0.backward_weight(
            dh1, x_last, B, T, 1, dest, status, want_w=n_w0, want_b=n_b0), dh1, x_last)
    if want_g:
        head0.backward_data(dh1, None, B, T, 1, g, status)
    return g, dw0, db0, dw2, db2


@dataclasses.dataclass
class _Needs:
    """Which gradients a backward is asked for (`ctx.needs_input_grad`, fixed at forward time), stage by stage from the input.
    below[k]: the data gradient at the input of conv layer k is needed, i.e. `meg` or a parameter of an earlier stage
    requires grad (below[depth]: at the input of the head).  With several input streams `streams[i]` is the requires-grad
    of stream plan.streams[i] and `enc[j]` the needs of encoder plan.encoders[j] (its front: its stream)."""
    front: tp.Tuple[bool, ...]                 # meg, heads, il_w, il_b, subj_w, sub_emb
    head: tp.Tuple[bool, ...]                  # w0, b0, w2, b2
    layer: tp.List[tp.Tuple[bool, ...]]        # conv_w, conv_b, gamma, beta (+ rewrite_w, rewrite_b, scale, post_skip_w)
    glu: tp.Dict[int, tp.Tuple[bool, ...]]     # glu_w, glu_b of the GLU block after layer k
    below: tp.List[bool]
    streams: tp.Tuple[bool, ...] = ()
    enc: tp.List["_Needs"] = dataclasses.field(default_factory=list)

    @staticmethod
    def of(needs_input_grad, plan: "EncoderPlan") -> "_Needs":
        n = [bool(v) for v in needs_input_grad]
        front = tuple(n[1:6]) + ((n[-1],) if plan.has_sub_emb else (False,))
        layer, glu, at = _stack_needs(n, 10, plan)
        streams = tuple(n[at:at + len(plan.streams)])
        at += len(plan.streams)
        below = _below(any(front) or (plan.concatenate and any(streams)), layer, glu)
        enc = []
        for name, sp in plan.encoders:
            e_layer, e_glu, at = _stack_needs(n, at, sp)
            own = streams[plan.streams.index(name)]
            enc.append(_Needs(front=(own,), head=(), layer=e_layer, glu=e_glu, below=_below(own, e_layer, e_glu)))
        return _Needs(front=front, head=tuple(n[6:10]), layer=layer, glu=glu, below=below, streams=streams, enc=enc)

    def layer_up(self, k: int) -> bool:
        """the gradient at layer k's output (below its GLU block) is needed"""
        return self.below[k] or any(self.layer[k])


def _stack_needs(n, at, plan: SequencePlan):
    """(layer, glu, next position) of the requires-grad flags n[at:] of one encoder's layer parameters"""
    layer, glu = [], {}
    for k in range(len(plan.dilations)):
        layer.append(tuple(n[at:at + layer_width(plan, k)]))
        at += layer_width(plan, k)
    for k in range(len(plan.dilations)):
        if plan.glu_after[k]:
            glu[k] = tuple(n[at:at + 2])
            at += 2
    return layer, glu, at


def _below(first, layer, glu):
    below = [first]
    for k in range(len(layer)):
        below.append(below[-1] or any(layer[k]) or any(glu.get(k, ())))
    return below


def _stack_params(plan: SequencePlan, flat):
    """(conv_p, glu_p, rest) of one encoder's parameters at the front of `flat` (see `_EncoderFn`)"""
    conv_p, at = [], 0
    for k in range(len(plan.dilations)):
        conv_p.append(flat[at:at + layer_width(plan, k)])
        at += layer_width(plan, k)
    glu_p = {}
    for k in range(len(plan.dilations)):
        if plan.glu_after[k]:
            glu_p[k] = flat[at:at + 2]
            at += 2
    return conv_p, glu_p, flat[at:]


# ----------------------------------------------------------------------------------------------------
# Several input streams (simpleconv.py:234-243): `bm_channel_join` places channel-major raw streams and channels-last
# activations side by side in one channels-last tensor, `bm_channel_split` hands each column range's gradient back.
# ----------------------------------------------------------------------------------------------------
def _view_ptr(t):
    """Device pointer of a channel-major [B, C, T] view whose channel stride is >= T and sample stride C * stride(1)"""
    assert t.is_cuda, "brainmagick_b200 kernels need CUDA tensors (no CPU fallback)"
    return _lib.c_void_p(t.data_ptr())


def channel_major_operand(x):
    """(x or a contiguous copy, its channel stride) for `bm_channel_join` / `bm_channel_split`: a view cropped in time (the
    solver's offset crop) is read in place"""
    B, C, T = x.shape
    if x.is_contiguous():
        return x, T
    ld = x.stride(1)
    if x.stride(2) == 1 and ld >= T and (B == 1 or x.stride(0) == C * ld):
        return x, ld
    return x.contiguous(), T


def channel_join(parts, B, T, Cp, like):
    """parts [(tensor, C, cm, col)], cm: the tensor is channel-major [B, C, T] (else channels-last [B, T, C]) -> [B, T, Cp]
    channels-last, the parts in their columns and every other column zero"""
    out = _empty((B, T, Cp), like)
    args = []
    for t, C, cm, col in parts:
        if cm:
            t, ld = channel_major_operand(t)
            args += [ptr(t) if t.is_contiguous() else _view_ptr(t), C, ld, 1, col]
        else:
            args += [ptr(t), C, t.shape[2], 0, col]
    args += [None, 0, 0, 0, 0] * (4 - len(parts))
    call("bm_channel_join", B, T, Cp, len(parts), *args, ptr(out), stream())
    return out


def channel_split(g, parts):
    """g [B, T, Cp] -> the tensors of parts [(C, cm, col, wanted[, ld])]: [B, C, T] if cm else [B, T, ld] (ld default C,
    the columns past C zero), None where not wanted"""
    B, T, Cp = g.shape
    outs, args = [], []
    for C, cm, col, wanted, *rest in parts:
        ld = rest[0] if rest and not cm else (T if cm else C)
        o = None
        if wanted:
            o = _empty((B, C, T), g) if cm else \
                (torch.zeros((B, T, ld), device=g.device) if ld > C else _empty((B, T, C), g))
        outs.append(o)
        args += [ptr(o), C, ld, int(cm), col]
    args += [None, 0, 0, 0, 0] * (4 - len(parts))
    if any(o is not None for o in outs):
        call("bm_channel_split", ptr(g), B, T, Cp, len(parts), *args, stream())
    return outs


def stack_conv0(w0, T, width, tc, skip, want_bwd, fit_wgrad=False):
    """(layer 0's `_Conv`, Cp): its input zero-padded to Cp = a multiple of 64 channels when the tensor-core conv takes it
    (a layer 0 with a residual keeps the true width), as the stand-alone ConvSequence pads its input.  `fit_wgrad`: pad
    by up to two more 64-channel steps where that puts the layer's weight gradient on the tensor cores too (a joined
    width such as 390 -> 448 misses the weight-gradient gate, 512 passes it)."""
    if w0.shape[1] != width:
        raise ValueError(f"layer 0 takes {w0.shape[1]} input channels, the input has {width}")
    Cp = width if (skip and w0.shape[0] == width) else _round_up(width, 64)
    if fit_wgrad and tc and Cp != width:
        lib = _lib.load()
        for extra in (0, 64, 128):
            if lib.bm_tc_wgrad_supported(w0.shape[0], Cp + extra):
                Cp += extra
                break
    conv0 = _Conv(w0, T, False, tc, pad_cin_to=Cp, want_bwd=want_bwd)
    if not conv0.fwd_tc and Cp != width:
        Cp = width
        conv0 = _Conv(w0, T, False, False, want_bwd=want_bwd)
    return conv0, Cp


class _EncoderFn(torch.autograd.Function):
    """inputs: plan, meg, heads, il_w, il_b, subj_w, w0, b0, w2, b2, then per layer k of encoder 0: (conv_w, conv_b, gamma,
    beta) (+ (rewrite_w, rewrite_b, layer_scale, post_skip_w) on a layer with a residual-branch option, see `layer_width`)
    and, appended in layer order, (glu_w, glu_b) for every layer followed by a GLU block; then the input streams of
    plan.streams, then the layer parameters of each encoder of plan.encoders laid out like encoder 0's, then the [B, E]
    subject-embedding rows when plan.has_sub_emb.

    Encoder 0 reads the front's output ("meg"), or with plan.concatenate the join of the front's output and the raw streams
    in sorted key order ("concat"); every other encoder reads its raw stream.  With several encoders their outputs are
    joined in sorted key order before the head (simpleconv.py:234-243).

    Only what requires grad is backpropagated: a frozen parameter's gradient is not computed, the backward stops at the
    deepest stage that still needs a data gradient, and the forward saves only what those gradients read (nothing when no
    tensor argument requires grad: it then issues the calls of a `torch.no_grad()` forward)."""

    @staticmethod
    def forward(ctx, plan: EncoderPlan, meg, heads, il_w, il_b, subj_w, w0, b0, w2, b2, *params):
        ctx.bf16 = _lib.bf16()                   # the mode the backward replays
        sub_emb = None
        if plan.has_sub_emb:                     # [B, E] rows of the (scaled) subject embedding, appended by the caller
            sub_emb, params = params[-1], params[:-1]
        conv_p, glu_p, params = _stack_params(plan, params)
        xs, params = params[:len(plan.streams)], params[len(plan.streams):]
        enc_p = []
        for _, sp in plan.encoders:
            e_conv, e_glu, params = _stack_params(sp, params)
            enc_p.append((e_conv, e_glu))
        st = stream()
        meg = meg.contiguous()
        B, C, T = meg.shape
        if plan.channel_mask is not None:
            # inside the node, so that the gradient reaches the caller's unmasked tensor (the backward applies the mask)
            call("bm_channel_mask", ptr(meg), ptr(plan.channel_mask), B, C, T, ptr(plan.masked_meg), st)
            meg = plan.masked_meg
        nd = _Needs.of(ctx.needs_input_grad, plan)
        save = plan.keep_for_backward and any(ctx.needs_input_grad)
        status = tc_status_tensor(meg.device)

        x, conv0, front = front_forward(plan, meg, heads, il_w, il_b, subj_w, sub_emb,
                                        None if plan.concatenate else conv_p[0][0], nd, save, status)
        join_in = None
        if plan.concatenate:
            # "concat" reads the streams joined in sorted key order, zero-padded for layer 0 as a stand-alone input
            # the front's x keeps its tensor-core padding (rows of x.shape[2]); the join reads its valid columns
            widths = dict(zip(plan.streams, (t.shape[1] for t in xs)), meg=front["width"])
            cols, at = {}, 0
            for name in sorted(widths):
                cols[name] = at
                at += widths[name]
            conv0, Cp = stack_conv0(conv_p[0][0], T, at, plan.use_tensor_cores, plan.skip, save and nd.below[0],
                                    fit_wgrad=True)
            parts = [(x, widths["meg"], False, cols["meg"]) if name == "meg" else
                     (xs[plan.streams.index(name)], widths[name], True, cols[name]) for name in sorted(widths)]
            x = channel_join(parts, B, T, Cp, meg)
            join_in = (widths, cols, front["pad_width"])
        x, layers = conv_stack_forward(plan, x, conv0, conv_p, glu_p, nd, save, B, T, status, bare_slope=0.0)
        outs = {"concat" if plan.concatenate else "meg": x}
        enc_layers = []
        for (name, sp), (e_conv, e_glu), e_nd in zip(plan.encoders, enc_p, nd.enc):
            xi = xs[plan.streams.index(name)]
            c0, Cp = stack_conv0(e_conv[0][0], T, xi.shape[1], sp.use_tensor_cores, sp.skip, save and e_nd.below[0],
                                 fit_wgrad=True)
            x0 = channel_join([(xi, xi.shape[1], True, 0)], B, T, Cp, meg)
            outs[name], e_layers = conv_stack_forward(sp, x0, c0, e_conv, e_glu, e_nd, save, B, T, status, bare_slope=0.0)
            enc_layers.append((e_layers, Cp))
        want_top = nd.below[-1] or any(e.below[-1] for e in nd.enc)
        out_cols = None
        if len(outs) > 1:
            out_cols, at = {}, 0
            for name in sorted(outs):
                out_cols[name] = at
                at += outs[name].shape[2]
            x = channel_join([(outs[name], outs[name].shape[2], False, out_cols[name]) for name in sorted(outs)],
                             B, T, at, meg)
        est, head = head_forward(plan, x, w0, b0, w2, b2, nd, save, B, T, status, want_g=want_top)
        if save:
            ctx.plan, ctx.needs, ctx.dims = plan, nd, (B, T)
            ctx.saved = dict(front=front, layers=layers, conv_p=conv_p, head=head, params=(heads, il_w, subj_w, sub_emb),
                             enc=[(e_conv, e_layers, Cp) for (e_conv, _), (e_layers, Cp) in zip(enc_p, enc_layers)],
                             widths={k: v.shape[2] for k, v in outs.items()}, out_cols=out_cols, join_in=join_in,
                             stream_widths=[t.shape[1] for t in xs])
        return est

    @staticmethod
    @torch.autograd.function.once_differentiable
    @replays_bf16
    def backward(ctx, dest):
        plan: EncoderPlan = ctx.plan
        s = ctx.saved
        if s is None:
            raise RuntimeError("brainmagick_b200.SimpleConv: backward through the graph a second time -- the saved activations "
                               "(~5 GB at B=256) are released by the first backward; retain_graph is not supported")
        B, T = ctx.dims
        depth = len(plan.dilations)
        nd: _Needs = ctx.needs
        status = tc_status_tensor(dest.device)
        # The weight gradient and the data gradient of a layer are independent given dy: the tensor-core weight-gradient
        # kernels go to a side stream so that their CTAs fill the SMs left idle by the partial last wave of the
        # data-gradient kernel.  What they read stays in ctx_keep until the main stream has waited on them.
        side = _side_stream(dest.device) if (OVERLAP_WGRAD and plan.use_tensor_cores) else None
        ctx_keep: tp.List[tp.Any] = []
        g, *head_grads = head_backward(plan, s["head"], dest, nd.head, B, T, status, side, ctx_keep)
        name0 = "concat" if plan.concatenate else "meg"
        g_enc = dict([(name0, g)] + [(name, None) for name, _ in plan.encoders])
        if s["out_cols"] is not None and g is not None:     # the head's input gradient, split per encoder
            wanted = dict([(name0, nd.below[-1])] + [(name, e.below[-1]) for (name, _), e in zip(plan.encoders, nd.enc)])
            names = sorted(s["out_cols"])
            g_enc = dict(zip(names, channel_split(g, [(s["widths"][n], False, s["out_cols"][n], wanted[n]) for n in names])))
        layer_grads, glu_grads, g = conv_stack_backward(plan, s["conv_p"], s["layers"], g_enc[name0], nd, B, T, status,
                                                        side=side, keep_alive=ctx_keep)
        stream_grads = [None] * len(plan.streams)
        enc_grads = []
        for (name, sp), (e_conv, e_layers, Cp), e_nd in zip(plan.encoders, s["enc"], nd.enc):
            e_lg, e_gg, e_g = conv_stack_backward(sp, e_conv, e_layers, g_enc[name], e_nd, B, T, status, side=side,
                                                  keep_alive=ctx_keep)
            enc_grads.append((e_lg, e_gg))
            i = plan.streams.index(name)
            if nd.streams[i]:                            # inputs[name].grad, channel-major
                stream_grads[i] = channel_split(e_g, [(s["stream_widths"][i], True, 0, True)])[0]
        if ctx_keep:                                   # something ran on the side stream
            torch.cuda.current_stream().wait_stream(side)
        ctx_keep.clear()
        if s["join_in"] is not None and nd.below[0]:    # "concat": the layer-0 input gradient back to the front and streams
            widths, cols, meg_ld = s["join_in"]
            wanted = dict(zip(plan.streams, nd.streams), meg=any(nd.front))
            names = sorted(widths)
            parts = channel_split(g, [(widths[n], n != "meg", cols[n], wanted[n], meg_ld) for n in names])
            got = dict(zip(names, parts))
            g = got["meg"]
            stream_grads = [got[n] for n in plan.streams]
        dheads = d_il_w = d_il_b = d_subj = d_sub_emb = dmeg = None
        if any(nd.front):                              # else the sensor side is frozen and meg does not require grad
            dheads, d_il_w, d_il_b, d_subj, d_sub_emb, dmeg = front_backward(plan, s["front"], g, *s["params"], nd.front,
                                                                             status)
        grads = [None, dmeg, dheads, d_il_w, d_il_b, d_subj, *head_grads]
        _extend_stack_grads(grads, plan, layer_grads, glu_grads)
        grads.extend(stream_grads)
        for (_, sp), (e_lg, e_gg) in zip(plan.encoders, enc_grads):
            _extend_stack_grads(grads, sp, e_lg, e_gg)
        if plan.has_sub_emb:
            grads.append(d_sub_emb)
        ctx.saved = None
        return tuple(grads)


def _extend_stack_grads(grads, plan: SequencePlan, layer_grads, glu_grads):
    for k in range(len(plan.dilations)):
        grads.extend(layer_grads[k])
    for k in range(len(plan.dilations)):
        if plan.glu_after[k]:
            grads.extend(glu_grads[k])


def encoder_forward(plan: EncoderPlan, meg, heads, il_w, il_b, subj_w, w0, b0, w2, b2, layer_params, sub_emb=None,
                    streams=(), encoder_params=()):
    """`sub_emb` [B, E]: rows of the scaled subject embedding to append as channels (plan.has_sub_emb).  `streams`: the
    [B, C_s, T] tensors of plan.streams; `encoder_params`: the flat layer parameters of each encoder of plan.encoders."""
    extra = [] if sub_emb is None else [sub_emb]
    enc = [p for params in encoder_params for p in params]
    return _EncoderFn.apply(plan, meg, heads, il_w, il_b, subj_w, w0, b0, w2, b2, *layer_params, *streams, *enc, *extra)


# ----------------------------------------------------------------------------------------------------
# ClipLoss
# ----------------------------------------------------------------------------------------------------
_clip_ws: tp.Dict[torch.device, torch.Tensor] = {}


def _clip_workspace(like: torch.Tensor, Bn: int, Bc: int, KT: int) -> torch.Tensor:
    """Scratch of the CLIP score GEMM (split-K partial tiles, partial sums of squares, finalize ticket): one buffer per
    device, grown on demand to what the library asks for (`bm_clip_workspace`), handed to every call explicitly."""
    need = max(int(_lib.load().bm_clip_workspace(Bn, Bc, KT)), 2)
    dev = like.device
    ws = _clip_ws.get(dev)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, device=dev, dtype=torch.float32)
        _clip_ws[dev] = ws
    return ws


def _check_clip_operands(est: torch.Tensor, cand: torch.Tensor) -> None:
    if est.dtype != torch.float32 or cand.dtype != torch.float32:
        raise TypeError(f"ClipLoss kernels are fp32 (bm/losses.py computes in the input dtype; the reference trains in "
                        f"fp32): got {est.dtype} / {cand.dtype}")
    if est.device != cand.device:
        raise ValueError(f"estimate on {est.device}, candidate on {cand.device}")


def clip_scores(estimates: torch.Tensor, candidates: torch.Tensor, want_probs: bool = False):
    """ClipLoss.get_scores / get_probabilities (bm/losses.py:77-102) without autograd (evaluation, retrieval); see
    `clip_scores_grad` for the differentiable form."""
    est = estimates.detach().contiguous().float()
    cand = candidates.detach().contiguous().float()
    Bn, Bc = est.shape[0], cand.shape[0]
    KT = est[0].numel()
    assert cand[0].numel() == KT
    inv = _empty((Bc,), est)
    scores = _empty((Bn, Bc), est)
    probs = _empty((Bn, Bc), est) if want_probs else None
    ws = _clip_workspace(est, Bn, Bc, KT)
    _tc_call("bm_clip_scores", ptr(est), ptr(cand), Bn, Bc, KT, 0, ptr(inv), ptr(scores), ptr(probs), ptr(ws), ws.numel(),
             ptr(tc_status_tensor(est.device)), stream())
    return probs if want_probs else scores


class _ClipScoresFn(torch.autograd.Function):
    """get_scores / get_probabilities with a backward to the estimates and the candidates (gradient-based attribution).
    The forward is clip_scores' bm_clip_scores call, so the values are the same."""

    @staticmethod
    def forward(ctx, estimate, candidate, want_probs: bool):
        ctx.bf16 = _lib.bf16()                   # the mode the backward replays
        _check_clip_operands(estimate, candidate)
        est, cand = estimate.contiguous(), candidate.contiguous()
        Bn, Bc = est.shape[0], cand.shape[0]
        KT = est[0].numel()
        assert cand[0].numel() == KT
        inv = _empty((Bc,), est)
        scores = _empty((Bn, Bc), est)
        probs = _empty((Bn, Bc), est) if want_probs else None
        ws = _clip_workspace(est, Bn, Bc, KT)
        _tc_call("bm_clip_scores", ptr(est), ptr(cand), Bn, Bc, KT, 0, ptr(inv), ptr(scores), ptr(probs), ptr(ws),
                 ws.numel(), ptr(tc_status_tensor(est.device)), stream())
        ctx.save_for_backward(est, cand, inv, scores, probs)
        ctx.meta = (Bn, Bc, KT, estimate.shape, candidate.shape)
        return probs if want_probs else scores

    @staticmethod
    @torch.autograd.function.once_differentiable
    @replays_bf16
    def backward(ctx, gout):
        est, cand, inv, scores, probs = ctx.saved_tensors
        Bn, Bc, KT, est_shape, cand_shape = ctx.meta
        st = stream()
        dscores = gout.contiguous().float()
        if probs is not None:                    # get_probabilities: through the row softmax first
            ds = _empty((Bn, Bc), est)
            call("bm_softmax_bwd", ptr(probs), ptr(dscores), Bn, Bc, ptr(ds), st)
            dscores = ds
        dest = _empty(est_shape, est) if ctx.needs_input_grad[0] else None
        dcand = _empty(cand_shape, est) if ctx.needs_input_grad[1] else None
        G = _empty((Bn, Bc), est)
        coef = _empty((Bc,), est) if dcand is not None else None
        _tc_call("bm_clip_scores_bwd", ptr(dscores), ptr(scores), ptr(inv), ptr(est), ptr(cand), Bn, Bc, KT, ptr(G),
                 ptr(coef), ptr(dest), ptr(dcand), ptr(tc_status_tensor(est.device)), st)
        return dest, dcand, None


def clip_scores_grad(estimates: torch.Tensor, candidates: torch.Tensor, want_probs: bool = False):
    """clip_scores as an autograd node: scores (or probabilities) whose backward reaches the estimates and candidates."""
    return _ClipScoresFn.apply(estimates, candidates, want_probs)


def candidate_inv_norms(candidates: torch.Tensor) -> torch.Tensor:
    """inv_norm[o] = 1 / (1e-8 + ||candidate_o||) (bm/losses.py:91), for a candidate set that is scored many times."""
    cand = candidates.detach().contiguous().float()
    Bc, KT = cand.shape[0], cand[0].numel()
    ss = _empty((Bc,), cand, torch.float64)
    inv = _empty((Bc,), cand)
    _reducing_call("bm_candidate_inv_norms", cand, None, ptr(cand), Bc, KT, ptr(ss), ptr(inv), stream())
    return inv


def clip_scores_prenormed(estimates: torch.Tensor, candidates: torch.Tensor, inv_norms: torch.Tensor) -> torch.Tensor:
    """ClipLoss.get_scores against a candidate set whose `candidate_inv_norms` are already known (retrieval evaluation:
    the same candidates serve every query batch, so they are normed once)."""
    est = estimates.detach().contiguous().float()
    cand = candidates if (candidates.is_contiguous() and candidates.dtype == torch.float32) \
        else candidates.contiguous().float()
    Bn, Bc = est.shape[0], cand.shape[0]
    KT = est[0].numel()
    assert cand[0].numel() == KT and inv_norms.numel() == Bc
    scores = _empty((Bn, Bc), est)
    ws = _clip_workspace(est, Bn, Bc, KT)
    _tc_call("bm_clip_scores", ptr(est), ptr(cand), Bn, Bc, KT, 1, ptr(inv_norms), ptr(scores), None, ptr(ws), ws.numel(),
             ptr(tc_status_tensor(est.device)), stream())
    return scores


class _ClipLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, estimate, candidate, target_offset: int):
        ctx.bf16 = _lib.bf16()                   # the mode the backward replays
        _check_clip_operands(estimate, candidate)
        est = estimate.contiguous()
        cand = candidate.contiguous()
        Bn, Bc = est.shape[0], cand.shape[0]
        KT = est[0].numel()
        inv = _empty((Bc,), est)
        scores = _empty((Bn, Bc), est)
        probs = _empty((Bn, Bc), est)
        row_loss = _empty((Bn,), est)
        loss = _empty((1,), est)
        ws = _clip_workspace(est, Bn, Bc, KT)
        _tc_call("bm_clip_loss_fwd", ptr(est), ptr(cand), Bn, Bc, KT, int(target_offset), ptr(inv), ptr(scores),
                 ptr(probs), ptr(row_loss), ptr(loss), ptr(ws), ws.numel(), ptr(tc_status_tensor(est.device)), stream())
        if candidate.requires_grad:      # a trainable feature model produced the candidates (solver.py:304-320)
            ctx.save_for_backward(probs, inv, cand, scores, est)
        else:
            ctx.save_for_backward(probs, inv, cand)
        ctx.meta = (Bn, Bc, KT, int(target_offset), est.shape, cand.shape)
        return loss.reshape(())

    @staticmethod
    @torch.autograd.function.once_differentiable
    @replays_bf16
    def backward(ctx, gout):
        probs, inv, cand = ctx.saved_tensors[:3]
        Bn, Bc, KT, off, shape, cand_shape = ctx.meta
        gout = gout.reshape(1).contiguous().float()
        status = tc_status_tensor(probs.device)
        dest = dcand = None
        if ctx.needs_input_grad[0]:
            G = _empty((Bn, Bc), probs)
            dest = _empty(shape, probs)
            _tc_call("bm_clip_loss_bwd", ptr(probs), ptr(inv), ptr(cand), ptr(gout), Bn, Bc, KT, off, ptr(G), ptr(dest),
                     ptr(status), stream())
        if ctx.needs_input_grad[1]:
            scores, est = ctx.saved_tensors[3:]
            G = _empty((Bn, Bc), probs)
            coef = _empty((Bc,), probs)
            dcand = _empty(cand_shape, probs)
            _tc_call("bm_clip_loss_bwd_cand", ptr(probs), ptr(scores), ptr(inv), ptr(est), ptr(cand), ptr(gout), Bn, Bc,
                     KT, off, ptr(G), ptr(coef), ptr(dcand), ptr(status), stream())
        return dest, dcand, None


def clip_loss(estimate, candidate, target_offset: int = 0):
    return _ClipLossFn.apply(estimate, candidate, target_offset)


def clip_pooled_supported(KT: int) -> bool:
    """Whether the pooled CLIP entry points take rows of KT floats (the tensor-core forms' 16-byte row pitch)."""
    return KT >= 32 and KT % 4 == 0 and KT < (1 << 31)


class _ClipLossPooledFn(torch.autograd.Function):
    """ClipLoss.forward over a negatives.PooledCandidates: the candidates are read where they lie (the batch rows in
    place, the pool rows in the pool's device storage through the slot table).  The candidates carry no gradient, as in
    the reference, which builds them under no_grad.  The node keeps the PooledCandidates, and with it the lease on its
    slots, until its backward has run."""

    @staticmethod
    def forward(ctx, estimate, pooled):
        ctx.bf16 = _lib.bf16()                   # the mode the backward replays
        _check_clip_operands(estimate, pooled.batch)
        est = estimate.contiguous()
        Bn, Bc, Bb = est.shape[0], len(pooled), pooled.batch.shape[0]
        KT = est[0].numel()
        assert pooled.row_elems == KT, f"estimate rows of {KT} values, candidate rows of {pooled.row_elems}"
        inv = _empty((Bc,), est)
        scores = _empty((Bn, Bc), est)
        probs = _empty((Bn, Bc), est)
        row_loss = _empty((Bn,), est)
        loss = _empty((1,), est)
        ws = _clip_workspace(est, Bn, Bc, KT)
        _tc_call("bm_clip_loss_fwd_pooled", ptr(est), ptr(pooled.batch), Bb, ptr(pooled.storage), ptr(pooled.slots), Bn, Bc,
                 KT, 0, ptr(inv), ptr(scores), ptr(probs), ptr(row_loss), ptr(loss), ptr(ws), ws.numel(),
                 ptr(tc_status_tensor(est.device)), stream())
        ctx.save_for_backward(probs, inv)
        ctx.pooled = pooled
        ctx.meta = (Bn, Bc, Bb, KT, est.shape)
        return loss.reshape(())

    @staticmethod
    @torch.autograd.function.once_differentiable
    @replays_bf16
    def backward(ctx, gout):
        probs, inv = ctx.saved_tensors
        pooled, ctx.pooled = ctx.pooled, None    # the lease on the slots ends here
        Bn, Bc, Bb, KT, shape = ctx.meta
        gout = gout.reshape(1).contiguous().float()
        G = _empty((Bn, _round_up(Bc, 4)), probs)
        dest = _empty(shape, probs)
        _tc_call("bm_clip_loss_bwd_pooled", ptr(probs), ptr(inv), ptr(pooled.batch), Bb, ptr(pooled.storage),
                 ptr(pooled.slots), ptr(gout), Bn, Bc, KT, 0, ptr(G), ptr(dest), ptr(tc_status_tensor(probs.device)),
                 stream())
        return dest, None


def clip_loss_pooled(estimate, pooled):
    """ClipLoss.forward over a negatives.PooledCandidates (targets: the first Bn candidates); needs
    clip_pooled_supported(KT)."""
    return _ClipLossPooledFn.apply(estimate, pooled)


# ----------------------------------------------------------------------------------------------------
# L1Loss / L2Loss (bm/losses.py:11-26): torch's L1Loss / MSELoss over estimate[mask.expand_as(estimate)] and the same
# entries of output, without the boolean indexing: the kernels read the mask through its broadcast strides, so the True
# count never reaches the host, and the operands are read in place (the encode task's estimate[..., limit:] included).
# ----------------------------------------------------------------------------------------------------
MASKED_L1, MASKED_L2 = 0, 1      # `kind` of bm_masked_loss_fwd / _bwd


def _require_cuda_operands(*ts) -> None:
    if not all(t.is_cuda for t in ts):
        raise RuntimeError("brainmagick_b200 L1Loss / L2Loss run on CUDA (sm_90a) only; there is no CPU fallback: got "
                           f"{', '.join(str(t.device) for t in ts)}")


def _bct(t: torch.Tensor, unit_t: bool = True) -> torch.Tensor:
    """t as a [B, C, T] view (leading dimensions of size 1 added); `unit_t`: with t-stride 1, a copy only when the last
    dimension is not unit-stride (the mask keeps its broadcast strides)"""
    if t.dim() > 3:
        raise ValueError(f"brainmagick_b200 L1Loss / L2Loss take [B, C, T] operands, got {t.dim()} dimensions")
    while t.dim() < 3:
        t = t.unsqueeze(0)
    if unit_t and t.shape[2] > 1 and t.stride(2) != 1:
        t = t.contiguous()
    return t


def _strides(t: torch.Tensor):
    return [int(s) for s in t.stride()]


class _MaskedLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kind: int, estimate, output, mask):
        est, out, m = _bct(estimate), _bct(output), _bct(mask, unit_t=False)
        B, C, T = est.shape
        loss, inv_n = _empty((1,), est), _empty((1,), est)
        ws = _empty((max(int(_lib.load().bm_masked_loss_workspace(B, C, T)), 2),), est)
        call("bm_masked_loss_fwd", kind, _view_ptr(est), *_strides(est)[:2], _view_ptr(out), *_strides(out)[:2],
             _view_ptr(m), *_strides(m), B, C, T, ptr(ws), ws.numel(), ptr(loss), ptr(inv_n), stream())
        ctx.save_for_backward(est, out, m, inv_n)
        ctx.kind, ctx.shape = kind, estimate.shape
        return loss.reshape(())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        est, out, m, inv_n = ctx.saved_tensors
        B, C, T = est.shape
        want_est, want_out = ctx.needs_input_grad[1:3]
        d_est = _empty((B, C, T), est) if want_est else None
        d_out = _empty((B, C, T), est) if want_out else None
        if want_est or want_out:
            g = gout.reshape(1).contiguous().float()
            call("bm_masked_loss_bwd", ctx.kind, ptr(g), ptr(inv_n), _view_ptr(est), *_strides(est)[:2], _view_ptr(out),
                 *_strides(out)[:2], _view_ptr(m), *_strides(m), B, C, T, ptr(d_est), ptr(d_out), stream())
        return (None, None if d_est is None else d_est.view(ctx.shape),
                None if d_out is None else d_out.view(ctx.shape), None)


def masked_loss(kind: int, estimate: torch.Tensor, output: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """L1Loss (kind MASKED_L1) / L2Loss (MASKED_L2).forward: the mean of |e - o| or (e - o)^2 over the entries where
    `mask` (bool, broadcast to estimate's shape) is True; NaN when there is none.  fp32 CUDA operands."""
    if mask is None:
        raise TypeError("L1Loss / L2Loss need a bool mask that broadcasts to the estimate (bm/losses.py:13 expands it); "
                        "got None")
    _require_cuda_operands(estimate, output, mask)
    if estimate.dtype != torch.float32 or output.dtype != torch.float32:
        raise TypeError(f"L1Loss / L2Loss kernels are fp32 (the reference trains in fp32): got {estimate.dtype} / "
                        f"{output.dtype}")
    if mask.dtype != torch.bool:
        raise TypeError(f"L1Loss / L2Loss take a bool mask, got {mask.dtype}")
    if not (estimate.device == output.device == mask.device):
        raise RuntimeError(f"estimate on {estimate.device}, output on {output.device}, mask on {mask.device}")
    mask = mask.expand_as(estimate)          # RuntimeError when it does not broadcast, as in the reference
    if output.shape != estimate.shape:       # the reference's output[mask] raises IndexError
        raise IndexError(f"The shape of the mask {list(mask.shape)} does not match the shape of the indexed tensor "
                         f"{list(output.shape)}")
    return _MaskedLossFn.apply(kind, estimate, output, mask)


# ----------------------------------------------------------------------------------------------------
# FeatureDecodingLoss (bm/losses.py:117-173): per feature of the builder, F.mse_loss over the masked entries of a regression
# feature's channels or torch's weighted cross-entropy over the masked (b, t) of a categorical one, summed in feature order.
# One forward call (partials + finalize) and one backward call (every row of both gradients) whatever the features; the
# mask is never indexed on the host and the operands are read in place.  The feature table and the class weights are the
# module's (losses.FeatureDecodingLoss), built once per device.
# ----------------------------------------------------------------------------------------------------
DECODING_REGRESSION, DECODING_CATEGORICAL = 0, 1     # `kind` column of the bm_decoding_loss_* feature table
DECODING_TABLE_WIDTH = 6                             # (kind, est_start, width, out_start, weight_offset, lse_slot)
DECODING_MAX_FEATURES = 15                           # features of one loss: the flag word's bits


def _decoding_error(code: int, where: str) -> Exception:
    """The exception the reference raises for a bm_decoding_loss_fwd error code"""
    if code == DECODING_NO_MASK:
        return AssertionError(f"FeatureDecodingLoss: mask.any() is False, no entry is masked in ({where})")
    if code == DECODING_TARGET_TOO_LARGE:
        return AssertionError(f"FeatureDecodingLoss: output contains a category >= the feature's output_dim, or NaN ({where})")
    return IndexError(f"FeatureDecodingLoss: Target out of bounds: a masked class target is negative and not the "
                      f"ignore_index -100 ({where})")


def _require_cuda_decoding(*ts) -> None:
    if not all(t.is_cuda for t in ts):
        raise RuntimeError("brainmagick_b200 FeatureDecodingLoss runs on CUDA (sm_90a) only; there is no CPU fallback: got "
                           f"{', '.join(str(t.device) for t in ts)}")


def _mask_strides(m: torch.Tensor):
    """a [B, C, T] mask's strides, 0 along every dimension of size 1 (it broadcasts there)"""
    return [int(s) if n > 1 else 0 for s, n in zip(m.stride(), m.shape)]


class _DecodingLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, n_cat: int, weights, flag, estimate, output, mask):
        est, out = _bct(estimate), _bct(output)
        B, _, T = est.shape
        F = table.shape[0]
        lse = _empty((max(n_cat * B * T, 1),), est)
        loss, scale = _empty((1,), est), _empty((F,), est)
        ws = _empty((max(int(_lib.load().bm_decoding_loss_workspace(B, T, F)), 2),), est)
        status = tc_status_tensor(est.device)        # created eagerly: a captured step only writes it
        call("bm_decoding_loss_fwd", _view_ptr(est), *_strides(est)[:2], _view_ptr(out), *_strides(out)[:2], _view_ptr(mask),
             *_mask_strides(mask), B, T, ptr(table), F, ptr(weights), ptr(lse), ptr(ws), ws.numel(), ptr(loss), ptr(scale),
             ptr(flag), ptr(status) if capturing() else None, stream())
        ctx.save_for_backward(est, out, mask, table, weights, lse, scale)
        ctx.shapes = (estimate.shape, output.shape)
        return loss.reshape(())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        est, out, mask, table, weights, lse, scale = ctx.saved_tensors
        B, Ce, T = est.shape
        Co = out.shape[1]
        want_est, want_out = ctx.needs_input_grad[4:6]
        d_est = _empty((B, Ce, T), est) if want_est else None
        d_out = _empty((B, Co, T), est) if want_out else None
        if want_est or want_out:
            g = gout.reshape(1).contiguous().float()
            call("bm_decoding_loss_bwd", ptr(g), ptr(scale), ptr(lse), _view_ptr(est), *_strides(est)[:2], _view_ptr(out),
                 *_strides(out)[:2], _view_ptr(mask), *_mask_strides(mask), B, T, Ce, Co, ptr(table), table.shape[0],
                 ptr(weights), ptr(d_est), ptr(d_out), stream())
        return (None, None, None, None, None if d_est is None else d_est.view(ctx.shapes[0]),
                None if d_out is None else d_out.view(ctx.shapes[1]), None)


def decoding_loss(table: torch.Tensor, n_cat: int, weights: tp.Optional[torch.Tensor], estimate: torch.Tensor,
                  output: torch.Tensor, mask: torch.Tensor) -> tp.Tuple[torch.Tensor, torch.Tensor]:
    """FeatureDecodingLoss.forward on checked operands: `table` the int32 [F, DECODING_TABLE_WIDTH] feature table on the
    operands' device, `n_cat` its categorical features, `weights` the fp32 class weights its weight offsets index (None:
    unweighted), estimate [B, F_out, T] and output [B, F, T] fp32 with t-stride 1 where T > 1, mask bool [B, 1 or width, T]
    (broadcast views allowed).  -> (loss, flag): flag the int32 [1] word bm_decoding_loss_fwd writes (0: no error), which the
    caller reads in an eager step; a captured step gets the error code in the status word instead."""
    _require_cuda_decoding(estimate, output, mask)
    if estimate.dtype != torch.float32 or output.dtype != torch.float32:
        raise TypeError(f"FeatureDecodingLoss kernels are fp32 (the reference trains in fp32): got {estimate.dtype} / "
                        f"{output.dtype}")
    if mask.dtype != torch.bool:
        raise TypeError(f"FeatureDecodingLoss takes a bool mask, got {mask.dtype}")
    if not (estimate.device == output.device == mask.device):
        raise RuntimeError(f"estimate on {estimate.device}, output on {output.device}, mask on {mask.device}")
    flag = _empty((1,), estimate, torch.int32)
    return _DecodingLossFn.apply(table, n_cat, weights, flag, estimate, output, mask), flag


# ----------------------------------------------------------------------------------------------------
# Test metrics (bm/metrics.py): each update adds its per-column sums over dim 0 into fp64 accumulators on the device in one
# bm_metric_update call (one or two launches, set by the shape); get() is one bm_metric_finalize call and one flag word.
# The operands and the mask are read in place through their strides.  The metric objects are in metrics.py.
# ----------------------------------------------------------------------------------------------------
METRIC_CORRELATION, METRIC_L1, METRIC_L2, METRIC_ACCURACY = 0, 1, 2, 3
# bits of bm_metric_finalize's flag word
METRIC_LEFT_UNSTABLE, METRIC_LEFT_NAN, METRIC_RIGHT_UNSTABLE, METRIC_RIGHT_NAN, METRIC_RESULT_NAN, METRIC_COUNTED = \
    1, 2, 4, 8, 16, 32
_METRIC_DTYPES = {torch.float32: 0, torch.float64: 1}


def metric_planes(kind: int) -> int:
    """fp64 accumulator planes of a metric kind: (Σ l·r·m, Σ l·m, Σ r·m, Σ (l·m)², Σ (r·m)², count) or (sum, count)"""
    return 6 if kind == METRIC_CORRELATION else 2


def _require_cuda_metric(*ts) -> None:
    if not all(t.is_cuda for t in ts):
        raise RuntimeError("brainmagick_b200 test metrics run on CUDA (sm_90a) only; there is no CPU fallback: got "
                           f"{', '.join(str(t.device) for t in ts)}")


def _nct(t: torch.Tensor) -> torch.Tensor:
    """a [N, C, T] operand as it is, a [N, D] one as the view [N, D, 1]"""
    if t.dim() not in (2, 3):
        raise ValueError(f"brainmagick_b200 test metrics take [N, C, T] or [N, D] tensors, got {t.dim()} dimensions")
    return t if t.dim() == 3 else t.unsqueeze(-1)


def metric_operands(kind: int, left: torch.Tensor, right: torch.Tensor, mask: torch.Tensor) -> None:
    """Raises what the reference (or this port) raises for these sliced operands, before anything is allocated"""
    if left.is_complex() or right.is_complex():
        raise NotImplementedError("brainmagick_b200 test metrics take real operands (no CUDA model here is complex)")
    if mask.dtype != torch.bool:
        raise TypeError(f"brainmagick_b200 test metrics take a bool mask, got {mask.dtype}")
    _require_cuda_metric(left, right, mask)
    if left.dtype not in _METRIC_DTYPES or right.dtype != left.dtype:
        raise TypeError(f"brainmagick_b200 test metrics take fp32 or fp64 operands of one dtype, got {left.dtype} / "
                        f"{right.dtype}")
    if not (left.device == right.device == mask.device):
        raise RuntimeError(f"left on {left.device}, right on {right.device}, mask on {mask.device}")
    if not (left.dim() == right.dim() == mask.dim()) or left.dim() not in (2, 3):
        raise RuntimeError(f"the operands and the mask must all be [N, C, T] or all [N, D]: got {tuple(left.shape)}, "
                           f"{tuple(right.shape)}, {tuple(mask.shape)}")
    if kind == METRIC_ACCURACY:
        want = (left.shape[0], 1) + tuple(left.shape[2:])
        if tuple(mask.shape) != want or tuple(right.shape) != want:   # preds[~mask], expected[~mask] in the reference
            raise IndexError(f"ClassificationAcc takes targets and a mask of the predictions' shape {want}: got "
                             f"{tuple(right.shape)} and {tuple(mask.shape)}")
        if left.shape[1] == 0:
            raise IndexError("ClassificationAcc: argmax over zero class channels")
    else:
        if left.shape != right.shape:
            raise RuntimeError(f"left {tuple(left.shape)} and right {tuple(right.shape)} differ")
        if any(m not in (1, n) for m, n in zip(mask.shape, left.shape)):
            raise RuntimeError(f"the mask {tuple(mask.shape)} does not broadcast to {tuple(left.shape)}")


def metric_update(kind: int, left: torch.Tensor, right: torch.Tensor, mask: torch.Tensor, acc: torch.Tensor,
                  seen: torch.Tensor, parity: int) -> None:
    """One update of a metric's accumulators on operands metric_operands() accepted: `acc` fp64 [metric_planes(kind), cols]
    (cols = C*T, T for the accuracy), `seen` the int32 [2] ping-pong word read at `parity` (the caller flips it after the
    call).  Reads nothing on the host."""
    l, r, m = _nct(left), _nct(right), _nct(mask)
    N, C, T = l.shape
    K, C = (C, 1) if kind == METRIC_ACCURACY else (0, C)
    ws = _empty((max(int(_lib.load().bm_metric_workspace(N, C, T)), 2),), l)
    call("bm_metric_update", kind, _METRIC_DTYPES[l.dtype], _view_ptr(l), *_strides(l), _view_ptr(r), *_strides(r),
         _view_ptr(m), *_mask_strides(m), m.shape[0], N, C, T, K, ptr(acc), ptr(seen), parity, ptr(ws), ws.numel(),
         stream())


def metric_finalize(kind: int, acc: torch.Tensor, cols: int, tol: float, dtype: torch.dtype):
    """get() of a metric's accumulators -> (out [cols] in `dtype`, flag int32 [1] of METRIC_* bits), both on the device"""
    out = _empty((cols,), acc, dtype)
    flag = _empty((1,), acc, torch.int32)
    call("bm_metric_finalize", kind, ptr(acc), 1, cols, float(tol), ptr(out), _METRIC_DTYPES[dtype], ptr(flag), stream())
    return out, flag


# ----------------------------------------------------------------------------------------------------
# Spectral-norm penalty (bm/svd.py: svd_penalty): the estimate of every selected weight's top squared singular value by
# randomized subspace iteration, summed, in one bm_svd_penalty_fwd call (a fixed number of grouped launches whatever the
# number of weights) and its gradient in one bm_svd_penalty_bwd call.  The weights are read in place; the draws are torch's.
# The weight table is built on an eager call and kept per (weights, shapes, grad flags, q, niter, device), so a captured
# call copies nothing from the host.  A table is kept while its weights live: a graph captured with it reads it on every
# replay, so it is dropped only once its first weight is gone or has moved.  The drop-in function is in svd.py.
# ----------------------------------------------------------------------------------------------------
SVD_MAX_DIM = 32                      # largest projection dimension q of the kernels


class SvdPlan(tp.NamedTuple):
    table: torch.Tensor               # int64 [W, 12] on the weights' device (bm_svd_table)
    q: int
    niter: int
    ws_floats: int
    ws64_doubles: int
    r_offsets: tp.List[tp.Tuple[int, int]]     # per weight: (offset, rows) of its [rows, q] draw in the draw buffer
    r_floats: int
    g_offsets: tp.List[int]                    # per weight: offset of its gradient block, -1 when it gets none
    g_floats: int
    tiles: tp.Tuple[int, int, int]             # tiles_m, tiles_n, tiles_w


_svd_plans: tp.Dict[tuple, tp.Tuple[SvdPlan, "weakref.ref[torch.Tensor]"]] = {}    # key -> (plan, its first weight)


def _require_cuda_svd(weights) -> None:
    if not all(p.is_cuda for p in weights):
        raise RuntimeError("brainmagick_b200 svd_penalty runs on CUDA (sm_90a) only; there is no CPU fallback: got "
                           f"{', '.join(sorted({str(p.device) for p in weights}))}")


def svd_plan(weights: tp.Sequence[torch.Tensor], q: int, niter: int) -> SvdPlan:
    """The table and buffer sizes of these weights (contiguous fp32 on one device) at (q, niter): built once, on an eager
    call, then returned from the cache without touching the host."""
    key = (tuple((p.data_ptr(), tuple(p.shape), p.requires_grad) for p in weights), q, niter, weights[0].device)
    cached = _svd_plans.get(key)
    if cached is not None:
        return cached[0]
    if capturing():
        raise RuntimeError("svd_penalty: these weights' table is built on an eager call: run one eager step on this device "
                           "before capturing")
    for k in [k for k, (_, ref) in _svd_plans.items() if ref() is None or ref().data_ptr() != k[0][0][0]]:
        del _svd_plans[k]                                # tables of weights that are gone or have moved
    W = len(weights)
    ptrs = torch.tensor([p.data_ptr() for p in weights], dtype=torch.int64)
    rows = torch.tensor([p.shape[0] for p in weights], dtype=torch.int64)
    cols = torch.tensor([p.numel() // p.shape[0] for p in weights], dtype=torch.int64)
    grad = torch.tensor([int(p.requires_grad) for p in weights], dtype=torch.int32)
    table = torch.empty((W, 12), dtype=torch.int64)
    sizes = torch.empty((7,), dtype=torch.int64)
    lib = _lib.load()
    if lib.bm_svd_table(W, ptrs.data_ptr(), rows.data_ptr(), cols.data_ptr(), grad.data_ptr(), q, niter, table.data_ptr(),
                        sizes.data_ptr()) != 0:
        raise _lib.BmB200Error(f"bm_svd_table failed: {lib.bm_last_error().decode()}")
    ws, ws64, r, g, tm, tn, tw = (int(v) for v in sizes.tolist())
    t = table.tolist()
    plan = SvdPlan(table.to(weights[0].device), q, niter, max(ws, 2), max(ws64, 1),
                   [(row[7], min(row[1], row[2])) for row in t], r, [row[8] for row in t], g, (tm, tn, tw))
    _svd_plans[key] = (plan, weakref.ref(weights[0]))
    return plan


def svd_draws(plan: SvdPlan, like: torch.Tensor) -> torch.Tensor:
    """Every weight's draw R [min(m, n), q] from torch's generator, one normal_ per weight in weight order -- what
    torch.randn(min(m, n), q) inside each torch.svd_lowrank call draws -- into one fp32 buffer"""
    R = _empty((max(plan.r_floats, 1),), like)
    for off, n in plan.r_offsets:
        R[off:off + n * plan.q].view(n, plan.q).normal_()
    return R


class _SvdPenaltyFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, plan: SvdPlan, proba: float, R, *weights):
        ws = _empty((plan.ws_floats,), R)
        ws64 = _empty((plan.ws64_doubles,), R, torch.float64)
        out = _empty((1,), R)
        tm, tn, _ = plan.tiles
        call("bm_svd_penalty_fwd", ptr(plan.table), len(weights), plan.q, plan.niter, tm, tn, ptr(R), ptr(ws), ptr(ws64),
             float(proba), ptr(out), stream())
        ctx.save_for_backward(R, ws, ws64, *weights)
        ctx.plan, ctx.proba = plan, proba
        return out.reshape(())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        R, ws, ws64, *weights = ctx.saved_tensors
        plan = ctx.plan
        grad = _empty((max(plan.g_floats, 1),), R)
        g = gout.reshape(1).contiguous().float()
        call("bm_svd_penalty_bwd", ptr(plan.table), len(weights), plan.q, plan.niter, *plan.tiles, ptr(R), ptr(ws), ptr(ws64),
             ptr(g), float(ctx.proba), ptr(grad), stream())
        grads = [grad[off:off + p.numel()].view(p.shape) if off >= 0 and need else None
                 for p, off, need in zip(weights, plan.g_offsets, ctx.needs_input_grad[3:])]
        return (None, None, None, *grads)


def svd_penalty(weights: tp.Sequence[torch.Tensor], q: int, niter: int, proba: float) -> torch.Tensor:
    """Σ over `weights` of torch.svd_lowrank(p.view(p.shape[0], -1), q, niter)[1][0] ** 2, divided by proba, as a 0-dim fp32
    tensor on their device; differentiable in every weight that requires grad.  The weights are contiguous fp32 CUDA
    tensors on one device (checked by the caller).  The draws come from torch's CUDA generator, one per weight in order."""
    plan = svd_plan(weights, q, niter)
    R = svd_draws(plan, weights[0])
    return _SvdPenaltyFn.apply(plan, float(proba), R, *weights)


# ----------------------------------------------------------------------------------------------------
# Stand-alone ChannelMerger.forward / SubjectLayers.forward (bm/models/common.py:334-362, 55-58): inside SimpleConv both are
# fused into the encoder; called on their own (analysis notebooks, user code) they run the same stage kernels.  Channel-major
# tensors in and out, like the reference; gradients flow to the parameters and to the input (`meg` / `x`).
# ----------------------------------------------------------------------------------------------------
class _MergerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, meg, heads, positions, rec_of_sample, rec_order, rec_off, freq, ban_centre, radius: float):
        meg = meg.contiguous()
        B, C, T = meg.shape
        R = positions.shape[0]
        O, P = heads.shape
        st = stream()
        emb, att = _attention_fwd(heads, positions, freq, ban_centre, radius, C)
        u = _empty((B, T, O), meg)
        _mix_fwd(meg, att, rec_of_sample, u)
        out = _empty((B, O, T), meg)
        call("bm_transpose_nt", ptr(u), B, T, O, ptr(out), st)
        if any(ctx.needs_input_grad):                  # else nothing is kept: there will be no backward
            ctx.save_for_backward(meg, emb, att, rec_of_sample, rec_order, rec_off)
        ctx.dims = (B, C, T, R, O, P)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        meg, emb, att, rec_of_sample, rec_order, rec_off = ctx.saved_tensors
        B, C, T, R, O, P = ctx.dims
        st = stream()
        g = _empty((B, T, O), meg)
        call("bm_transpose_nt", ptr(gout.contiguous()), B, O, T, ptr(g), st)
        dheads = None
        if ctx.needs_input_grad[1]:                    # frozen heads: no mix or attention gradient
            dheads = _attention_bwd(_mix_bwd(g, meg, att, rec_order, rec_off), att, emb)
        dmeg = None
        if ctx.needs_input_grad[0]:
            dmeg = _mix_bwd_data(g, att, rec_of_sample, None)
        return dmeg, dheads, None, None, None, None, None, None, None


def channel_merger_forward(meg, heads, positions, rec_of_sample, rec_order, rec_off, freq, ban_centre, radius):
    return _MergerFn.apply(meg, heads, positions, rec_of_sample, rec_order, rec_off, freq, ban_centre, radius)


class _SubjectLayersFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weights, subject):
        x = x.contiguous()
        B, Cin, T = x.shape
        S, _, D = weights.shape
        st = stream()
        xl = _empty((B, T, Cin), x)
        call("bm_transpose_nt", ptr(x), B, Cin, T, ptr(xl), st)
        yl = _empty((B, T, D), x)
        w = weights.contiguous()
        _subject_fwd(xl, w, subject, yl)
        out = _empty((B, D, T), x)
        call("bm_transpose_nt", ptr(yl), B, T, D, ptr(out), st)
        if any(ctx.needs_input_grad):                  # else nothing is kept: there will be no backward
            # x for the weight gradient, the weights for the data gradient
            ctx.save_for_backward(xl if ctx.needs_input_grad[1] else None, w if ctx.needs_input_grad[0] else None, subject)
        ctx.dims = (B, Cin, T, S, D)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        xl, w, subject = ctx.saved_tensors
        B, Cin, T, S, D = ctx.dims
        want_dx, want_dw = ctx.needs_input_grad[:2]
        st = stream()
        g = _empty((B, T, D), gout)
        call("bm_transpose_nt", ptr(gout.contiguous()), B, D, T, ptr(g), st)
        dxl, dw = _subject_bwd(g, xl, w, subject, (S, Cin, D), Cin, want_dx, want_dw)
        dx = None
        if want_dx:
            dx = _empty((B, Cin, T), g)
            call("bm_transpose_nt", ptr(dxl), B, T, Cin, ptr(dx), st)
        return dx, dw, None


def subject_layers_forward(x, weights, subject):
    return _SubjectLayersFn.apply(x, weights, subject)


def library_loaded() -> bool:
    return _lib._lib is not None
