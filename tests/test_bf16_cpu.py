"""torch.autocast(dtype=torch.bfloat16) without a GPU: which entry points the host code reaches (tests/abi_trace.py), and
that the bf16 call stream computes the reference's numbers to bf16 accuracy (tests/bf16_emulator.py against the oracle).

Without CUDA, `torch.autocast("cuda", ...)` disables itself, so `_autocast` below sets the same thread-local state that
its __enter__ sets (enabled flag, dtype, nesting) and restores it; the recorder's tensors live on the CPU, where the CUDA
autocast state changes no torch op."""
import contextlib
import json
import os

import pytest
import torch

import abi_trace
import bf16_emulator
import test_deterministic_cpu as det_cpu
import test_tf32_cpu as tf32_cpu
from conftest import GOLDEN_DIR, rel_err

BF16_TOL = 3e-2          # relative Frobenius error of a bf16 step against the fp32 reference (bf16 keeps 8 significant bits)


@contextlib.contextmanager
def _autocast(dtype=torch.bfloat16, enabled=True):
    """The CUDA autocast state of `torch.autocast("cuda", dtype=dtype, enabled=enabled)`, set directly."""
    was_on, was_dtype = torch.is_autocast_enabled("cuda"), torch.get_autocast_dtype("cuda")
    torch.set_autocast_enabled("cuda", enabled)
    torch.set_autocast_dtype("cuda", dtype)
    torch.autocast_increment_nesting()
    try:
        yield
    finally:
        torch.autocast_decrement_nesting()
        torch.set_autocast_enabled("cuda", was_on)
        torch.set_autocast_dtype("cuda", was_dtype)


def _forms():
    from brainmagick_b200 import _lib
    return set(_lib.TF32_FORMS)


def _base(name):
    for suffix in ("_bf16", "_tf32"):
        if name.endswith(suffix):
            return name[:-len(suffix)]
    return name


def _tc_calls(trace):
    forms = _forms()
    return [c[0] for c in trace if _base(c[0]) in forms]


def _stripped(trace):
    return [[_base(c[0])] + c[1:] for c in trace]


def test_reader_follows_the_autocast_state():
    from brainmagick_b200 import _lib
    assert not _lib.bf16()
    with _autocast():
        assert _lib.bf16()
        with _autocast(enabled=False):
            assert not _lib.bf16()
        with _autocast(torch.float16):
            assert not _lib.bf16()
        assert _lib.bf16()
        with _lib.recorded_bf16(False):
            assert not _lib.bf16()
    assert not _lib.bf16()
    with _lib.recorded_bf16(True):
        assert _lib.bf16()
    assert not _lib.bf16()


@pytest.mark.parametrize("stream_name", list(tf32_cpu.STREAMS))
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_every_tensor_core_call_takes_its_bf16_form(stream_name, det):
    """Under bf16 autocast every tensor-core call is its `_bf16` form (with `_det` under the determinism flag where that
    exists) and the rest of the call stream -- FP32-FMA kernels, weight preparation, arguments, order -- is exactly the one
    issued without it."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        plain = tf32_cpu.STREAMS[stream_name]()
        with _autocast():
            bf = tf32_cpu.STREAMS[stream_name]()
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    tc = _tc_calls(bf)
    assert tc and all(n.endswith("_bf16") for n in tc), sorted(set(tc))
    assert _stripped(bf) == plain
    if det:
        assert det_cpu._atomic_calls(_stripped(bf)) == []
        if stream_name in ("full.train", "clip", "deepmel"):
            assert any(c[0] in ("bm_clip_loss_fwd_det_bf16", "bm_clip_scores_det_bf16") for c in bf)


@pytest.mark.parametrize("override", [{}, dict(glu=0), dict(skip=False), dict(merger=False), dict(initial_linear=0),
                                      dict(subject_layers=False, subject_dim=5), dict(subsample_meg_channels=150)],
                         ids=["default", "no_glu", "no_skip", "no_merger", "no_initial_linear", "subject_embedding",
                              "subsample"])
def test_ablation_rows_take_their_bf16_forms(override):
    plain = abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True, **override)
    with _autocast():
        bf = abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True, **override)
    tc = _tc_calls(bf)
    assert tc and all(n.endswith("_bf16") for n in tc), sorted(set(tc))
    assert _stripped(bf) == plain


def test_tf32_flag_does_not_override_bf16():
    with tf32_cpu._precision(tf32_cpu.SETTERS["matmul_fp32_precision"]):
        tf = abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True)
        with _autocast():
            bf = abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True)
    assert all(n.endswith("_tf32") for n in _tc_calls(tf))
    tc = _tc_calls(bf)
    assert tc and all(n.endswith("_bf16") for n in tc), sorted(set(tc))


def _forward_inside_backward_outside(kind):
    """A training step whose forward runs under bf16 autocast and whose backward runs after the context has closed, as in
    the usual `with autocast(): loss = ...` then `loss.backward()`."""
    import brainmagick_b200 as bb
    import brainmagick_b200.convseq as CS
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import synthetic

    def simpleconv():
        torch.manual_seed(0)
        B, C, T, F, S, hidden, MC, IL, P = abi_trace.CONFIGS["full"]
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, hidden=dict(meg=hidden), depth=10,
                              dilation_period=5, kernel_size=3, skip=True, subject_layers=True, subject_dim=0,
                              complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL,
                              merger_channels=MC, gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2,
                              n_subjects=S).train()
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T, requires_grad=True), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg.detach(), subj, synthetic.normalised_positions(S, C), subj)
        with _autocast():
            loss = BF.clip_loss(model(dict(meg=meg), batch), cand, 0)
        loss.backward()

    def deepmel():
        torch.manual_seed(3)
        model = bb.DeepMel(n_in_channels=120, n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3,
                           stride=1, dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False,
                           skip=True, glu_context=1, glu=2).train()
        mel, est = torch.randn(2, 120, 40), torch.randn(2, 768, 40, requires_grad=True)
        with _autocast():
            loss = bb.ClipLoss()(est, model(mel), torch.ones(2, 1, 40, dtype=torch.bool))
            scores = bb.ClipLoss().get_scores(est, model(mel))
        (loss + scores.sum()).backward()

    fn = dict(simpleconv=simpleconv, deepmel=deepmel)[kind]
    saved, CS._require_cuda = CS._require_cuda, lambda x: None      # the recorder's tensors live on the CPU
    try:
        return abi_trace.record(fn)
    finally:
        CS._require_cuda = saved


@pytest.mark.parametrize("kind", ["simpleconv", "deepmel"])
def test_backward_outside_autocast_replays_the_recorded_mode(kind):
    from brainmagick_b200 import _lib
    trace = _forward_inside_backward_outside(kind)
    assert not _lib.bf16()
    tc = _tc_calls(trace)
    assert tc and all(n.endswith("_bf16") for n in tc), sorted(set(tc))
    bwd = {"simpleconv": {"bm_tc_wgrad_conv_bf16", "bm_tc_wgrad_grouped_bf16", "bm_clip_loss_bwd_bf16"},
           "deepmel": {"bm_tc_wgrad_conv_bf16", "bm_clip_loss_bwd_bf16", "bm_clip_scores_bwd_bf16"}}[kind]
    assert bwd <= set(tc), sorted(set(tc))


@pytest.mark.parametrize("ctx", ["off", "fp16", "disabled_inside_bf16"])
def test_steps_outside_bf16_keep_their_recorded_call_streams(ctx):
    """Without autocast, under fp16 autocast and in an `autocast(enabled=False)` region nested in a bf16 one, every
    recorded step issues exactly its committed call stream."""
    want = json.load(open(os.path.join(GOLDEN_DIR, "abi_trace_steps.json")))
    region = {"off": contextlib.nullcontext, "fp16": lambda: _autocast(torch.float16),
              "disabled_inside_bf16": lambda: _nested(_autocast(), _autocast(enabled=False))}[ctx]
    with region():
        got = {tag: abi_trace.simpleconv_step(abi_trace.CONFIGS[tag.split(".")[0]], tag.split(".")[1] == "train")
               for tag in ("full.train", "full.eval", "mid.train", "small.train")}
    got = json.loads(json.dumps(got))
    for tag, calls in got.items():
        assert calls == want[tag], tag


@contextlib.contextmanager
def _nested(outer, inner):
    with outer, inner:
        yield


@pytest.mark.parametrize("train", [True, False])
def test_tensor_core_widths_match_oracle_in_bf16(train):
    """BASELINE widths (every contraction on a tensor-core entry point, so every one on its `_bf16` form), short in batch
    and time, on the bf16 emulator against the fp32 oracle."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
    shape = dict(B=3, C=208, T=48, F=1024, S=4, hidden=320, MC=270, IL=270, P=2048, n_valid=(208, 150, 208, 97))
    cfg = bm_oracle.Config(in_channels=shape["C"], out_channels=shape["F"], n_subjects=shape["S"], hidden=shape["hidden"],
                           merger_channels=shape["MC"], initial_linear=shape["IL"], merger_pos_dim=shape["P"])
    params = bm_oracle.init_state_dict(cfg, seed=11)
    d = bm_oracle.synthetic_batch(cfg, batch=shape["B"], T=shape["T"], seed=5, n_valid=shape["n_valid"])
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, shape["n_valid"], seed=3)
    ref = bm_oracle.training_step(params, cfg, d["meg"], d["rec_positions"], d["rec_of_sample"], d["subject_index"],
                                  d["candidates"], ban_centre=d["ban_centre"], training=train)
    model = bb.SimpleConv(
        in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden),
        depth=cfg.depth, dilation_period=cfg.dilation_period, kernel_size=cfg.kernel_size, skip=True, subject_layers=True,
        subject_dim=0, complex_out=True, glu=cfg.glu, glu_context=cfg.glu_context, merger=True,
        initial_linear=cfg.initial_linear, merger_channels=cfg.merger_channels, gelu=True, batch_norm=True,
        merger_pos_dim=cfg.merger_pos_dim, merger_dropout=cfg.merger_dropout, n_subjects=cfg.n_subjects)
    model.load_state_dict(params, strict=True)
    model.train(train)
    model.merger.ban_centre_override = d["ban_centre"]
    batch = synthetic.make_batch(d["meg"], d["subject_index"], d["rec_positions"], d["rec_of_sample"])
    meg = d["meg"].clone().requires_grad_(True)
    with bf16_emulator.emulated() as emu:
        with _autocast():
            est = model(dict(meg=meg), batch)
            loss = bb.ClipLoss().train(train)(est, d["candidates"], torch.ones(len(meg), 1, meg.shape[2],
                                                                                dtype=torch.bool))
        loss.backward()
    tc = [n for n in emu.calls if _base(n) in _forms()]
    assert tc and all(n.endswith("_bf16") for n in tc)
    assert {"bm_tc_conv1d_persistent_bf16", "bm_tc_wgrad_conv_bf16", "bm_tc_pointwise_sel_bf16",
            "bm_tc_wgrad_grouped_bf16", "bm_tc_sensor_mix_bwd_data_bf16"} <= set(tc)
    assert est.dtype == torch.float32
    e_est = rel_err(est.detach(), ref["estimate"])
    assert 1e-4 < e_est < BF16_TOL                      # bf16 rounding is visible, and bounded
    assert abs(loss.item() - ref["loss"].item()) < BF16_TOL * abs(ref["loss"].item())
    assert meg.grad is not None and torch.isfinite(meg.grad).all()
    for name, p in model.named_parameters():
        g = ref["grads"].get(name)
        if g is not None and p.grad is not None and g.norm() > 1e-3 * max(1.0, float(p.detach().norm())):
            assert rel_err(p.grad, g) < 0.25, name
