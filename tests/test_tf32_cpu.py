"""PyTorch's TF32 matmul precision without a GPU: which entry points the host code reaches (tests/abi_trace.py), and that the
TF32 call stream computes the reference's numbers to TF32 accuracy (tests/tf32_emulator.py against the verbatim-reference
fixtures and the oracle)."""
import contextlib

import pytest
import torch

import abi_trace
import test_deterministic_cpu as det_cpu
import test_emulated_host_path as host_path
import tf32_emulator
from conftest import GOLDEN_CASES, load_golden, rel_err

TF32_TOL = 5e-3          # relative Frobenius error of a TF32 step against the fp32 reference (tf32 keeps 11 significant bits)


def _tf32_forms():
    from brainmagick_b200 import _lib
    return set(_lib.TF32_FORMS)


@contextlib.contextmanager
def _precision(setter=None):
    """Runs the body with PyTorch's float32 matmul precision set by `setter` (None: left at its default), then restores both
    the legacy and the new form of the flag."""
    m = torch.backends.cuda.matmul
    saved_new, saved_legacy = m.fp32_precision, torch.get_float32_matmul_precision()
    try:
        if setter is not None:
            setter()
        yield
    finally:
        torch.set_float32_matmul_precision(saved_legacy)
        m.fp32_precision = saved_new


SETTERS = {
    "set_float32_matmul_precision_high": lambda: torch.set_float32_matmul_precision("high"),
    "set_float32_matmul_precision_medium": lambda: torch.set_float32_matmul_precision("medium"),
    "matmul_allow_tf32": lambda: setattr(torch.backends.cuda.matmul, "allow_tf32", True),
    "matmul_fp32_precision": lambda: setattr(torch.backends.cuda.matmul, "fp32_precision", "tf32"),
}


@pytest.fixture
def tf32():
    with _precision(SETTERS["matmul_fp32_precision"]):
        yield


def _base(name):
    return name[:-len("_tf32")] if name.endswith("_tf32") else name


def _tc_calls(trace):
    forms = _tf32_forms()
    return [c[0] for c in trace if _base(c[0]) in forms]


def _deepmel_step():
    """DeepMel at conf/feature_model/deep_mel.yaml's widths (every conv on the tensor cores), short in batch and time: a
    training step through ClipLoss with the candidate gradient, then an eval forward."""
    import brainmagick_b200 as bb
    import brainmagick_b200.convseq as CS

    def run():
        torch.manual_seed(3)
        model = bb.DeepMel(n_in_channels=120, n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3,
                           stride=1, dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False,
                           skip=True, glu_context=1, glu=2).train()
        B, T = 2, 40
        mel, est = torch.randn(B, 120, T), torch.randn(B, 768, T)
        bb.ClipLoss()(est, model(mel), torch.ones(B, 1, T, dtype=torch.bool)).backward()
        model.eval()
        with torch.no_grad():
            model(mel)
    saved, CS._require_cuda = CS._require_cuda, lambda x: None      # the recorder's tensors live on the CPU
    try:
        return abi_trace.record(run)
    finally:
        CS._require_cuda = saved


def _clip_stream():
    """ClipLoss on its own: loss with both gradients, get_scores / get_probabilities and their gradients, and retrieval-style
    scoring against pre-normed candidates."""
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF

    def run():
        torch.manual_seed(0)
        est, cand = torch.randn(6, 64, 40, requires_grad=True), torch.randn(9, 64, 40, requires_grad=True)
        clip = bb.ClipLoss()
        clip(est, cand[:6], torch.ones(6, 1, 40, dtype=torch.bool)).backward()
        clip.get_scores(est, cand).sum().backward()
        clip.get_probabilities(est, cand).sum().backward()
        BF.clip_loss(est, cand, 2).backward()
        inv = BF.candidate_inv_norms(cand.detach())
        BF.clip_scores_prenormed(est.detach(), cand.detach(), inv)
    return abi_trace.record(run)


STREAMS = {"full.train": lambda: abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True),
           "full.eval": lambda: abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], False),
           "mid.train": lambda: abi_trace.simpleconv_step(abi_trace.CONFIGS["mid"], True),
           "deepmel": _deepmel_step, "clip": _clip_stream}


@pytest.mark.parametrize("how", list(SETTERS))
def test_each_way_of_allowing_tf32_selects_the_tf32_forms(how):
    from brainmagick_b200 import _lib
    with _precision(SETTERS[how]):
        assert _lib.tf32()
        trace = abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True)
    assert not _lib.tf32()
    tc = _tc_calls(trace)
    assert tc and all(n.endswith("_tf32") for n in tc), sorted(set(tc))


def test_default_flag_issues_no_tf32_call():
    """The library's default precision is 3xTF32 whatever cuDNN's conv flag says: it defaults to "tf32" and is not read."""
    from brainmagick_b200 import _lib
    assert torch.backends.cudnn.conv.fp32_precision == "tf32"
    assert not _lib.tf32()
    for name, fn in STREAMS.items():
        trace = fn()
        assert _tc_calls(trace), name
        assert not any(c[0].endswith("_tf32") for c in trace), name


@pytest.mark.parametrize("stream_name", list(STREAMS))
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_every_tensor_core_call_takes_its_tf32_form(stream_name, det):
    """With the flag on, every tensor-core call is its `_tf32` form (with `_det` under the determinism flag where that exists)
    and the rest of the call stream -- FP32-FMA kernels, weight preparation, arguments, order -- is exactly the one issued
    without it."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        plain = STREAMS[stream_name]()
        with _precision(SETTERS["matmul_fp32_precision"]):
            tf = STREAMS[stream_name]()
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    tc = _tc_calls(tf)
    assert tc and all(n.endswith("_tf32") for n in tc), sorted(set(tc))
    assert [[_base(c[0])] + c[1:] for c in tf] == plain
    if det:
        assert det_cpu._atomic_calls([[_base(c[0])] + c[1:] for c in tf]) == []
        if stream_name in ("full.train", "clip", "deepmel"):
            assert any(c[0] in ("bm_clip_loss_fwd_det_tf32", "bm_clip_scores_det_tf32") for c in tf)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_simpleconv_clip_loss_match_reference_in_tf32(name, tf32):
    """The committed verbatim-reference fixtures on the TF32 emulator (their widths run the convs on FP32-FMA kernels, which
    TF32 leaves exact; ClipLoss runs on its `_tf32` forms)."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    cfg, train, t = load_golden(name)
    model = bb.SimpleConv(
        in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden),
        depth=cfg.depth, dilation_period=cfg.dilation_period, kernel_size=cfg.kernel_size, skip=True,
        subject_layers=True, subject_dim=0, complex_out=True, glu=cfg.glu, glu_context=cfg.glu_context, merger=True,
        initial_linear=cfg.initial_linear, merger_channels=cfg.merger_channels, gelu=True, batch_norm=True,
        merger_pos_dim=cfg.merger_pos_dim, merger_dropout=cfg.merger_dropout, n_subjects=cfg.n_subjects)
    model.load_state_dict({k[2:]: v for k, v in t.items() if k.startswith("p.")}, strict=True)
    model.train(train)
    model.merger.ban_centre_override = t["ban_centre"]
    batch = synthetic.make_batch(t["meg"], t["subject_index"], t["rec_positions"], t["rec_of_sample"])
    clip = bb.ClipLoss().train(train)
    with tf32_emulator.emulated() as emu:
        est = model(dict(meg=t["meg"]), batch)
        loss = clip(est, t["candidates"], torch.ones(len(t["meg"]), 1, t["meg"].shape[2], dtype=torch.bool))
        loss.backward()
        probs = clip.get_probabilities(est.detach(), t["candidates"])
    assert "bm_clip_loss_fwd_tf32" in emu.calls and "bm_clip_loss_bwd_tf32" in emu.calls
    assert rel_err(est.detach(), t["estimate"]) < 2e-5              # the FP32-FMA convs: exact as before
    assert abs(loss.item() - t["loss"].item()) < TF32_TOL * abs(t["loss"].item())
    assert rel_err(probs, t["probs"]) < TF32_TOL
    host_path._check_grads(model, {k[2:]: v.numpy() for k, v in t.items() if k.startswith("g.")}, tol=2 * TF32_TOL)


@pytest.mark.parametrize("train", [True, False])
def test_tensor_core_widths_match_oracle_in_tf32(train, tf32):
    """BASELINE widths (every contraction on a tensor-core entry point, so every one on its `_tf32` form), short in batch and
    time, on the TF32 emulator against the fp32 oracle."""
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
    with tf32_emulator.emulated() as emu:
        est = model(dict(meg=meg), batch)
        loss = bb.ClipLoss().train(train)(est, d["candidates"], torch.ones(len(meg), 1, meg.shape[2], dtype=torch.bool))
        loss.backward()
    tc = [n for n in emu.calls if _base(n) in _tf32_forms()]
    assert tc and all(n.endswith("_tf32") for n in tc)
    assert {"bm_tc_conv1d_persistent_tf32", "bm_tc_wgrad_conv_tf32", "bm_tc_pointwise_sel_tf32",
            "bm_tc_wgrad_grouped_tf32", "bm_tc_sensor_mix_bwd_data_tf32"} <= set(tc)
    e_est = rel_err(est.detach(), ref["estimate"])
    assert 1e-6 < e_est < TF32_TOL                      # TF32 rounding is visible, and bounded
    assert abs(loss.item() - ref["loss"].item()) < TF32_TOL * abs(ref["loss"].item())
    # 0.4 % for most parameters; up to 4.2 % for the head's first weight in eval mode, whose gradient is ~1e-6
    host_path._check_grads(model, {k: v.numpy() for k, v in ref["grads"].items()}, tol=0.06)
    assert meg.grad is not None and torch.isfinite(meg.grad).all()


def test_deepmel_tensor_core_widths_in_tf32(tf32):
    """The stand-alone ConvSequence (DeepMel) at its real widths and the candidate-side ClipLoss gradient, on the TF32
    emulator against the oracle."""
    import brainmagick_b200 as bb
    from oracle import bm_oracle, deepmel_oracle
    kw = dict(n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3, stride=1, dilation_growth=2,
              dilation_period=5, batch_norm=True, activation_on_last=False, skip=True, glu_context=1, glu=2)
    torch.manual_seed(3)
    model = bb.DeepMel(n_in_channels=120, **kw).train()
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    okw = {k: v for k, v in kw.items() if k not in ("stride", "n_hidden_channels", "n_hidden_layers", "n_out_channels")}
    spec = deepmel_oracle.deep_mel_spec(120, 320, 10, 768, activation="lrelu", **okw)
    B, T = 3, 40
    mel, est = torch.randn(B, 120, T), torch.randn(B, 768, T)
    p = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in params.items()}
    e_ref = est.clone().requires_grad_(True)
    cand_ref = deepmel_oracle.conv_sequence(mel.clone(), p, spec, training=True)
    loss_ref = bm_oracle.clip_loss(e_ref, cand_ref)
    loss_ref.backward()
    e = est.clone().requires_grad_(True)
    with tf32_emulator.emulated() as emu:
        cand = model(mel.clone())
        loss = bb.ClipLoss()(e, cand, torch.ones(B, 1, T, dtype=torch.bool))
        loss.backward()
    assert "bm_tc_conv1d_persistent_tf32" in emu.calls and "bm_clip_loss_bwd_cand_tf32" in emu.calls
    assert rel_err(cand.detach(), cand_ref.detach()) < TF32_TOL
    assert abs(loss.item() - loss_ref.item()) < TF32_TOL * abs(loss_ref.item())
    assert rel_err(e.grad, e_ref.grad) < TF32_TOL
    # 10 BatchNorm layers over only B * T = 120 rows: their backward removes most of the gradient (its row mean and its
    # projection on the normalised activations), so the TF32 rounding of the forward leaves the parameter gradients 6-7 %
    # off the fp32 oracle at this size
    host_path._check_grads(model, {k: v.grad.numpy() for k, v in p.items() if v.grad is not None}, tol=0.1)
