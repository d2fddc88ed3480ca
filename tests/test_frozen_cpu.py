"""Backpropagating only what requires grad, without a GPU.

For each freezing pattern (attribution, head-only, subject-layer adaptation, merger-only, frozen BatchNorm affine, frozen GLU
convs, half-frozen DeepMel, stand-alone ChannelMerger / SubjectLayers):
  * the C-ABI call stream (tests/abi_trace.py) has no weight-gradient work for a frozen parameter and no call below the
    deepest stage that needs a gradient;
  * the gradients of what stays trainable (and of meg) are bitwise those of the same step with everything trainable, on the
    emulator (tests/frozen_emulator.py), and match the verbatim-reference fixtures; frozen parameters keep `.grad` None;
  * a forward in grad mode with nothing requiring grad issues the calls of a `torch.no_grad()` forward and records no node.
Every case runs with and without torch.use_deterministic_algorithms."""
import pytest
import torch

import abi_trace
import frozen_emulator
import test_emulated_host_path as host_path
from conftest import GOLDEN_CASES, load_arrays, load_golden, rel_err

# entry points that compute a weight gradient (or its bias sum) and nothing else
WGRAD = {"bm_tc_wgrad", "bm_tc_wgrad_conv", "bm_tc_wgrad_conv_f16", "bm_conv1d_bwd_weight", "bm_col_sum", "bm_tc_wgrad_grouped",
         "bm_sensor_mix_bwd", "bm_attention_weights_bwd", "bm_softmax_bwd", "bm_head_bwd_params"}
SENSOR_BWD = {"bm_subject_layers_bwd", "bm_initial_linear_bwd", "bm_sensor_chain_bwd", "bm_sensor_mix_bwd",
              "bm_sensor_mix_bwd_data", "bm_tc_sensor_mix_bwd_data", "bm_attention_weights_bwd", "bm_softmax_bwd",
              "bm_tc_wgrad_grouped", "bm_tc_pointwise_sel"}
LAYER_BWD = {"bm_bn_gelu_skip_bwd", "bm_bn_act_skip_bwd", "bm_glu_bwd"}
PATTERNS = ["attribution", "head", "subject", "merger", "bn", "glu"]
ROWS = {"default": {}, "no_merger": dict(merger=False), "no_initial_linear": dict(initial_linear=0),
        "no_subject_layers": dict(subject_layers=False, subject_dim=64), "bare_last": dict(complex_out=False),
        "no_glu": dict(glu=0), "subsample": dict(subsample_meg_channels=5)}


@pytest.fixture(params=[False, True], ids=["default", "deterministic"])
def det(request):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(request.param)
    try:
        yield request.param
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _trainable(model, pattern):
    """name -> requires_grad under the freezing pattern (meg requires grad only for 'attribution')."""
    seq = model.encoders["meg"]
    last_conv = f"encoders.meg.sequence.{len(seq.sequence) - 1}.0."
    bn = {f"encoders.meg.sequence.{k}.1." for k in range(len(seq.sequence))}
    out = {}
    for name, _ in model.named_parameters():
        if pattern == "attribution":
            t = False
        elif pattern == "head":
            t = name.startswith("final.") if model.final is not None else name.startswith(last_conv)
        elif pattern == "subject":
            t = name == "subject_layers.weights"
        elif pattern == "merger":
            t = name == "merger.heads"
        elif pattern == "bn":
            t = not any(name.startswith(p) for p in bn)
        else:
            t = ".glus." not in name
        out[name] = t
    return out


def _step(cfg, row, pattern, T=None, record=False):
    """One ClipLoss step of SimpleConv at `cfg` (abi_trace.CONFIGS), recorded (record=True) or on the emulator ->
    (trace or None, {name: grad}, meg.grad, model)."""
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import synthetic
    B, C, T0, F, S, hidden, MC, IL, P = cfg
    T = T or T0
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(ROWS[row])
    res = {}

    def run():
        torch.manual_seed(0)
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).train(pattern != "attribution")
        if pattern is not None:
            trainable = _trainable(model, pattern)
            if pattern != "attribution" and not any(trainable.values()):
                pytest.skip(f"the {row} row has no parameter that the {pattern} pattern trains")
            for name, p in model.named_parameters():
                p.requires_grad_(trainable[name])
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T), torch.randn(B, F, T)
        meg.requires_grad_(pattern in (None, "attribution"))
        batch = synthetic.make_batch(meg.detach(), subj, synthetic.normalised_positions(S, C), subj)
        BF.clip_loss(model(dict(meg=meg), batch), cand, 0).backward()
        res.update(model=model, meg=meg)

    if record:
        trace = abi_trace.record(run)
    else:
        trace = None
        with frozen_emulator.emulated():
            run()
    model = res["model"]
    return trace, {n: p.grad for n, p in model.named_parameters()}, res["meg"].grad, model


def _backward_part(trace):
    """the calls after the forward (the ClipLoss forward is the forward's last call)"""
    names = [c[0] for c in trace]
    last = max(i for i, n in enumerate(names) if n.startswith("bm_clip_loss_fwd"))
    return trace[last + 1:]


@pytest.mark.parametrize("cfg", list(abi_trace.CONFIGS))
@pytest.mark.parametrize("row", list(ROWS))
@pytest.mark.parametrize("pattern", PATTERNS)
def test_call_stream_does_no_frozen_work(cfg, row, pattern, det):
    trace, _, _, model = _step(abi_trace.CONFIGS[cfg], row, pattern, record=True)
    bwd = _backward_part(trace)
    names = {c[0].removesuffix("_det") for c in bwd}
    full = {c[0].removesuffix("_det") for c in _backward_part(_step(abi_trace.CONFIGS[cfg], row, None, record=True)[0])}
    # bm_gelu_bwd: the head's GELU backward on its own where bm_head_bwd_params would also compute the frozen head's gradients
    assert names - {"bm_gelu_bwd"} <= full, sorted(names - full)
    if pattern == "attribution":
        assert not names & WGRAD, sorted(names & WGRAD)
        for c in bwd:                                   # eval BatchNorm / GLU backward: no reduction, no gradient pointer
            if c[0].removesuffix("_det") == "bm_bn_gelu_skip_bwd":
                assert c[10:14] == [False, True, False, False]        # sums, dy, dgamma, dbeta
            if c[0].removesuffix("_det") == "bm_bn_act_skip_bwd":
                assert c[12:16] == [False, True, False, False]
            if c[0].removesuffix("_det") == "bm_glu_bwd":
                assert c[6] is False                               # dbias
    elif pattern == "head":
        # complex_out=False: the GLU block after the bare last conv passes the gradient down to it
        forbidden = SENSOR_BWD | LAYER_BWD if model.final is not None else SENSOR_BWD | {"bm_bn_gelu_skip_bwd", "bm_bn_act_skip_bwd"}
        assert not names & forbidden, sorted(names & forbidden)
        assert len(bwd) < len(_backward_part(_step(abi_trace.CONFIGS[cfg], row, None, record=True)[0])) // 4
    elif pattern == "subject":
        if model.subject_layers is None:
            assert not names & SENSOR_BWD
        else:
            assert not names & {"bm_initial_linear_bwd", "bm_sensor_mix_bwd", "bm_sensor_mix_bwd_data", "bm_attention_weights_bwd",
                                "bm_softmax_bwd", "bm_tc_sensor_mix_bwd_data"}, sorted(names)
            for c in bwd:
                if c[0].removesuffix("_det") == "bm_sensor_chain_bwd":
                    assert c[21:27] == [False, False, True, False, False, False]   # dv du d_subj d_il_w d_il_b d_weights
                if c[0] == "bm_subject_layers_bwd":
                    assert c[15:17] == [False, True]                             # dv, d_subj_w
    elif pattern == "merger":
        assert not names & {"bm_sensor_mix_bwd_data", "bm_tc_sensor_mix_bwd_data"}
        if model.merger is None:
            assert not names & SENSOR_BWD
    # no non-NULL gradient pointer of a frozen parameter: the bias-gradient pointer of the GLU backward
    if pattern in ("glu", "attribution", "head", "subject", "merger"):
        assert all(c[6] is False for c in bwd if c[0].removesuffix("_det") == "bm_glu_bwd")


def _assert_same(grads, meg_grad, want_grads, want_meg, trainable, meg_wanted):
    for name, g in grads.items():
        if trainable[name]:
            assert g is not None and torch.equal(g, want_grads[name]), name
        else:
            assert g is None, name
    if meg_wanted:
        assert torch.equal(meg_grad, want_meg)


@pytest.mark.parametrize("cfg,T", [("small", None), ("mid", 40), ("full", 24)])
@pytest.mark.parametrize("row", list(ROWS))
@pytest.mark.parametrize("pattern", PATTERNS)
def test_gradients_bitwise_equal_full_backward(cfg, T, row, pattern, det):
    c = abi_trace.CONFIGS[cfg]
    _, grads, meg_grad, model = _step(c, row, pattern, T=T)
    # the reference point: the same step with everything trainable (for attribution: the same eval-mode step)
    _, full, full_meg, _ = _step(c, row, None, T=T) if pattern != "attribution" else _attribution_full(c, row, T)
    _assert_same(grads, meg_grad, full, full_meg, _trainable(model, pattern), pattern == "attribution")


def _attribution_full(cfg, row, T):
    """the attribution step (eval mode, meg requires grad) with every parameter trainable"""
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import synthetic
    B, C, T0, F, S, hidden, MC, IL, P = cfg
    T = T or T0
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(ROWS[row])
    with frozen_emulator.emulated():
        torch.manual_seed(0)
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).eval()
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T).requires_grad_(True), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg.detach(), subj, synthetic.normalised_positions(S, C), subj)
        BF.clip_loss(model(dict(meg=meg), batch), cand, 0).backward()
    return None, {n: p.grad for n, p in model.named_parameters()}, meg.grad, model


class _Trainable:
    """the trainable parameters of a model, for host_path._check_grads"""
    def __init__(self, model, trainable):
        self.params = [(n, p) for n, p in model.named_parameters() if trainable[n]]

    def named_parameters(self):
        return self.params


@pytest.mark.parametrize("name", GOLDEN_CASES[:2])
@pytest.mark.parametrize("pattern", ["head", "subject", "merger", "bn", "glu"])
def test_trainable_gradients_match_reference(name, pattern, det):
    """the default-configuration fixtures with part of the model frozen: what stays trainable still matches the reference"""
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
    trainable = _trainable(model, pattern)
    for n, p in model.named_parameters():
        p.requires_grad_(trainable[n])
    model.merger.ban_centre_override = t["ban_centre"]
    batch = synthetic.make_batch(t["meg"], t["subject_index"], t["rec_positions"], t["rec_of_sample"])
    with frozen_emulator.emulated():
        est = model(dict(meg=t["meg"]), batch)
        loss = bb.ClipLoss().train(train)(est, t["candidates"], torch.ones(len(t["meg"]), 1, t["meg"].shape[2], dtype=torch.bool))
        loss.backward()
    assert abs(loss.item() - t["loss"].item()) < 1e-5
    ref = {k[2:]: v.numpy() for k, v in t.items() if k.startswith("g.")}
    host_path._check_grads(_Trainable(model, trainable), ref)
    assert all(p.grad is None for n, p in model.named_parameters() if not trainable[n])
    sd = model.state_dict()                           # BatchNorm running statistics update whatever is frozen
    for key, v in t.items():
        if key.startswith("bn.") and "num_batches" not in key:
            assert rel_err(sd[key[3:]], v) < 2e-5, key
        elif key.startswith("bn."):
            assert int(sd[key[3:]]) == int(v)


@pytest.mark.parametrize("cfg", ["small", "full"])
@pytest.mark.parametrize("row", ["default", "no_merger", "no_subject_layers", "bare_last"])
def test_forward_with_nothing_requiring_grad_is_a_no_grad_forward(cfg, row, det):
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    B, C, T, F, S, hidden, MC, IL, P = abi_trace.CONFIGS[cfg]
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(ROWS[row])
    out = {}

    def run(grad_mode):
        def fn():
            torch.manual_seed(0)
            model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).train()
            model.requires_grad_(False)
            subj = torch.randint(0, S, (B,))
            meg = torch.randn(B, C, T)
            batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
            with torch.set_grad_enabled(grad_mode):
                out[grad_mode] = model(dict(meg=meg), batch)
        return abi_trace.record(fn)
    assert run(True) == run(False)
    assert out[True].grad_fn is None and not out[True].requires_grad


# ---------------------------------------------------------------- DeepMel, stand-alone ChannelMerger / SubjectLayers
def _deepmel_step(case, n_frozen):
    import brainmagick_b200 as bb
    from oracle.make_golden import DEEPMEL_CASES
    g = load_arrays(case)
    c = DEEPMEL_CASES[case]
    res = {}

    def run():
        model = bb.DeepMel(n_in_channels=c["n_in"], **c["params"])
        model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
        model.train()
        for k, blk in enumerate(model.sequence):
            if k < n_frozen:
                blk.requires_grad_(False)
                if model.glus[k] is not None:
                    model.glus[k].requires_grad_(False)
        mel = torch.from_numpy(g["mel"])
        est = torch.from_numpy(g["estimate"]).requires_grad_(True)
        cand = model(mel)
        loss = bb.ClipLoss()(est, cand, torch.ones(len(est), 1, est.shape[2], dtype=torch.bool))
        loss.backward()
        res.update(model=model, est=est, loss=loss.item())
    with frozen_emulator.emulated() as emu:
        run()
    res["calls"] = [n for n in emu.calls if not n.endswith("_workspace")]
    return res


def _deepmel_cases():
    from oracle.make_golden import DEEPMEL_CASES
    return list(DEEPMEL_CASES)


@pytest.mark.parametrize("case", _deepmel_cases())
def test_deepmel_first_half_frozen(case, det):
    import brainmagick_b200.convseq  # noqa: F401
    full = _deepmel_step(case, 0)
    depth = len(full["model"].sequence)
    half = _deepmel_step(case, depth // 2)
    assert half["loss"] == full["loss"]
    assert torch.equal(half["est"].grad, full["est"].grad)
    fp = dict(full["model"].named_parameters())
    g = load_arrays(case)
    for name, p in half["model"].named_parameters():
        frozen = any(name.startswith(f"{m}.{k}.") for m in ("sequence", "glus") for k in range(depth // 2))
        if frozen:
            assert p.grad is None, name
        else:
            assert p.grad is not None and torch.equal(p.grad, fp[name].grad), name
            want = torch.from_numpy(g["g." + name])
            if want.norm() > 1e-6:
                assert rel_err(p.grad, want) < 5e-5, name
    # the half-frozen backward stops at the first trainable layer: fewer calls, fewer weight gradients
    t_full = [n.removesuffix("_det") for n in full["calls"]]
    t_half = [n.removesuffix("_det") for n in half["calls"]]
    assert len(t_half) < len(t_full)
    assert sum(n in WGRAD for n in t_half) < sum(n in WGRAD for n in t_full)


def test_standalone_merger_and_subject_layers_frozen(det):
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    gen = torch.Generator().manual_seed(5)
    B, C, T, O, P, S, D = 6, 19, 40, 12, 32, 3, 10
    meg = torch.randn(B, C, T, generator=gen)
    subj = torch.tensor([0, 2, 1, 2, 0, 1])
    rec = torch.tensor([1, 0, 1, 1, 0, 0])
    pos = synthetic.normalised_positions(2, C, n_valid=(C, C - 3), seed=3)
    gout = torch.randn(B, D, T, generator=gen)
    res = {}
    for frozen in (False, True):
        torch.manual_seed(1)
        merger = bb.ChannelMerger(O, pos_dim=P, dropout=0.2).train()
        merger.ban_centre_override = torch.tensor([0.4, 0.6])
        layer = bb.SubjectLayers(O, D, S)
        merger.heads.requires_grad_(not frozen)
        layer.weights.requires_grad_(not frozen)
        m = meg.clone().requires_grad_(True)
        calls = []

        def run():
            layer(merger(m, synthetic.make_batch(meg, subj, pos, rec)), subj).backward(gout)
        with frozen_emulator.emulated() as emu:
            run()
            calls = list(emu.calls)
        res[frozen] = (m.grad, merger.heads.grad, layer.weights.grad, calls)
    assert torch.equal(res[True][0], res[False][0])
    assert res[True][1] is None and res[True][2] is None
    assert res[False][1] is not None and res[False][2] is not None
    assert "bm_sensor_mix_bwd" in res[False][3] and "bm_sensor_mix_bwd" not in res[True][3]
    assert not any(n.startswith("bm_attention_weights_bwd") for n in res[True][3])
