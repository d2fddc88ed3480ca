"""CPU checks of CUDA graph capture support: `StaticBatch.fill_` against `PositionGetter.batch_layout` and its padding rule,
its refusals, SimpleConv on a StaticBatch against the verbatim-reference fixtures on the ABI emulator, the call stream of a
StaticBatch step against a reference batch's, ClipLoss's mask check on the device while capturing, and the clear errors of
what a capture cannot hold.  The capture itself is simulated by patching `functional.capturing`."""
import contextlib

import pytest
import torch

import abi_emulator
import abi_trace
import frozen_emulator
from conftest import GOLDEN_CASES, load_arrays, load_golden, rel_err
from graph_emulator import CheckAllTrue

TOL = 2e-5


class _Emulator(CheckAllTrue, frozen_emulator.FrozenEmulator):
    """bm_check_all_true on top of the emulator of the training step"""


@contextlib.contextmanager
def capturing(monkeypatch):
    import brainmagick_b200.functional as BF
    with monkeypatch.context() as m:
        m.setattr(BF, "capturing", lambda: True)
        yield


def _recordings_batch(subjects, rec_of_sample, n_rec=5, C=9, T=6, seed=4):
    from brainmagick_b200 import synthetic
    pos = synthetic.normalised_positions(n_rec, C, (9, 5, 7), seed=seed)
    meg = torch.zeros(len(rec_of_sample), C, T)
    return synthetic.make_batch(meg, torch.tensor(subjects), pos, torch.tensor(rec_of_sample))


def _check_padded_layout(sb, batch):
    from brainmagick_b200.common import PositionGetter
    table, rows, order, off = PositionGetter().batch_layout(batch, sb.n_channels, "cpu")
    R, B = table.shape[0], sb.batch_size
    assert torch.equal(sb.rec_positions[:R], table)
    assert torch.equal(sb.rec_positions[R:], table[:1].expand(sb.max_recordings - R, -1, -1))
    assert torch.equal(sb.rec_of_sample, rows) and torch.equal(sb.rec_order, order)
    assert torch.equal(sb.rec_off[:R + 1], off)
    assert (sb.rec_off[R + 1:] == B).all()
    assert sb.subject_index.dtype == torch.int32
    assert torch.equal(sb.subject_index.long(), batch.subject_index)


def test_fill_gives_the_reference_layout_padded_with_slot_0():
    import brainmagick_b200 as bb
    sb = bb.StaticBatch(7, 9, 6, "cpu")
    first = _recordings_batch([2, 0, 1, 2, 0, 1, 1], [4, 0, 2, 4, 0, 2, 2])
    _check_padded_layout(sb.fill_(first), first)
    # a refill with fewer recordings re-pads every slot it no longer uses
    second = _recordings_batch([1] * 7, [3] * 7)
    _check_padded_layout(sb.fill_(second), second)
    assert sb.rec_off.tolist() == [0] + [7] * 6
    # exactly max_recordings recordings: no padding
    full = _recordings_batch([0, 1, 2, 3, 4, 0, 1], [0, 1, 2, 3, 4, 0, 1], n_rec=6)
    _check_padded_layout(bb.StaticBatch(7, 9, 5, "cpu").fill_(full), full)


def test_fill_refuses_other_shapes_and_a_capture(monkeypatch):
    import brainmagick_b200 as bb
    sb = bb.StaticBatch(4, 9, 2, "cpu")
    with pytest.raises(ValueError, match="3 distinct recordings"):
        sb.fill_(_recordings_batch([0, 1, 2, 0], [0, 1, 2, 0]))
    with pytest.raises(ValueError, match="batch_size"):
        sb.fill_(_recordings_batch([0, 1, 0], [0, 1, 0]))
    with pytest.raises(ValueError, match="n_channels"):
        sb.fill_(_recordings_batch([0, 1, 0, 1], [0, 1, 0, 1], C=8))
    ok = _recordings_batch([0, 1, 0, 1], [0, 1, 0, 1])
    with capturing(monkeypatch), pytest.raises(RuntimeError, match="capture"):
        sb.fill_(ok)
    sb.fill_(ok)
    with pytest.raises(ValueError, match="StaticBatch"):
        sb.check(torch.zeros(4, 8, 3))
    with pytest.raises(ValueError):
        bb.StaticBatch(4, 9, 0, "cpu")


def _static(batch, meg, extra=3):
    """A StaticBatch with R + extra recording slots, filled from `batch`"""
    import brainmagick_b200 as bb
    R = len({r.recording_index for r in batch._recordings})
    return bb.StaticBatch(meg.shape[0], meg.shape[1], R + extra, meg.device).fill_(batch)


def _check_grads(model, ref, tol=5e-5):
    """as tests/test_emulated_host_path.py holds the reference batch's gradients: gradients that are rounding noise around
    zero (a conv bias in front of a training-mode BatchNorm) only to an absolute bound"""
    scale = max(float(torch.as_tensor(v).norm()) for k, v in ref.items() if k.endswith("weight") and v.size)
    for name, p in model.named_parameters():
        want = torch.as_tensor(ref[name])
        if want.numel() == 0:
            continue
        if want.norm() < 1e-5 * scale:
            assert p.grad.abs().max().item() < 1e-4 * scale + 1e-6, name
        else:
            assert rel_err(p.grad, want) < tol, (name, rel_err(p.grad, want))


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_static_batch_reproduces_the_default_configuration_fixtures(name):
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
    sb = _static(synthetic.make_batch(t["meg"], t["subject_index"], t["rec_positions"], t["rec_of_sample"]), t["meg"])
    clip = bb.ClipLoss().train(train)
    with abi_emulator.emulated():
        est = model(dict(meg=t["meg"]), sb)
        loss = clip(est, t["candidates"], torch.ones(len(t["meg"]), 1, t["meg"].shape[2], dtype=torch.bool))
        loss.backward()
    assert rel_err(est.detach(), t["estimate"]) < TOL
    assert abs(loss.item() - t["loss"].item()) < 1e-5
    _check_grads(model, {k[2:]: v.numpy() for k, v in t.items() if k.startswith("g.")})


@pytest.mark.parametrize("name", ["ablation_reference", "ablation_no_merger", "ablation_subject_embedding",
                                  "ablation_subsample_channels"])
def test_static_batch_reproduces_the_ablation_fixtures(name):
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle.make_golden import ABLATION_BASE as c, ABLATIONS
    from oracle.ref_loader import clip_conv_kwargs
    g = load_arrays(name)
    kw = clip_conv_kwargs(hidden=c["hidden"], depth=c["depth"], merger_channels=c["MC"], initial_linear=c["IL"],
                          merger_pos_dim=c["P"])
    kw.update(ABLATIONS[name])
    model = bb.SimpleConv(in_channels=dict(meg=c["C"]), out_channels=c["F"], n_subjects=c["S"], **kw)
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
    model.train()
    if model.merger is not None:
        model.merger.ban_centre_override = torch.from_numpy(g["ban_centre"])
    meg, subj = torch.from_numpy(g["meg"]), torch.from_numpy(g["subject_index"])
    sb = _static(synthetic.make_batch(meg, subj, torch.from_numpy(g["rec_positions"]), subj), meg)
    with abi_emulator.emulated():
        est = model(dict(meg=meg), sb)
        loss = bb.ClipLoss()(est, torch.from_numpy(g["candidates"]), torch.ones(len(meg), 1, meg.shape[2], dtype=torch.bool))
        loss.backward()
    assert rel_err(est.detach(), torch.from_numpy(g["estimate"])) < TOL
    assert abs(loss.item() - float(g["loss"])) < 1e-5
    _check_grads(model, {k[2:]: v for k, v in g.items() if k.startswith("g.")})


def _step_trace(cfg, train, extra, capture=None, **overrides):
    """abi_trace.simpleconv_step with the batch given as a StaticBatch of R + extra slots (extra None: the reference batch);
    capture: a pytest monkeypatch to run the step under a simulated capture"""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    B, C, T, F, S, hidden, MC, IL, P = cfg
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(overrides)
    box = {}

    def run():
        torch.manual_seed(0)
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).train(train)
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
        box["R"] = len(set(subj.tolist()))
        if extra is not None:
            batch = _static(batch, meg, extra)
        with (capturing(capture) if capture is not None else contextlib.nullcontext()):
            if train:
                bb.ClipLoss()(model(dict(meg=meg), batch), cand, torch.ones(B, 1, T, dtype=torch.bool)).backward()
            else:
                with torch.no_grad():
                    model(dict(meg=meg), batch)
    return abi_trace.record(run), box["R"]


def _same_apart_from_R(ref, got, R, R_max):
    """Every call equal, except integer arguments that scale with the number of recording slots (k*R -> k*R_max)."""
    assert [c[0] for c in ref] == [c[0] for c in got]
    n_diff = 0
    for a, b in zip(ref, got):
        for x, y in zip(a[1:], b[1:]):
            if x != y:
                assert isinstance(x, int) and x % R == 0 and x // R * R_max == y, (a, b)
                n_diff += 1
    return n_diff


@pytest.mark.parametrize("tag", ["small", "full"])
@pytest.mark.parametrize("train", [True, False])
def test_static_batch_call_stream_equals_the_reference_batch_apart_from_R(tag, train):
    ref, R = _step_trace(abi_trace.CONFIGS[tag], train, None)
    got, _ = _step_trace(abi_trace.CONFIGS[tag], train, 3)
    assert _same_apart_from_R(ref, got, R, R + 3) > 0


@pytest.mark.parametrize("override", [dict(merger=False), dict(subject_layers=False, subject_dim=5),
                                      dict(subsample_meg_channels=6)])
def test_static_batch_call_stream_of_the_ablation_rows(override):
    ref, R = _step_trace(abi_trace.CONFIGS["small"], True, None, **override)
    got, _ = _step_trace(abi_trace.CONFIGS["small"], True, 3, **override)
    n_diff = _same_apart_from_R(ref, got, R, R + 3)
    if "merger" in override:
        assert n_diff == 0


def test_captured_step_checks_the_mask_on_the_device(monkeypatch):
    """Under a capture a StaticBatch step runs, and ClipLoss enqueues bm_check_all_true instead of reading the mask."""
    import brainmagick_b200.functional as BF
    eager, R = _step_trace(abi_trace.CONFIGS["small"], True, 3)
    captured, _ = _step_trace(abi_trace.CONFIGS["small"], True, 3, capture=monkeypatch)
    B, _, T = abi_trace.CONFIGS["small"][:3]
    checks = [c for c in captured if c[0] == "bm_check_all_true"]
    assert checks == [["bm_check_all_true", True, B * T, BF.MASK_NOT_ALL_TRUE, True, True]]
    assert [c for c in captured if c[0] != "bm_check_all_true"] == eager


def test_mask_check_on_the_emulator(monkeypatch):
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    est, cand = torch.randn(3, 4, 20), torch.randn(3, 4, 20)
    good = torch.ones(3, 1, 20, dtype=torch.bool)
    for n_false, where in ((1, -1), (1, 0), (2, 7)):
        bad = good.clone()
        bad.view(-1)[where] = False
        if n_false == 2:
            bad.view(-1)[-3] = False
        with frozen_emulator.emulated(_Emulator):
            with pytest.raises(AssertionError, match="mask is not supported"):     # eager: the host check
                bb.ClipLoss()(est, cand, bad)
            with capturing(monkeypatch):
                bb.ClipLoss()(est, cand, good)
            BF.check_tc_status()
            with capturing(monkeypatch):
                bb.ClipLoss()(est, cand, bad)                  # nothing raised while capturing ...
            with pytest.raises(AssertionError, match="mask is not supported"):
                BF.check_tc_status()                           # ... the next status read does, and clears the word
            BF.check_tc_status()


def test_refusals_while_capturing(monkeypatch):
    import brainmagick_b200 as bb
    import brainmagick_b200.distrib as D
    from brainmagick_b200 import synthetic
    torch.manual_seed(0)
    model = bb.SimpleConv(in_channels=dict(meg=10), out_channels=8, **dict(
        hidden=dict(meg=16), depth=2, kernel_size=3, skip=True, subject_layers=True, subject_dim=0, complex_out=True,
        merger=True, initial_linear=12, merger_channels=12, gelu=True, batch_norm=True, merger_pos_dim=32, n_subjects=3))
    meg, subj = torch.randn(4, 10, 6), torch.tensor([0, 1, 2, 1])
    batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(3, 10), subj)
    sb = _static(batch, meg)
    # a reference batch to a model with a merger, on its own and inside SimpleConv
    with capturing(monkeypatch), abi_emulator.emulated():
        with pytest.raises(RuntimeError, match="StaticBatch"):
            model(dict(meg=meg), batch)
        with pytest.raises(RuntimeError, match="StaticBatch"):
            model.merger(meg, batch)
        model(dict(meg=meg), sb)
        model.merger(meg, sb)
        # the frequency table is copied to the device once, not on every call
        assert model.merger.frequencies(meg.device) is model.merger.frequencies(meg.device)
    # a host subject_index without a merger
    no_merger = bb.SimpleConv(in_channels=dict(meg=10), out_channels=8, hidden=dict(meg=16), depth=2, kernel_size=3,
                              batch_norm=True, complex_out=True, n_subjects=3, subject_layers=True)
    with capturing(monkeypatch), abi_emulator.emulated():
        with pytest.raises(RuntimeError, match="subject_index"):
            no_merger(dict(meg=meg), batch)
        no_merger(dict(meg=meg), sb)
    # global_negatives over more than one rank
    monkeypatch.setattr(D, "world_size", lambda: 2)
    with capturing(monkeypatch), pytest.raises(RuntimeError, match="global_negatives"):
        bb.ClipLoss(global_negatives=True)(meg, meg, torch.ones(4, 1, 6, dtype=torch.bool))
    # a SyncBatchNorm layer that syncs over more than one rank
    import torch.distributed as dist
    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    synced = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model, process_group=object())   # a group of 2 ranks
    with capturing(monkeypatch), abi_emulator.emulated(), pytest.raises(RuntimeError, match="SyncBatchNorm"):
        synced(dict(meg=meg), sb)
