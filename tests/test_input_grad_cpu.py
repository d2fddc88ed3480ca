"""Input gradients without a GPU: the drop-in SimpleConv, ChannelMerger and ClipLoss.get_scores / get_probabilities, run
through `tests/abi_emulator.py` (with the input-gradient entry points of `tests/input_grad_emulator.py`), backpropagate
to `meg` (and to the estimates / candidates) like the verbatim reference (`tests/golden/live_input_grad_*.npz`, made by
oracle/make_input_grad_golden.py).  A step whose `meg` does not require grad
issues the same C-ABI call stream as before input gradients existed (`tests/golden/abi_trace_steps.json`)."""
import json
import os

import pytest
import torch

import abi_emulator
import abi_trace
import input_grad_emulator
from input_grad_emulator import InputGradEmulator
from conftest import GOLDEN_DIR, load_arrays, rel_err

TOL = 1e-4


def _model(C, F, S, hidden, MC, IL, P, depth, **change):
    import brainmagick_b200 as bb
    from oracle.ref_loader import clip_conv_kwargs
    kw = clip_conv_kwargs(hidden=hidden, depth=depth, merger_channels=MC, initial_linear=IL, merger_pos_dim=P)
    kw.update(change)
    return bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **kw)


def _meg_grad(model, meg, subj, pos, cand, ban=None, emulator_class=InputGradEmulator):
    """meg.grad of the ClipLoss through the drop-in, on the emulator (recording = subject, as in the fixtures)."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    if model.merger is not None and ban is not None:
        model.merger.ban_centre_override = ban
    x = meg.clone().requires_grad_(True)
    batch = synthetic.make_batch(x.detach(), subj, pos, subj)
    with input_grad_emulator.emulated(emulator_class):
        est = model(dict(meg=x), batch)
        loss = bb.ClipLoss()(est, cand, torch.ones(len(meg), 1, meg.shape[2], dtype=torch.bool))
        loss.backward()
    return x.grad, loss.item()


def _dead_channels(pos, subj, ban, radius=0.2):
    """[B, C] True where the sensor's attention weight is 0: INVALID (padding) or inside the spatial-dropout disc."""
    dead = (pos == abi_emulator.INVALID).all(-1)
    if ban is not None:
        dead = dead | ((pos - ban).norm(dim=-1) <= radius)
    return dead[subj.long()]


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_simpleconv_meg_grad_matches_reference(mode):
    g = load_arrays("live_input_grad_clip_conv")
    t = lambda k: torch.from_numpy(g[k])     # noqa: E731
    model = _model(C=13, F=9, S=4, hidden=24, MC=16, IL=20, P=72, depth=10)
    model.load_state_dict({k[2:]: t(k) for k in g if k.startswith("p.")}, strict=True)
    model.train(mode == "train")
    ban = t(f"{mode}.ban") if mode == "train" else None
    grad, loss = _meg_grad(model, t("meg"), t("subj"), t("pos"), t("cand"), ban)
    assert abs(loss - float(g[f"{mode}.loss"])) < 1e-5
    want = t(f"{mode}.meg_grad")
    assert rel_err(grad, want) < TOL, rel_err(grad, want)
    dead = _dead_channels(t("pos"), t("subj"), ban)
    assert dead.sum() > (10 if mode == "train" else 5)
    if mode == "train":
        assert (dead & ~_dead_channels(t("pos"), t("subj"), None)).any()       # the centre bans some valid sensors
    assert (want[dead] == 0).all() and (grad[dead] == 0).all()
    assert (grad[~dead].abs().sum(-1) > 0).all()


@pytest.mark.parametrize("row", ["no_merger", "subsample"])
def test_ablation_rows_meg_grad_match_reference(row):
    from oracle.make_golden import ABLATION_BASE as c
    g = load_arrays("live_input_grad_ablations")
    t = lambda k: torch.from_numpy(g[f"{row}.{k}"])     # noqa: E731
    change = dict(merger=False) if row == "no_merger" else dict(subsample_meg_channels=6)
    model = _model(C=c["C"], F=c["F"], S=c["S"], hidden=c["hidden"], MC=c["MC"], IL=c["IL"], P=c["P"], depth=c["depth"],
                   **change)
    pre = f"{row}.p."
    model.load_state_dict({k[len(pre):]: torch.from_numpy(v) for k, v in g.items() if k.startswith(pre)}, strict=True)
    model.train()
    grad, loss = _meg_grad(model, t("meg"), t("subj"), t("pos"), t("cand"), t("ban"))
    assert abs(loss - float(t("loss"))) < 1e-5
    assert rel_err(grad, t("meg_grad")) < TOL, rel_err(grad, t("meg_grad"))
    if row == "subsample":
        dropped = torch.ones(c["C"], dtype=torch.bool)
        dropped[model.subsampled_meg_channels] = False
        assert dropped.sum() == c["C"] - 6
        assert (grad[:, dropped] == 0).all() and (t("meg_grad")[:, dropped] == 0).all()


@pytest.mark.parametrize("name", ["get_scores", "get_probabilities"])
def test_clip_scores_grads_match_reference(name):
    import brainmagick_b200 as bb
    g = load_arrays("live_input_grad_clip_scores")
    t = lambda k: torch.from_numpy(g[k])     # noqa: E731
    e, c = t("est").requires_grad_(True), t("cand").requires_grad_(True)
    with input_grad_emulator.emulated():
        y = getattr(bb.ClipLoss(), name)(e, c)
        y.backward(t("up"))
    assert rel_err(y.detach(), t(f"{name}.out")) < 1e-5
    assert rel_err(e.grad, t(f"{name}.est_grad")) < TOL
    want = t(f"{name}.cand_grad")
    live = torch.ones(len(want), dtype=torch.bool)
    live[3] = False                              # candidate 3 is all zeros: 1/(1e-8 + 0) scales its gradient by 1e8
    assert rel_err(c.grad[live], want[live]) < TOL
    assert rel_err(c.grad[3], want[3]) < TOL
    # without an input that requires grad, no autograd node is recorded (retrieval / evaluation path)
    with input_grad_emulator.emulated():
        assert getattr(bb.ClipLoss(), name)(t("est"), t("cand")).grad_fn is None


def test_standalone_merger_meg_grad_matches_autograd():
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
    gen = torch.Generator().manual_seed(8)
    B, C, T, O, P = 5, 17, 30, 12, 32
    meg = torch.randn(B, C, T, generator=gen)
    rec_of_sample = torch.tensor([1, 0, 1, 1, 0])
    pos = synthetic.normalised_positions(2, C, n_valid=(C, C - 4), seed=3)
    merger = bb.ChannelMerger(O, pos_dim=P, dropout=0.2).train()
    ban = torch.tensor([0.4, 0.6])
    merger.ban_centre_override = ban
    gout = torch.randn(B, O, T, generator=gen)
    x = meg.clone().double().requires_grad_(True)
    att = bm_oracle.attention_weights(pos.double(), merger.heads.detach().double(), ban.double(), 0.2)
    torch.einsum("bct,boc->bot", x, att[rec_of_sample]).backward(gout.double())
    m = meg.clone().requires_grad_(True)
    with input_grad_emulator.emulated():
        merger(m, synthetic.make_batch(meg, rec_of_sample, pos, rec_of_sample)).backward(gout)
    assert rel_err(m.grad, x.grad) < TOL
    dead = _dead_channels(pos, rec_of_sample, ban)
    assert dead.any() and (m.grad[dead] == 0).all()


@pytest.mark.parametrize("change", [{}, dict(subsample_meg_channels=150), dict(merger=False), dict(initial_linear=0),
                                    dict(subject_layers=False, subject_dim=64)],
                         ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()) or "clip_conv")
def test_meg_grad_at_baseline_widths_on_the_emulator(change):
    """At the BASELINE widths the fused chain's mix runs on the tensor cores, so its data gradient does too
    (bm_tc_sensor_mix_bwd_data: transposed, zero-padded weight sets, channel-major store of the live sensors);
    the ablation rows take their stage-by-stage paths.  Against `oracle/ablation_oracle.py` differentiated by autograd."""
    from brainmagick_b200 import synthetic
    from oracle import ablation_oracle, bm_oracle
    B, C, T, Fo, S = 2, 208, 48, 1024, 4
    torch.manual_seed(19)
    model = _model(C=C, F=Fo, S=S, hidden=320, MC=270, IL=270, P=2048, depth=10, **change).train()
    v = ablation_oracle.Variant(in_channels=C, out_channels=Fo, n_subjects=S)._replace(**change)
    p = {k: t.detach().clone() for k, t in model.state_dict().items()}
    meg = torch.randn(B, C, T)
    cand = torch.randn(B + 1, Fo, T)
    subj = torch.tensor([3, 1])
    n_valid = (208, 150, 208, 97)
    pos = synthetic.normalised_positions(S, C, n_valid, seed=4)
    ban = torch.tensor([0.31, 0.64])
    x = meg.clone().requires_grad_(True)
    bm_oracle.clip_loss(ablation_oracle.forward(p, v, x, pos, subj, subj, training=True, ban_centre=ban), cand).backward()
    calls = []

    class Spy(InputGradEmulator):
        def __getattribute__(self, name):
            if name.startswith("bm_"):
                calls.append(name)
            return InputGradEmulator.__getattribute__(self, name)
    grad, _ = _meg_grad(model, meg, subj, pos, cand, ban, emulator_class=Spy)
    assert rel_err(grad, x.grad) < TOL, rel_err(grad, x.grad)
    if not change:
        assert "bm_tc_sensor_mix_bwd_data" in calls and "bm_sensor_mix_bwd_data" not in calls


# ---------------------------------------------------------------- the C-ABI call stream
def _trace(cfg, train, meg_grad, **overrides):
    """abi_trace.simpleconv_step, optionally with meg.requires_grad."""
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import synthetic
    B, C, T, F, S, hidden, MC, IL, P = cfg
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2, n_subjects=S)
    kw.update(overrides)

    def run():
        torch.manual_seed(0)
        model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, **kw).train(train)
        subj = torch.randint(0, S, (B,))
        meg, cand = torch.randn(B, C, T).requires_grad_(meg_grad), torch.randn(B, F, T)
        batch = synthetic.make_batch(meg.detach(), subj, synthetic.normalised_positions(S, C), subj)
        BF.clip_loss(model(dict(meg=meg), batch), cand, 0).backward()
    return abi_trace.record(run)


def test_steps_without_meg_grad_keep_their_call_stream():
    """Training and evaluation steps, default and ablation rows: exactly the calls recorded before input gradients existed."""
    want = json.load(open(os.path.join(GOLDEN_DIR, "abi_trace_steps.json")))
    got = abi_trace.all_traces()
    for tag, change in (("small.train.subsample", dict(subsample_meg_channels=6)),
                        ("full.train.subsample", dict(subsample_meg_channels=150)),
                        ("small.train.no_merger", dict(merger=False)),
                        ("small.train.no_initial_linear", dict(initial_linear=0))):
        cfg, mode = tag.split(".")[:2]
        got[tag] = abi_trace.simpleconv_step(abi_trace.CONFIGS[cfg], mode == "train", **change)
    got = json.loads(json.dumps(got))
    assert set(got) == set(want)
    for tag in want:
        assert got[tag] == want[tag], tag


@pytest.mark.parametrize("cfg,change,extra", [
    ("full", {}, ["bm_tc_weight_split", "bm_tc_sensor_mix_bwd_data"]),
    ("small", {}, ["bm_sensor_mix_bwd_data"]),
    ("small", dict(merger=False), ["bm_transpose_nt"]),
    ("small", dict(merger=False, subsample_meg_channels=6), ["bm_transpose_nt", "bm_channel_mask"]),
])
def test_meg_grad_only_adds_its_own_calls(cfg, change, extra):
    """With meg.requires_grad the step issues the same calls plus the input-gradient ones, in one block."""
    base = _trace(abi_trace.CONFIGS[cfg], True, False, **change)
    with_grad = _trace(abi_trace.CONFIGS[cfg], True, True, **change)
    assert len(with_grad) == len(base) + len(extra)
    names = [c[0] for c in with_grad]
    pos = [i for i, n in enumerate(names) if n == extra[-1]][-1]
    assert names[pos - len(extra) + 1:pos + 1] == extra
    assert with_grad[:pos - len(extra) + 1] + with_grad[pos + 1:] == base
