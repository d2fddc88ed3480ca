"""The drop-in modules run on the CPU through `tests/abi_emulator.py` (a torch restatement of each FP32 entry point's
documented contract) against the verbatim-reference fixtures.

  * The fixtures of the default configuration pass on the GPU; that they also pass here validates the emulator's reading of
    the C-ABI contracts AND pins the host-side composition numerically without a GPU.
  * Compositions that have not had their first GPU run (the ablation rows) are held to their fixtures the same way, so what
    remains unverified for them is only kernels that are individually verified elsewhere.
The CUDA kernels themselves are never exercised here; `-m gpu` tests do that."""
import numpy as np
import pytest
import torch

import abi_emulator
from conftest import GOLDEN_CASES, load_arrays, load_golden, rel_err

TOL = 2e-5


def _check_grads(model, ref, tol=5e-5):
    scale = max(float(np.linalg.norm(np.asarray(v))) for k, v in ref.items() if k.endswith("weight") and np.asarray(v).size)
    for name, p in model.named_parameters():
        want = torch.as_tensor(np.asarray(ref[name]))
        if want.numel() == 0:
            continue
        assert p.grad is not None, name
        if want.norm() < 1e-5 * scale:
            assert p.grad.abs().max().item() < 1e-4 * scale + 1e-6, name
        else:
            assert rel_err(p.grad, want) < tol, (name, rel_err(p.grad, want))


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_default_configuration_on_the_emulator(name):
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
    with abi_emulator.emulated():
        est = model(dict(meg=t["meg"]), batch)
        loss = clip(est, t["candidates"], torch.ones(len(t["meg"]), 1, t["meg"].shape[2], dtype=torch.bool))
        loss.backward()
        probs = clip.get_probabilities(est.detach(), t["candidates"])
    assert rel_err(est.detach(), t["estimate"]) < TOL
    assert abs(loss.item() - t["loss"].item()) < 1e-5
    assert rel_err(probs, t["probs"]) < TOL
    _check_grads(model, {k[2:]: v.numpy() for k, v in t.items() if k.startswith("g.")})
    sd = model.state_dict()
    for key, v in t.items():
        if key.startswith("bn."):
            if "num_batches" in key:
                assert int(sd[key[3:]]) == int(v)
            else:
                assert rel_err(sd[key[3:]], v) < TOL, key


def _ablation_names():
    from oracle.make_golden import ABLATIONS
    return list(ABLATIONS)


@pytest.mark.parametrize("name", _ablation_names())
def test_ablation_rows_on_the_emulator(name):
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
    batch = synthetic.make_batch(meg, subj, torch.from_numpy(g["rec_positions"]), subj)
    with abi_emulator.emulated():
        est = model(dict(meg=meg), batch)
        loss = bb.ClipLoss()(est, torch.from_numpy(g["candidates"]), torch.ones(len(meg), 1, meg.shape[2], dtype=torch.bool))
        loss.backward()
    assert rel_err(est.detach(), torch.from_numpy(g["estimate"])) < TOL
    assert abs(loss.item() - float(g["loss"])) < 1e-5
    _check_grads(model, {k[2:]: v for k, v in g.items() if k.startswith("g.")})


def _deepmel_names():
    from oracle.make_golden import DEEPMEL_CASES
    return list(DEEPMEL_CASES)


@pytest.mark.parametrize("case", _deepmel_names())
def test_deepmel_on_the_emulator(case):
    import brainmagick_b200 as bb
    from oracle.make_golden import DEEPMEL_CASES
    g = load_arrays(case)
    c = DEEPMEL_CASES[case]
    model = bb.DeepMel(n_in_channels=c["n_in"], **c["params"])
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
    model.train()
    mel = torch.from_numpy(g["mel"]).requires_grad_(True)
    est = torch.from_numpy(g["estimate"]).requires_grad_(True)
    with abi_emulator.emulated():
        cand = model(mel)
        cand.retain_grad()
        loss = bb.ClipLoss()(est, cand, torch.ones(len(est), 1, est.shape[2], dtype=torch.bool))
        loss.backward()
        model.eval()
        with torch.no_grad():
            out_eval = model(mel.detach())
    assert rel_err(cand.detach(), torch.from_numpy(g["candidates"])) < TOL
    assert abs(loss.item() - float(g["loss"])) < 1e-5
    assert rel_err(est.grad, torch.from_numpy(g["g.estimate"])) < 5e-5
    assert rel_err(cand.grad, torch.from_numpy(g["g.candidates"])) < 5e-5
    assert mel.grad is not None and torch.isfinite(mel.grad).all()
    _check_grads(model, {k[2:]: v for k, v in g.items() if k.startswith("g.") and k[2:] not in ("estimate", "candidates")})
    assert rel_err(out_eval, torch.from_numpy(g["candidates_eval"])) < TOL


def test_retrieval_host_path_on_the_emulator():
    """builds_probs / accuracies / the batched get_wer ranking (vocabulary bookkeeping, own-candidate column) against the
    retrieval fixture.  These run green on the GPU too; here they guard the host logic between GPU sessions."""
    import types
    import brainmagick_b200 as bb
    from brainmagick_b200 import retrieval
    g = load_arrays("retrieval_small")
    t = lambda k: torch.from_numpy(g[k])     # noqa: E731
    clip = bb.ClipLoss().eval()
    args = types.SimpleNamespace(tmin=-0.5, sample_rate=120.0)
    with abi_emulator.emulated():
        probs = retrieval.builds_probs(clip, t("preds"), t("trues"), args, batch_size=10)
        pw = retrieval.builds_probs(clip, t("preds"), t("trues"), args, batch_size=7, tmin=-0.45, tmax=-0.4)
        acc = retrieval.retrieval_accuracy(clip, t("preds"), t("trues"), t("target_labels"), t("vocab_labels"),
                                           topk=(1, 5, 10), batch_size=9)
        acc10 = retrieval._get_accuracy_from_probs(t("probs"), t("target_labels"), t("vocab_labels"), topk=10)
        res = [retrieval.wer_ranking(clip, t("wer_estimates"), t("wer_word_hashes"), t("wer_outputs"), t("wer_negatives"),
                                     t("wer_negative_hashes"), int(g["wer_topx"]), batch_size=bs) for bs in (5, 64)]
    assert np.abs(probs.numpy() - g["probs"]).max() < 2e-6
    assert np.abs(pw.numpy() - g["probs_window"]).max() < 2e-6
    assert [acc[1], acc[5], acc[10]] == pytest.approx([float(a) for a in g["acc"]])
    assert acc10 == pytest.approx(float(g["acc"][2]))
    for r in res:
        assert r["wer"] == pytest.approx(float(g["wer"])) and r["wer_vocab"] == pytest.approx(float(g["wer_vocab"]))
        assert r["soft_correct"] == pytest.approx(float(g["wer_soft"]), rel=1e-4)


@pytest.mark.parametrize("clip", [0, 1])
@pytest.mark.parametrize("excl", [0, 1])
def test_batch_preparation_host_path_on_the_emulator(clip, excl):
    import types
    from brainmagick_b200 import norm as bnorm, synthetic
    g = load_arrays("prep_small")
    off = int(g["offset"])

    class Builder(dict):
        dimension = 5

        def __init__(self):
            super().__init__(a=types.SimpleNamespace(normalizable=True, categorical=False, cardinality=0),
                             b=types.SimpleNamespace(normalizable=False, categorical=False, cardinality=0))

        def get_slice(self, name):
            return dict(a=slice(0, 3), b=slice(3, 5))[name]

    for tag in ("pc0.", "pc1."):
        sc = bnorm.BatchScaler(Builder(), per_channel=(tag == "pc1."))
        for i, r in enumerate(g["rec_ids"]):
            s = bnorm.Scaler()
            s.center_, s.scale_ = torch.from_numpy(g[tag + "meg_center"][i]), torch.from_numpy(g[tag + "meg_scale"][i])
            sc.meg_scalers[int(r)] = s
        sc.feature_scalers["a"].center_ = torch.from_numpy(g[tag + "feat_center"][:3])
        sc.feature_scalers["a"].scale_ = torch.from_numpy(g[tag + "feat_scale"][:3])
        batch = synthetic.SyntheticBatch(torch.from_numpy(g["meg"]), torch.zeros(len(g["meg"]), dtype=torch.long), [],
                                         features=torch.from_numpy(g["features"]),
                                         features_mask=torch.from_numpy(g["features_mask"]),
                                         recording_index=torch.from_numpy(g["recording_index"]))
        k = f"{tag}clip{clip}.excl{excl}."
        with abi_emulator.emulated():
            sr = bnorm.ScaleReject(sc, limit=float(g["limit"]), exclude_empty_features=bool(excl), clip=bool(clip))
            kept, keep = sr(batch)
            meg, feats, mask, keep2 = sr.prepare(batch, off)
            back = sc.inverse_transform(sc.transform(batch))
        assert np.array_equal(keep.numpy(), g[k + "keep"]) and np.array_equal(keep2.numpy(), g[k + "keep"])
        assert np.array_equal(kept.meg[..., off:].numpy(), g[k + "meg"])
        assert np.array_equal(meg.numpy(), g[k + "meg"])
        assert np.array_equal(feats.numpy(), g[k + "features"])
        assert np.array_equal(mask.numpy(), g[k + "features_mask"])
        assert np.array_equal(back.meg.numpy(), g[tag + "inverse.meg"])


@pytest.mark.parametrize("shape", [
    # the "tensor-core-eligible widths" case of tests/test_gpu_parity.py (mixed tensor-core / FMA kernels)
    dict(B=8, C=40, T=130, F=128, S=3, hidden=160, MC=48, IL=24, P=128, n_valid=()),
    # BASELINE widths (every contraction through a tensor-core entry point), short and narrow in batch/time only
    dict(B=3, C=208, T=48, F=1024, S=4, hidden=320, MC=270, IL=270, P=2048, n_valid=(208, 150, 208, 97)),
])
@pytest.mark.parametrize("train", [True, False])
def test_tensor_core_host_path_on_the_emulator(shape, train):
    """The tensor-core host path (channel paddings, tf32 hi/lo operand layouts, per-recording / per-subject weight sets,
    grouped weight gradients, fused statistics, in-place reduce-add) with the tensor-core entry points emulated in exact
    fp32, against the oracle."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
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
    clip = bb.ClipLoss().train(train)
    with abi_emulator.emulated() as emu:
        est = model(dict(meg=d["meg"]), batch)
        loss = clip(est, d["candidates"], torch.ones(len(d["meg"]), 1, d["meg"].shape[2], dtype=torch.bool))
        loss.backward()
    assert rel_err(est.detach(), ref["estimate"]) < TOL
    assert abs(loss.item() - ref["loss"].item()) < 1e-5
    _check_grads(model, {k: v.numpy() for k, v in ref["grads"].items()}, tol=2e-4)     # fp32 summation-order noise
    if train:
        sd = model.state_dict()
        for key, v in ref["bn_updates"].items():
            assert rel_err(sd[key], v) < TOL, key


@pytest.mark.parametrize("activation", [None, "gelu"])
def test_deepmel_tensor_core_widths_on_the_emulator(activation):
    """conf/feature_model/deep_mel.yaml at its real widths (120 mel padded to 128 -> 9 x 320 -> 768), short in batch/time:
    the stand-alone ConvSequence's tensor-core host path and the candidate-side ClipLoss gradient against the oracle."""
    import brainmagick_b200 as bb
    from oracle import bm_oracle, deepmel_oracle
    kw = dict(n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3, stride=1, dilation_growth=2,
              dilation_period=5, batch_norm=True, activation_on_last=False, skip=True, glu_context=1, glu=2)
    if activation == "gelu":
        kw["activation"] = torch.nn.GELU
    torch.manual_seed(3)
    model = bb.DeepMel(n_in_channels=120, **kw).train()
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    okw = {k: v for k, v in kw.items() if k not in ("stride", "activation", "n_hidden_channels", "n_hidden_layers",
                                                    "n_out_channels")}
    spec = deepmel_oracle.deep_mel_spec(120, 320, 10, 768, activation="gelu" if activation == "gelu" else "lrelu", **okw)
    B, T = 3, 40
    mel, est = torch.randn(B, 120, T), torch.randn(B, 768, T)
    p = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in params.items()}
    m_ref, e_ref = mel.clone().requires_grad_(True), est.clone().requires_grad_(True)
    cand_ref = deepmel_oracle.conv_sequence(m_ref, p, spec, training=True)
    cand_ref.retain_grad()
    loss_ref = bm_oracle.clip_loss(e_ref, cand_ref)
    loss_ref.backward()
    m, e = mel.clone().requires_grad_(True), est.clone().requires_grad_(True)
    with abi_emulator.emulated():
        cand = model(m)
        cand.retain_grad()
        loss = bb.ClipLoss()(e, cand, torch.ones(B, 1, T, dtype=torch.bool))
        loss.backward()
    assert rel_err(cand.detach(), cand_ref.detach()) < TOL
    assert abs(loss.item() - loss_ref.item()) < 1e-5
    assert rel_err(e.grad, e_ref.grad) < 5e-5 and rel_err(cand.grad, cand_ref.grad) < 5e-5
    assert rel_err(m.grad, m_ref.grad) < 5e-4
    _check_grads(model, {k: v.grad.numpy() for k, v in p.items() if v.grad is not None}, tol=5e-4)


@pytest.mark.parametrize("change", [dict(glu=0), dict(skip=False), dict(gelu=False), dict(complex_out=False),
                                    dict(merger=False), dict(initial_linear=0), dict(subject_layers=False),
                                    dict(subject_layers=False, subject_dim=64)],
                         ids=lambda c: ",".join(f"{k}={v}" for k, v in c.items()))
def test_ablation_rows_at_baseline_widths_on_the_emulator(change):
    """Every row of the ablation table at the BASELINE widths (where the convolutions, weight gradients and -- for the
    un-ablated sensor chain -- the sensor stages go through tensor-core entry points), against `oracle/ablation_oracle.py`."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import ablation_oracle, bm_oracle
    B, C, T, Fo, S = 3, 208, 48, 1024, 4
    kw = dict(hidden=dict(meg=320), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=270, merger_channels=270,
              gelu=True, batch_norm=True, merger_pos_dim=2048, merger_dropout=0.2, n_subjects=S)
    kw.update(change)
    torch.manual_seed(17)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=Fo, **kw).train()
    v = ablation_oracle.Variant(in_channels=C, out_channels=Fo, n_subjects=S)._replace(
        **{k: val for k, val in change.items()})
    p = {k: t.detach().clone().requires_grad_(t.is_floating_point() and "running" not in k)
         for k, t in model.state_dict().items()}
    meg = torch.randn(B, C, T).clamp_(-20, 20)
    cand = torch.randn(B + 2, Fo, T)
    subj = torch.tensor([2, 0, 2])
    pos = synthetic.normalised_positions(S, C, (208, 150, 208, 97), seed=4)
    for b in range(B):
        meg[b, (208, 150, 208, 97)[int(subj[b])]:] = 0
    ban = torch.tensor([0.31, 0.64])
    est_ref = ablation_oracle.forward(p, v, meg, pos, subj, subj, training=True, ban_centre=ban)
    loss_ref = bm_oracle.clip_loss(est_ref, cand)
    loss_ref.backward()
    if model.merger is not None:
        model.merger.ban_centre_override = ban
    batch = synthetic.make_batch(meg, subj, pos, subj)
    with abi_emulator.emulated():
        est = model(dict(meg=meg), batch)
        loss = bb.ClipLoss()(est, cand, torch.ones(B, 1, T, dtype=torch.bool))
        loss.backward()
    assert rel_err(est.detach(), est_ref.detach()) < TOL
    assert abs(loss.item() - loss_ref.item()) < 1e-5
    _check_grads(model, {k: t.grad.numpy() for k, t in p.items() if t.grad is not None}, tol=2e-4)


def test_multi_step_training_state_on_the_emulator():
    """Four Adam steps: parameters, BatchNorm running statistics and `num_batches_tracked` carried from step to step must
    follow the oracle trainer (solver.py:297,373,384-387 restated) -- the state handling around the encoder function."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
    cfg = bm_oracle.Config(in_channels=12, out_channels=10, n_subjects=3, hidden=16, merger_channels=12, initial_linear=12,
                           merger_pos_dim=32)
    params = bm_oracle.init_state_dict(cfg, seed=5)
    trainer = bm_oracle.CpuTrainer(cfg, params, lr=2e-4)
    model = bb.SimpleConv(
        in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden), depth=cfg.depth,
        dilation_period=5, kernel_size=3, skip=True, subject_layers=True, subject_dim=0, complex_out=True, glu=2,
        glu_context=1, merger=True, initial_linear=cfg.initial_linear, merger_channels=cfg.merger_channels, gelu=True,
        batch_norm=True, merger_pos_dim=cfg.merger_pos_dim, n_subjects=cfg.n_subjects)
    model.load_state_dict(params)
    model.train()
    clip = bb.ClipLoss().train()
    opt = torch.optim.Adam(model.parameters(), lr=2e-4, betas=(0.9, 0.999))
    pos = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, seed=2)
    with abi_emulator.emulated():
        for step in range(4):
            d = bm_oracle.synthetic_batch(cfg, batch=6, T=30, seed=100 + step)
            ref_loss = trainer.step(d["meg"], pos, d["rec_of_sample"], d["subject_index"], d["candidates"], d["ban_centre"])
            model.merger.ban_centre_override = d["ban_centre"]
            batch = synthetic.make_batch(d["meg"], d["subject_index"], pos, d["rec_of_sample"])
            opt.zero_grad(set_to_none=True)
            loss = clip(model(dict(meg=d["meg"]), batch), d["candidates"], torch.ones(6, 1, 30, dtype=torch.bool))
            loss.backward()
            opt.step()
            assert abs(loss.item() - ref_loss) < 5e-5 * max(1.0, abs(ref_loss)), (step, loss.item(), ref_loss)
        # Parameters whose true gradient is zero (a conv bias in front of BatchNorm, the heads' column of the constant
        # embedding term) are moved by Adam on rounding noise alone -- lr per step, in a direction the noise decides; the
        # CUDA path returns the exact zero for the conv biases and leaves them where they are.  So parameter tensors cannot
        # be compared one to one, and through the lag of the BatchNorm running means even the eval-mode function differs
        # by O(lr x steps); with a small lr the FUNCTION after training can be compared.
        d = bm_oracle.synthetic_batch(cfg, batch=5, T=30, seed=999)
        p_ref = {k: v.detach() for k, v in trainer.p.items()}
        want = bm_oracle.simpleconv_forward(p_ref, cfg, d["meg"], pos, d["rec_of_sample"], d["subject_index"], False)
        model.eval()
        with torch.no_grad():
            got = model(dict(meg=d["meg"]), synthetic.make_batch(d["meg"], d["subject_index"], pos, d["rec_of_sample"]))
    assert rel_err(got, want) < 1e-3, rel_err(got, want)
    sd = model.state_dict()
    for k, v in trainer.p.items():
        if "num_batches" in k:
            assert int(sd[k]) == 4
        elif "running" in k:          # the running mean tracks the (noise-walking) conv bias of the reference: O(lr x steps)
            assert rel_err(sd[k], v.detach()) < 5e-3, (k, rel_err(sd[k], v.detach()))


def _standalone_modules_case(device):
    """ChannelMerger.forward / SubjectLayers.forward called on their own (bm/models/common.py:334-362, 55-58) against the
    oracle's restatement: values and gradients."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
    g = torch.Generator().manual_seed(5)
    B, C, T, O, P, S, D = 6, 19, 40, 12, 32, 3, 10
    meg = torch.randn(B, C, T, generator=g)
    subj = torch.tensor([0, 2, 1, 2, 0, 1])
    rec_of_sample = torch.tensor([1, 0, 1, 1, 0, 0])
    pos = synthetic.normalised_positions(2, C, n_valid=(C, C - 3), seed=3)
    merger = bb.ChannelMerger(O, pos_dim=P, dropout=0.2).train()
    merger.ban_centre_override = torch.tensor([0.4, 0.6])
    layer = bb.SubjectLayers(O, D, S)
    batch = synthetic.make_batch(meg, subj, pos, rec_of_sample)
    gout = torch.randn(B, D, T, generator=g)

    heads = merger.heads.detach().double().requires_grad_()
    w = layer.weights.detach().double().requires_grad_()
    att = bm_oracle.attention_weights(pos.double(), heads, merger.ban_centre_override.double(), 0.2)
    u = torch.einsum("bct,boc->bot", meg.double(), att[rec_of_sample])
    want = torch.einsum("bct,bcd->bdt", u, w[subj])
    want.backward(gout.double())

    merger, layer = merger.to(device), layer.to(device)
    u_got = merger(meg.to(device), batch)
    got = layer(u_got, subj.to(device))
    got.backward(gout.to(device))
    assert rel_err(u_got.detach().cpu(), u.detach()) < TOL
    assert rel_err(got.detach().cpu(), want.detach()) < TOL
    assert rel_err(merger.heads.grad.cpu(), heads.grad) < 5e-5
    assert rel_err(layer.weights.grad.cpu(), w.grad) < 5e-5
    with pytest.raises(IndexError):
        layer(u_got.detach(), torch.full((B,), S, device=device))


def test_standalone_merger_and_subject_layers_on_the_emulator():
    with abi_emulator.emulated():
        _standalone_modules_case(torch.device("cpu"))


def test_second_backward_raises_a_clear_error():
    """The fused encoder releases its saved activations in backward (ctx.saved, not save_for_backward): a second backward
    through the same graph must say so instead of failing with an opaque TypeError."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    cfg, train, t = load_golden(GOLDEN_CASES[0])
    model = bb.SimpleConv(
        in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden),
        depth=cfg.depth, dilation_period=cfg.dilation_period, kernel_size=cfg.kernel_size, skip=True,
        subject_layers=True, subject_dim=0, complex_out=True, glu=cfg.glu, glu_context=cfg.glu_context, merger=True,
        initial_linear=cfg.initial_linear, merger_channels=cfg.merger_channels, gelu=True, batch_norm=True,
        merger_pos_dim=cfg.merger_pos_dim, merger_dropout=cfg.merger_dropout, n_subjects=cfg.n_subjects)
    model.load_state_dict({k[2:]: v for k, v in t.items() if k.startswith("p.")}, strict=True)
    model.train(True)
    batch = synthetic.make_batch(t["meg"], t["subject_index"], t["rec_positions"], t["rec_of_sample"])
    with abi_emulator.emulated():
        est = model(dict(meg=t["meg"]), batch)
        loss = est.square().mean()
        loss.backward(retain_graph=True)
        with pytest.raises(RuntimeError, match="second time"):
            loss.backward()
