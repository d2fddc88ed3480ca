"""GPU parity tests proper: the drop-in modules (CUDA through the C ABI) against
  (1) the golden vectors produced by the verbatim reference (tests/golden, oracle/make_golden.py), and
  (2) the oracle restatement on freshly seeded inputs at sizes the oracle finishes in seconds.
Tolerance: 1e-4 relative (north-star), measured as ||x - ref||_F / ||ref||_F."""
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _build_model(cfg, params, device="cuda"):
    import brainmagick_b200 as bb
    model = bb.SimpleConv(
        in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden),
        depth=cfg.depth, dilation_period=cfg.dilation_period, kernel_size=cfg.kernel_size, skip=True,
        subject_layers=True, subject_dim=0, complex_out=True, glu=cfg.glu, glu_context=cfg.glu_context, merger=True,
        initial_linear=cfg.initial_linear, merger_channels=cfg.merger_channels, gelu=True, batch_norm=True,
        merger_pos_dim=cfg.merger_pos_dim, merger_dropout=cfg.merger_dropout, n_subjects=cfg.n_subjects)
    missing = model.load_state_dict(params, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    return model.to(device)


def _run_step(model, cfg, t, train, target_offset=0):
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    dev = "cuda"
    meg = t["meg"].to(dev)
    batch = synthetic.make_batch(meg, t["subject_index"].to(dev), t["rec_positions"], t["rec_of_sample"])
    model.train(train)
    model.merger.ban_centre_override = t["ban_centre"]
    clip = bb.ClipLoss().to(dev)
    clip.train(train)
    est = model(dict(meg=meg), batch)
    cand = t["candidates"].to(dev)
    mask = torch.ones(meg.shape[0], 1, meg.shape[2], dtype=torch.bool, device=dev)
    loss = clip(est, cand, mask)
    loss.backward()
    scores = clip.get_scores(est.detach(), cand)
    probs = clip.get_probabilities(est.detach(), cand)
    torch.cuda.synchronize()
    from brainmagick_b200 import functional as BF
    BF.check_tc_status()
    return est.detach().cpu(), loss.detach().cpu(), scores.cpu(), probs.cpu()


def _check_grads(model, ref_grads, train, tol):
    wscale = max(v.norm().item() for k, v in ref_grads.items() if k.endswith("weight") and v.numel())
    for name, p in model.named_parameters():
        ref = ref_grads[name]
        assert p.grad is not None, name
        g = p.grad.detach().cpu()
        if train and "sequence" in name and name.endswith(".0.bias"):
            assert g.abs().max().item() < 1e-4 * wscale + 1e-6, name      # true gradient is 0 (BN follows)
            continue
        assert rel_err(g, ref) < tol, (name, rel_err(g, ref))


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_drop_in_matches_reference_golden(name):
    cfg, train, t = load_golden(name)
    params = {k[2:]: v for k, v in t.items() if k.startswith("p.")}
    model = _build_model(cfg, params)
    est, loss, scores, probs = _run_step(model, cfg, t, train)
    assert est.shape == t["estimate"].shape
    assert rel_err(est, t["estimate"]) < TOL
    assert rel_err(scores, t["scores"]) < TOL
    assert abs(loss.item() - t["loss"].item()) < TOL * max(1.0, abs(t["loss"].item()))
    assert rel_err(probs, t["probs"]) < TOL
    k = min(5, probs.shape[1])
    assert torch.equal(probs.topk(k, dim=1).indices, t["probs"].topk(k, dim=1).indices)
    _check_grads(model, {k2[2:]: v for k2, v in t.items() if k2.startswith("g.")}, train, TOL)
    sd = model.state_dict()
    for key, v in t.items():
        if key.startswith("bn."):
            got = sd[key[3:]].cpu()
            if "num_batches" in key:
                assert int(got) == int(v)
            else:
                assert rel_err(got, v) < TOL, key


@pytest.mark.parametrize("shape", [
    dict(B=16, C=64, T=120, F=40, S=4, hidden=64, MC=48, IL=56, P=288, n_valid=()),          # cfg1-like (mock, 64 sensors)
    dict(B=12, C=37, T=91, F=33, S=5, hidden=40, MC=30, IL=34, P=128, n_valid=(37, 20, 11)),   # ragged / padded
    dict(B=8, C=40, T=130, F=128, S=3, hidden=160, MC=48, IL=24, P=128, n_valid=()),           # tensor-core-eligible widths
])
@pytest.mark.parametrize("train", [True, False])
def test_drop_in_matches_oracle(shape, train):
    from oracle import bm_oracle
    cfg = bm_oracle.Config(in_channels=shape["C"], out_channels=shape["F"], n_subjects=shape["S"],
                           hidden=shape["hidden"], merger_channels=shape["MC"], initial_linear=shape["IL"],
                           merger_pos_dim=shape["P"])
    params = bm_oracle.init_state_dict(cfg, seed=11)
    from brainmagick_b200 import synthetic
    d = bm_oracle.synthetic_batch(cfg, batch=shape["B"], T=shape["T"], seed=5, n_valid=shape["n_valid"])
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, shape["n_valid"], seed=3)
    ref = bm_oracle.training_step(params, cfg, d["meg"], d["rec_positions"], d["rec_of_sample"], d["subject_index"],
                                  d["candidates"], ban_centre=d["ban_centre"], training=train)
    model = _build_model(cfg, params)
    est, loss, scores, probs = _run_step(model, cfg, d, train)
    assert rel_err(est, ref["estimate"]) < TOL
    assert rel_err(scores, ref["scores"]) < TOL
    assert abs(loss.item() - ref["loss"].item()) < TOL * max(1.0, abs(ref["loss"].item()))
    _check_grads(model, ref["grads"], train, TOL)
    if train:
        sd = model.state_dict()
        for key, v in ref["bn_updates"].items():
            assert rel_err(sd[key].cpu(), v) < TOL, key


def test_extra_negatives_and_target_offset():
    """B' > B (negatives beyond the targets, losses.py:105-109) and the multi-GPU target offset."""
    import brainmagick_b200.functional as BF
    from oracle import bm_oracle
    torch.manual_seed(0)
    est = torch.randn(6, 9, 31)
    cand = torch.randn(20, 9, 31)
    for off in (0, 6, 14):
        e = est.clone().cuda().requires_grad_(True)
        loss = BF.clip_loss(e, cand.cuda(), off)
        loss.backward()
        e_ref = est.clone().requires_grad_(True)
        ref = bm_oracle.clip_loss(e_ref, cand, off)
        ref.backward()
        assert abs(loss.item() - ref.item()) < 1e-5
        assert rel_err(e.grad.cpu(), e_ref.grad) < TOL


BASELINE_SHAPES = [
    dict(name="cfg2 gwilliams2022", B=16, C=208, T=360, F=1024, S=27, n_valid=()),
    dict(name="cfg3 audio_mous", B=12, C=273, T=360, F=1024, S=96, n_valid=()),
    dict(name="cfg4 broderick2019 mel", B=16, C=128, T=360, F=120, S=19, n_valid=()),
    dict(name="cfg5 mixed studies, real T", B=13, C=273, T=343, F=1024, S=175, n_valid=(273, 208, 128, 60)),
]


@pytest.mark.parametrize("case", BASELINE_SHAPES, ids=[c["name"].split()[0] for c in BASELINE_SHAPES])
def test_baseline_shapes_match_oracle(case):
    """BASELINE.json configs 2-5 at their REAL widths (hidden 320, merger 270, 2048-d positional embedding, F = 1024 / 120,
    sensors 208 / 273 / 128 / padded mixed studies, T = 360 and the real-training 343) against the oracle restatement of the
    reference (oracle/bm_oracle.training_step) on the same seeded inputs: estimate, scores, loss, BatchNorm running
    statistics and EVERY parameter gradient.  The truth is the oracle in fp64; the oracle in fp32 (= what the reference
    computes) is run beside it to show its own distance from that truth.  Bar: 1e-4 relative on everything (north star),
    gradients included; the conv biases in front of a training-mode BatchNorm have an exactly-zero true gradient (rounding
    noise in the reference) and are compared in absolute terms.  Only the batch is small (the CPU oracle needs ~1 s per
    8 segments); every tensor-core tiling of the full-size model is exercised (all widths are the full ones)."""
    from oracle import bm_oracle
    from brainmagick_b200 import synthetic
    cfg = bm_oracle.Config(in_channels=case["C"], out_channels=case["F"], n_subjects=case["S"])
    params = bm_oracle.init_state_dict(cfg, seed=21)
    d = bm_oracle.synthetic_batch(cfg, batch=case["B"], T=case["T"], seed=9, n_valid=case["n_valid"])
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, case["n_valid"], seed=4)

    def oracle(dtype):
        cast = lambda t: t.to(dtype) if t.is_floating_point() else t          # noqa: E731
        return bm_oracle.training_step({k: cast(v) for k, v in params.items()}, cfg, cast(d["meg"]), cast(d["rec_positions"]),
                                       d["rec_of_sample"], d["subject_index"], cast(d["candidates"]),
                                       ban_centre=cast(d["ban_centre"]), training=True)
    ref64, ref32 = oracle(torch.float64), oracle(torch.float32)
    model = _build_model(cfg, params)
    est, loss, scores, probs = _run_step(model, cfg, d, True)
    e_est, e_sc = rel_err(est, ref64["estimate"]), rel_err(scores, ref64["scores"])
    print(f"[{case['name']}] estimate {e_est:.2e} (oracle fp32: {rel_err(ref32['estimate'], ref64['estimate']):.2e}), "
          f"scores {e_sc:.2e}, loss {loss.item():.6f} vs {ref64['loss'].item():.6f}")
    assert e_est < TOL and e_sc < TOL
    assert abs(loss.item() - ref64["loss"].item()) < TOL * max(1.0, abs(ref64["loss"].item()))
    sd = model.state_dict()
    for key, v in ref64["bn_updates"].items():
        assert rel_err(sd[key].cpu(), v) < TOL, key
    wscale = max(v.norm().item() for k, v in ref64["grads"].items() if k.endswith("weight") and v.numel())
    worst, worst32 = ("", 0.0), 0.0
    for name, p in model.named_parameters():
        g, r64, r32 = p.grad.detach().cpu(), ref64["grads"][name], ref32["grads"][name]
        if "sequence" in name and name.endswith(".0.bias"):
            assert g.abs().max().item() < 1e-4 * wscale + 1e-6, name                 # true gradient is 0 (BatchNorm follows)
            continue
        e = rel_err(g, r64)
        worst32 = max(worst32, rel_err(r32, r64))
        if e > worst[1]:
            worst = (name, e)
        assert e < TOL, (case["name"], name, e)
    print(f"[{case['name']}] worst gradient {worst[1]:.2e} ({worst[0]}); the fp32 oracle's own worst: {worst32:.2e}")


@pytest.mark.parametrize("Bn,Bc", [(256, 256), (64, 512), (100, 256)])
def test_clip_tensor_core_shapes_match_oracle(Bn, Bc):
    """ClipLoss at tensor-core-eligible candidate counts (B' % 256 == 0, F*T % 320 == 0), incl. ragged row counts and the
    multi-GPU target offset, against the CPU oracle (F*T kept small so the oracle is instant)."""
    import brainmagick_b200.functional as BF
    from oracle import bm_oracle
    torch.manual_seed(Bn + Bc)
    F, T = 40, 64                                    # F*T = 2560 = 8 * 320
    est = torch.randn(Bn, F, T)
    cand = torch.randn(Bc, F, T)
    off = Bc - Bn if Bc > Bn else 0
    e = est.clone().cuda().requires_grad_(True)
    loss = BF.clip_loss(e, cand.cuda(), off)
    loss.backward()
    scores = BF.clip_scores(est.cuda(), cand.cuda())
    torch.cuda.synchronize()
    BF.check_tc_status()
    e_ref = est.clone().requires_grad_(True)
    ref = bm_oracle.clip_loss(e_ref, cand, off)
    ref.backward()
    assert rel_err(scores.cpu(), bm_oracle.clip_scores(est, cand)) < TOL
    assert abs(loss.item() - ref.item()) < 1e-5 * max(1.0, abs(ref.item()))
    assert rel_err(e.grad.cpu(), e_ref.grad) < TOL


@pytest.mark.gpu
def test_standalone_merger_and_subject_layers_match_oracle():
    """ChannelMerger.forward / SubjectLayers.forward on their own (bm/models/common.py:334-362, 55-58) run the stage kernels."""
    from test_emulated_host_path import _standalone_modules_case
    _standalone_modules_case(torch.device("cuda"))


@pytest.mark.gpu
def test_subject_index_out_of_range_is_reported():
    """A subject index beyond n_subjects: the reference's weight gather raises (bm/models/common.py:57).  The tensor-core
    per-sample 1x1 kernel must not read outside its weight sets and reports it through the status word (no host sync in the
    forward pass): `functional.check_tc_status()` raises IndexError."""
    from oracle import bm_oracle
    from brainmagick_b200 import functional as BF, synthetic
    cfg = bm_oracle.Config(in_channels=208, out_channels=1024, n_subjects=27)
    params = bm_oracle.init_state_dict(cfg, seed=21)
    d = bm_oracle.synthetic_batch(cfg, batch=4, T=120, seed=9)
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, (), seed=4)
    model = _build_model(cfg, params).eval()
    meg = d["meg"].cuda()
    bad = d["subject_index"].clone()
    bad[1] = cfg.n_subjects                                          # one past the last subject
    batch = synthetic.make_batch(meg, bad.cuda(), d["rec_positions"], d["rec_of_sample"])
    with torch.no_grad():
        model(dict(meg=meg), batch)
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        BF.check_tc_status()
    BF.check_tc_status()                                             # the flag is cleared once reported
    batch = synthetic.make_batch(meg, d["subject_index"].cuda(), d["rec_positions"], d["rec_of_sample"])
    with torch.no_grad():
        est = model(dict(meg=meg), batch)
    torch.cuda.synchronize()
    BF.check_tc_status()
    assert torch.isfinite(est).all()
