"""GPU parity for SURVEY 8(f) row 3: the DeepMel feature model (stand-alone ConvSequence forward/backward in CUDA) and the
candidate-side gradient of ClipLoss, against the verbatim-reference fixtures and the oracle.  Tolerance 1e-4 relative."""
import numpy as np
import pytest
import torch

from conftest import load_arrays, rel_err
from oracle import bm_oracle, deepmel_oracle
from oracle.make_golden import DEEPMEL_CASES
from brainmagick_b200 import functional as BF
from brainmagick_b200.features import DeepMel
from brainmagick_b200.losses import ClipLoss

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = "cuda"


def _check_param_grads(model, ref, tol, bn_training=True):
    wscale = max(float(np.linalg.norm(v)) for k, v in ref.items() if k.endswith("weight"))
    for name, p in model.named_parameters():
        want = torch.as_tensor(ref[name])
        assert p.grad is not None, name
        got = p.grad.detach().cpu()
        if want.norm() < 1e-5 * wscale:          # a conv bias in front of a training BatchNorm: exactly 0 up to rounding
            assert got.abs().max().item() < 1e-4 * wscale + 1e-6, name
        else:
            assert rel_err(got, want) < 5 * tol, (name, rel_err(got, want))


@pytest.mark.parametrize("case", list(DEEPMEL_CASES))
def test_deepmel_matches_reference_fixture(case):
    g = load_arrays(case)
    c = DEEPMEL_CASES[case]
    model = DeepMel(n_in_channels=c["n_in"], **c["params"])
    model.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("p.")}, strict=True)
    model = model.to(DEV).train()
    mel = torch.from_numpy(g["mel"]).to(DEV)
    est = torch.from_numpy(g["estimate"]).to(DEV).requires_grad_(True)
    cand = model(mel)
    cand.retain_grad()
    assert rel_err(cand.detach().cpu(), torch.from_numpy(g["candidates"])) < TOL
    clip = ClipLoss().to(DEV)
    loss = clip(est, cand, torch.ones(len(mel), 1, mel.shape[2], dtype=torch.bool, device=DEV))
    loss.backward()
    BF.check_tc_status()
    assert abs(loss.item() - float(g["loss"])) < TOL * max(1.0, abs(float(g["loss"])))
    assert rel_err(est.grad.cpu(), torch.from_numpy(g["g.estimate"])) < TOL
    assert rel_err(cand.grad.cpu(), torch.from_numpy(g["g.candidates"])) < TOL
    _check_param_grads(model, {k[2:]: v for k, v in g.items() if k.startswith("g.") and k[2:] not in
                               ("estimate", "candidates")}, TOL)
    sd = model.state_dict()
    for k, v in g.items():
        if k.startswith("bn."):
            got = sd[k[3:]].cpu()
            if "num_batches" in k:
                assert int(got) == int(v)
            else:
                assert rel_err(got, torch.from_numpy(v)) < TOL, k
    model.eval()
    with torch.no_grad():
        out = model(mel)
    assert rel_err(out.cpu(), torch.from_numpy(g["candidates_eval"])) < TOL


def _oracle_step(spec, params, mel, est, training=True):
    p = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in params.items()}
    e = est.clone().requires_grad_(True)
    m = mel.clone().requires_grad_(True)
    stats = {}
    cand = deepmel_oracle.conv_sequence(m, p, spec, training=training, new_stats=stats)
    cand.retain_grad()
    loss = bm_oracle.clip_loss(e, cand)
    loss.backward()
    grads = {k: v.grad for k, v in p.items() if v.grad is not None}
    return dict(cand=cand.detach(), loss=loss.detach(), d_est=e.grad, d_cand=cand.grad, d_mel=m.grad, grads=grads,
                stats=stats)


@pytest.mark.parametrize("cfg", [
    # tensor-core-eligible widths (N tiles of 160 / 256 / 320), mel channels padded 40 -> 64; input gradient requested
    dict(n_in=40, hidden=160, layers=4, out=320, B=4, T=72, act=None),
    dict(n_in=64, hidden=256, layers=3, out=256, B=3, T=130, act="gelu"),
])
def test_deepmel_tensor_core_widths_match_oracle(cfg):
    torch.manual_seed(21)
    kw = dict(kernel=3, stride=1, dilation_growth=2, dilation_period=5, batch_norm=True, activation_on_last=False,
              skip=True, glu_context=1, glu=2)
    if cfg["act"] == "gelu":
        kw["activation"] = torch.nn.GELU
    model = DeepMel(cfg["n_in"], cfg["hidden"], cfg["layers"], cfg["out"], **kw)
    with torch.no_grad():
        for mod in model.modules():
            if isinstance(mod, torch.nn.BatchNorm1d):
                mod.weight.add_(0.1 * torch.randn_like(mod.weight))
                mod.bias.add_(0.1 * torch.randn_like(mod.bias))
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    okw = {k: v for k, v in kw.items() if k not in ("stride", "activation")}
    spec = deepmel_oracle.deep_mel_spec(cfg["n_in"], cfg["hidden"], cfg["layers"], cfg["out"],
                                        activation="gelu" if cfg["act"] == "gelu" else "lrelu", **okw)
    mel = torch.randn(cfg["B"], cfg["n_in"], cfg["T"])
    est = torch.randn(cfg["B"], cfg["out"], cfg["T"])
    ref = _oracle_step(spec, params, mel, est)
    model = model.to(DEV).train()
    m = mel.to(DEV).requires_grad_(True)
    e = est.to(DEV).requires_grad_(True)
    cand = model(m)
    cand.retain_grad()
    loss = ClipLoss().to(DEV)(e, cand, torch.ones(cfg["B"], 1, cfg["T"], dtype=torch.bool, device=DEV))
    loss.backward()
    BF.check_tc_status()
    assert rel_err(cand.detach().cpu(), ref["cand"]) < TOL
    assert abs(loss.item() - ref["loss"].item()) < TOL * max(1.0, abs(ref["loss"].item()))
    assert rel_err(e.grad.cpu(), ref["d_est"]) < TOL
    assert rel_err(cand.grad.cpu(), ref["d_cand"]) < TOL
    assert rel_err(m.grad.cpu(), ref["d_mel"]) < 5 * TOL
    _check_param_grads(model, {k: v.numpy() for k, v in ref["grads"].items()}, TOL)
    sd = model.state_dict()
    for k, v in ref["stats"].items():
        assert rel_err(sd[k].cpu(), v) < TOL, k


@pytest.mark.parametrize("Bn,Bc,F,T", [(256, 256, 8, 64), (128, 320, 4, 96), (6, 20, 9, 31)])
def test_clip_candidate_gradient(Bn, Bc, F, T):
    """d loss / d candidates (and d estimate beside it) on the tensor-core shapes and on an FMA-only shape, with extra
    negatives (Bc > Bn)."""
    torch.manual_seed(3)
    est = torch.randn(Bn, F, T)
    cand = torch.randn(Bc, F, T) * 1.5
    e = est.to(DEV).requires_grad_(True)
    c = cand.to(DEV).requires_grad_(True)
    loss = BF.clip_loss(e, c, 0)
    loss.backward()
    BF.check_tc_status()
    er = est.clone().requires_grad_(True)
    cr = cand.clone().requires_grad_(True)
    ref = bm_oracle.clip_loss(er, cr, 0)
    ref.backward()
    assert abs(loss.item() - ref.item()) < TOL
    assert rel_err(e.grad.cpu(), er.grad) < TOL
    assert rel_err(c.grad.cpu(), cr.grad) < TOL
    # candidates only (the estimate is a constant): same candidate gradient, no estimate gradient computed
    c2 = cand.to(DEV).requires_grad_(True)
    BF.clip_loss(est.to(DEV), c2, 0).backward()
    assert rel_err(c2.grad.cpu(), cr.grad) < TOL


@pytest.mark.parametrize("activation", ["gelu", "lrelu"])
def test_deepmel_full_size_tensor_core_vs_fma(activation):
    """conf/feature_model/deep_mel.yaml at its real widths (120 mel -> 9 x 320 -> 768, T=360): the tensor-core path
    against the FP32-FMA path of the same library, forward and every gradient.

    With the smooth GELU the gradients agree to the usual tolerance.  The configuration's own LeakyReLU(0) has a
    discontinuous derivative: a pre-activation within rounding distance of 0 takes derivative 0 on one path and 1 on the
    other, and flipping a fraction f of the activations moves a gradient by ~sqrt(f) in relative Frobenius norm
    (f ~ 1e-5 -> a few 1e-3).  The oracle shows the same sensitivity on the CPU: a 2e-5 relative perturbation of its
    conv outputs moves the LeakyReLU(0) gradients by 1.8e-2 and the GELU gradients by 2e-4 (profiles/README.md).  So
    with LeakyReLU the forward is held to the tolerance and the gradients to a bound only a real defect would exceed."""
    torch.manual_seed(8)
    kw = dict(n_hidden_channels=320, n_hidden_layers=10, n_out_channels=768, kernel=3, stride=1, dilation_growth=2,
              dilation_period=5, batch_norm=True, activation_on_last=False, skip=True, glu_context=1, glu=2)
    if activation == "gelu":
        kw["activation"] = torch.nn.GELU
    model = DeepMel(n_in_channels=120, **kw).to(DEV).train()
    B, T = 8, 360
    mel = torch.randn(B, 120, T, device=DEV)
    gout = torch.randn(B, 768, T, device=DEV)
    results = []
    for tc in (True, False):
        model.use_tensor_cores = tc
        model.zero_grad(set_to_none=True)
        before = BF._lib.launch_count()
        out = model(mel)
        out.backward(gout)
        torch.cuda.synchronize()
        BF.check_tc_status()
        results.append((out.detach().clone(), {n: p.grad.detach().clone() for n, p in model.named_parameters()},
                        BF._lib.launch_count() - before))
    (o_tc, g_tc, n_tc), (o_fma, g_fma, n_fma) = results
    assert rel_err(o_tc, o_fma) < TOL
    wscale = max(v.norm().item() for k, v in g_fma.items() if k.endswith("weight"))
    worst, worst_name = 0.0, ""
    for name in g_fma:
        if g_fma[name].norm().item() < 1e-5 * wscale:
            assert g_tc[name].abs().max().item() < 1e-3 * wscale + 1e-6, name
            continue
        err = rel_err(g_tc[name], g_fma[name])
        if err > worst:
            worst, worst_name = err, name
    print(f"\n[deepmel] full size B={B} {activation}: forward {rel_err(o_tc, o_fma):.2e}, worst gradient {worst:.2e} "
          f"({worst_name}); {n_tc} launches (tensor cores) vs {n_fma} (fma)")
    assert worst < (5 * TOL if activation == "gelu" else 3e-2), (worst_name, worst)
