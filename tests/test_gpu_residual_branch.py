"""ConvSequence's residual-branch options on the H100: the residual-gain entry points element by element against fp64,
ConvSequence / SimpleConv with `scale`, `rewrite` and `post_skip` against an fp64 restatement of the reference layers, the
frozen-parameter, deterministic and TF32 contracts, and the SimpleConv fixture of the verbatim reference."""
import contextlib

import pytest
import torch

import brainmagick_b200.functional as BF
from brainmagick_b200._lib import call, ptr, stream
from conftest import load_arrays, rel_err
from test_residual_branch_cpu import seq_oracle
from tools.make_residual_golden import SIMPLECONV_CASE

pytestmark = pytest.mark.gpu
DEV = "cuda"
GELU, LRELU, NONE = 0, 1, 2


def _act64(act, z, slope):
    if act == GELU:
        return torch.nn.functional.gelu(z)
    return torch.where(z > 0, z, z * slope) if act == LRELU else z


def _gain_ref(y, g, bn, act, slope, scale, post, x_old, train, boost=5.0):
    """fp64 autograd of x_new = post * ((boost*scale) * act(bn(y))) + x_old -> (x_new, dy, dgamma, dbeta, dscale, dpost)."""
    d = lambda t: None if t is None else t.double().detach().requires_grad_(True)   # noqa: E731
    y64, s64, p64 = d(y), d(scale), d(post)
    z = y64
    gm = bt = None
    if bn is not None:
        mean, invstd, gamma, beta = bn
        gm, bt = d(gamma), d(beta)
        if train:
            mu = y64.mean(0)
            yh = (y64 - mu) / torch.sqrt(((y64 - mu) ** 2).mean(0) + 1e-5)
        else:
            yh = (y64 - mean.double()) * invstd.double()
        z = yh * gm + bt
    a = _act64(act, z, slope)
    if s64 is not None:
        a = (boost * s64) * a
    if p64 is not None:
        a = p64 * a
    out = a + (x_old.double() if x_old is not None else 0.0)
    out.backward(g.double())
    grad = lambda t: None if t is None else t.grad   # noqa: E731
    return out.detach(), y64.grad, grad(gm), grad(bt), grad(s64), grad(p64)


def _close(got, ref, what):
    ref = ref.to(got.device)
    assert rel_err(got, ref) < 1e-4, (what, rel_err(got, ref))
    assert (got.double() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item() + 1e-12, what


@pytest.mark.parametrize("C,rows", [(320, 1000), (10, 777)])
@pytest.mark.parametrize("mode", ["bn_train", "bn_eval", "no_bn"])
@pytest.mark.parametrize("act", [GELU, LRELU, NONE])
@pytest.mark.parametrize("gains", ["scale", "post", "both", "none"])
@pytest.mark.parametrize("det", [False, True])
def test_gain_entry_points_against_fp64(C, rows, mode, act, gains, det):
    """gains "none": scale and post NULL (gain 1) with dscale and dpost asked for: dpost = S, dscale = boost * S."""
    gen = torch.Generator(device=DEV).manual_seed(C + rows)
    r = lambda *s: torch.randn(*s, device=DEV, generator=gen)   # noqa: E731
    y, g, x_old = r(rows, C) * 2 + 0.5, r(rows, C), r(rows, C)
    scale = 0.02 * (1 + r(C)) if gains in ("scale", "both") else None
    post = r(C) if gains in ("post", "both") else None
    slope = 0.07
    bn, train = None, mode == "bn_train"
    mean = invstd = gamma = beta = None
    if mode != "no_bn":
        gamma, beta = 1 + 0.1 * r(C), 0.1 * r(C)
        if train:
            m64 = y.double().mean(0)
            mean, invstd = m64.float(), (1 / torch.sqrt(y.double().var(0, unbiased=False) + 1e-5)).float()
        else:
            mean, invstd = 0.3 * r(C), 1 / (1 + r(C).abs())
        bn = (mean, invstd, gamma, beta)
    ref_post = torch.ones(C, device=DEV) if gains == "none" else post
    ref = _gain_ref(y, g, bn, act, slope, scale, ref_post, x_old, train)
    if gains == "none":                     # the reference's post = 1 gives S as its gradient
        ref = ref[:4] + (5.0 * ref[5], ref[5])
    st = stream()
    x_new = torch.empty_like(y)
    call("bm_bn_act_gain_skip_fwd", ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(x_old), ptr(x_new), rows, C,
         act, slope, ptr(scale), 5.0, ptr(post), st)
    _close(x_new, ref[0], "x_new")
    outs = [torch.empty_like(y)] + [torch.empty(C, device=DEV) if t is not None else None for t in ref[2:]]
    sums = torch.full((3 * C,), float("nan"), device=DEV, dtype=torch.float64)
    args = [ptr(g), ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), int(train), rows, C, act, slope, ptr(scale), 5.0,
            ptr(post), ptr(sums)] + [ptr(t) for t in outs]

    def run():
        if not det:
            call("bm_bn_act_gain_skip_bwd", *args, st)
            return
        n = BF._lib.load().bm_bn_act_gain_skip_bwd_det_workspace(rows, C)
        ws = torch.full((n,), float("nan"), device=DEV)
        call("bm_bn_act_gain_skip_bwd_det", *args, ptr(ws), n, st)
    run()
    for got, want, name in zip(outs, ref[1:], ("dy", "dgamma", "dbeta", "dscale", "dpost")):
        if want is not None:
            _close(got, want.reshape(got.shape), name)
    if det:                                 # the deterministic form repeats bitwise
        first = [t.clone() for t in outs if t is not None]
        run()
        assert all(torch.equal(a, b) for a, b in zip(first, [t for t in outs if t is not None]))


@pytest.mark.parametrize("C,rows", [(320, 1000), (10, 777)])
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("det", [False, True])
def test_epilogue_entry_points_agree_bitwise(C, rows, train, det):
    """Where their contracts overlap -- BatchNorm + GELU without gains -- bm_bn_gelu_skip_*, bm_bn_act_skip_*(GELU) and
    bm_bn_act_gain_skip_* with NULL gains run one layer epilogue: the same bits forward and backward, at a column-stationary
    width (320) and a generic one (10)."""
    gen = torch.Generator(device=DEV).manual_seed(C + rows + train)
    r = lambda *s: torch.randn(*s, device=DEV, generator=gen)   # noqa: E731
    y, g, x_old = r(rows, C) * 2 + 0.5, r(rows, C), r(rows, C)
    mean, invstd, gamma, beta = 0.3 * r(C), 1 / (1 + r(C).abs()), 1 + 0.1 * r(C), 0.1 * r(C)
    st = stream()
    bn = [ptr(mean), ptr(invstd), ptr(gamma), ptr(beta)]
    fwd = {"bm_bn_gelu_skip_fwd": [None], "bm_bn_act_skip_fwd": [GELU, 0.0],
           "bm_bn_act_gain_skip_fwd": [GELU, 0.0, None, 5.0, None]}
    bwd = {"bm_bn_gelu_skip_bwd": ([], [None]), "bm_bn_act_skip_bwd": ([GELU, 0.0], []),
           "bm_bn_act_gain_skip_bwd": ([GELU, 0.0, None, 5.0, None], [None, None])}
    results = []
    for (fname, fextra), (bname, (act_args, tail)) in zip(fwd.items(), bwd.items()):
        x_new, dy = torch.empty_like(y), torch.empty_like(y)
        dgamma, dbeta = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
        call(fname, ptr(y), *bn, ptr(x_old), ptr(x_new), rows, C, *fextra, st)
        sums = torch.empty(3 * C, device=DEV, dtype=torch.float64)
        args = [ptr(g), ptr(y), *bn, int(train), rows, C, *act_args, ptr(sums), ptr(dy), ptr(dgamma), ptr(dbeta), *tail]
        if det:
            n = getattr(BF._lib.load(), bname + "_det_workspace")(rows, C)
            ws = torch.full((n,), float("nan"), device=DEV)
            call(bname + "_det", *args, ptr(ws), n, st)
        else:
            call(bname, *args, st)
        results.append((x_new, dy, dgamma, dbeta))
    for other in results[1:]:
        for a, b, what in zip(results[0], other, ("x_new", "dy", "dgamma", "dbeta")):
            assert torch.equal(a, b), what


# ---- module level ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _spy(monkeypatch):
    names = []
    real = BF.call

    def spy(name, *args):
        names.append(name)
        return real(name, *args)
    monkeypatch.setattr(BF, "call", spy)
    import brainmagick_b200.convseq as CS
    monkeypatch.setattr(CS, "call", spy)
    yield names


OPTIONS = {"scale": dict(scale=0.1), "rewrite": dict(rewrite=True), "post_skip": dict(post_skip=True),
           "all": dict(scale=0.1, rewrite=True, post_skip=True)}
ACTS = {"gelu_bn": dict(activation="gelu", batch_norm=True), "leaky_bn": dict(activation=None, batch_norm=True),
        "leaky_nobn": dict(activation=None, batch_norm=False)}


def _seq_case(width, option, acts, bare_last=False):
    c = dict(channels=[width] * 4, kernel=3, dilation_growth=2, skip=True, leakiness=0.1, **OPTIONS[option], **ACTS[acts])
    if bare_last:
        c["activation_on_last"] = False
    return c


def _build(c, seed=0):
    from brainmagick_b200.common import ConvSequence
    from tools.make_residual_golden import seq_kwargs
    torch.manual_seed(seed)
    model = ConvSequence(c["channels"], **seq_kwargs(dict(c, B=0, T=0, seed=0))).to(DEV)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.add_(0.1 * torch.randn_like(m.weight))
                m.bias.add_(0.1 * torch.randn_like(m.bias))
            if type(m).__name__ == "LayerScale":
                m.scale.mul_(1 + 0.5 * torch.randn_like(m.scale))
    return model


def _module_check(c, train, monkeypatch, B=2, T=50, tol=1e-4):
    model = _build(c).train(train)
    p = {k: v.detach().double().clone().requires_grad_(v.dtype == torch.float32 and "running" not in k
                                                        and "num_batches" not in k)
         for k, v in model.state_dict().items()}
    x = torch.randn(B, c["channels"][0], T, device=DEV)
    w = torch.randn(B, c["channels"][-1], T, device=DEV)
    x64 = x.double().requires_grad_(True)
    ref = seq_oracle(x64, p, c, train)
    (ref * w.double()).sum().backward()
    xg = x.clone().requires_grad_(True)
    with _spy(monkeypatch) as names:
        out = model(xg)
        (out * w).sum().backward()
        torch.cuda.synchronize()
    BF.check_tc_status()
    assert rel_err(out.detach(), ref.detach()) < tol
    assert rel_err(xg.grad, x64.grad) < tol
    for k, v in model.named_parameters():
        want = p[k].grad
        if want.norm() < 1e-6 * max(1.0, want.numel() ** 0.5):    # conv bias in front of a training BatchNorm
            assert v.grad.abs().max() < 1e-4, k
        else:
            assert rel_err(v.grad, want) < tol, (k, rel_err(v.grad, want))
    return names


@pytest.mark.parametrize("width", [8, 320])
@pytest.mark.parametrize("option", list(OPTIONS))
@pytest.mark.parametrize("acts", list(ACTS))
@pytest.mark.parametrize("train", [True, False])
def test_convsequence_options_against_fp64(width, option, acts, train, monkeypatch):
    names = _module_check(_seq_case(width, option, acts), train, monkeypatch)
    gains = option in ("scale", "post_skip", "all")
    assert ("bm_bn_act_gain_skip_fwd" in names) == gains
    assert ("bm_bn_act_gain_skip_bwd" in names) == gains
    tc = any(n.startswith("bm_tc_conv1d") for n in names)
    assert tc == (width == 320)                                 # tensor-core convolutions at 320, FP32-FMA at 8


@pytest.mark.parametrize("width", [8, 320])
@pytest.mark.parametrize("train", [True, False])
def test_bare_last_layer_against_fp64(width, train, monkeypatch):
    names = _module_check(_seq_case(width, "all", "gelu_bn", bare_last=True), train, monkeypatch)
    assert names.count("bm_bn_act_gain_skip_fwd") == 3        # every layer keeps its width: all three carry the gains


@pytest.mark.parametrize("frozen", ["gains", "rewrite"])
def test_frozen_options_skip_their_gradients(frozen, monkeypatch):
    c = _seq_case(320, "all", "gelu_bn")
    model = _build(c).train()
    x = torch.randn(2, 320, 40, device=DEV)
    for name, prm in model.named_parameters():
        index = name.split(".")[-2]                 # sequence.k.{0 conv, 1 bn, 3 rewrite, 5 LayerScale, 6 post_skip}
        is_gain, is_rewrite = index in ("5", "6"), index == "3"
        if (frozen == "gains" and is_gain) or (frozen == "rewrite" and is_rewrite):
            prm.requires_grad_(False)
    with _spy(monkeypatch) as names:
        model(x).sum().backward()
        torch.cuda.synchronize()
    for name, prm in model.named_parameters():
        assert (prm.grad is None) == (not prm.requires_grad), name
    wgrads = sum(n.startswith(("bm_tc_wgrad", "bm_conv1d_bwd_weight")) for n in names)
    if frozen == "rewrite":
        assert wgrads == 3                                      # the three layer convolutions only
    else:
        assert wgrads == 6
        assert "bm_bn_act_gain_skip_bwd" in names               # the rewrite's LeakyReLU backward still runs through it


def test_deterministic_repeats_bitwise():
    c = _seq_case(320, "all", "gelu_bn")
    x = torch.randn(2, 320, 40, device=DEV)
    results = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            model = _build(c).train()
            out = model(x)
            out.square().sum().backward()
            results.append([out.detach()] + [p.grad for p in model.parameters()])
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(a, b) for a, b in zip(*results))


@pytest.mark.parametrize("train", [True, False])
def test_tf32_subset(train, monkeypatch):
    """Single-pass TF32 contractions (10-bit mantissa operands) through 3 layers of conv + 1x1 rewrite: within TF32's error
    of fp64 (a training BatchNorm over 100 rows amplifies it in the first layer's weight gradient), and the _tf32 forms ran."""
    prev = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        names = _module_check(_seq_case(320, "all", "gelu_bn"), train, monkeypatch, tol=5e-2)
    finally:
        torch.backends.cuda.matmul.fp32_precision = prev
    assert any(n.startswith("bm_tc_") and n.endswith("_tf32") for n in names)


def test_simpleconv_fixture_with_meg_gradient():
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle.ref_loader import clip_conv_kwargs
    c = SIMPLECONV_CASE
    g = {k: torch.from_numpy(v) for k, v in load_arrays("residual_simpleconv").items()}
    kw = clip_conv_kwargs(hidden=c["hidden"], depth=c["depth"], merger_channels=c["MC"], initial_linear=c["IL"],
                          merger_pos_dim=c["P"])
    kw.update(c["extra"])
    model = bb.SimpleConv(in_channels=dict(meg=c["C"]), out_channels=c["F"], n_subjects=c["S"], **kw)
    model.load_state_dict({k[2:]: v for k, v in g.items() if k.startswith("p.")}, strict=True)
    model = model.to(DEV).train()
    model.merger.ban_centre_override = g["ban_centre"]
    subj = g["subject_index"]
    meg = g["meg"].to(DEV).requires_grad_(True)
    batch = synthetic.make_batch(meg.detach(), subj, g["rec_positions"], subj)
    est = model(dict(meg=meg), batch)
    loss = bb.ClipLoss()(est, g["candidates"].to(DEV), torch.ones(len(meg), 1, meg.shape[2], dtype=torch.bool, device=DEV))
    loss.backward()
    assert rel_err(est.detach().cpu(), g["estimate"]) < 1e-4
    assert abs(loss.item() - float(g["loss"])) < 1e-4
    assert rel_err(meg.grad.cpu(), g["g.meg"]) < 1e-4
    for k, v in model.named_parameters():
        ref = g["g." + k]
        if ref.norm() < 1e-5:
            assert v.grad.abs().max() < 1e-4, k
        else:
            assert rel_err(v.grad.cpu(), ref) < 1e-4, k
