"""torch.use_deterministic_algorithms(True) on the GPU: repeated training steps are bitwise identical, also while an unrelated
workload on another stream changes the order in which blocks finish, and the deterministic forms still match the fp64
oracle and the default forms."""
import random

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _busy_side_stream():
    """An unrelated long elementwise workload (no cuBLAS) on another stream, enqueued just before a step: the step's blocks
    share the SMs with it and finish in another order than in an idle run."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        x = torch.ones(1 << 26, device="cuda")           # not torch.rand: the step's own random draws must not move
        for _ in range(60):
            x.mul_(0.999).add_(1e-3)
    return side, x


def _train(kw, C, T, B, F, S, n_valid=(), steps=3, meg_grad=False, perturb=False, deepmel=None, eval_forward=False):
    """`steps` Adam steps of SimpleConv + ClipLoss from a fixed seed -> every output of every step, and the state after them."""
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, synthetic
    torch.manual_seed(0)
    random.seed(0)
    model = bb.SimpleConv(in_channels=dict(meg=C), out_channels=F, n_subjects=S, **kw).cuda().train()
    params = list(model.parameters())
    feat = None
    if deepmel is not None:
        feat = bb.DeepMel(n_in_channels=deepmel["n_in"], **dict(deepmel["params"], n_out_channels=F)).cuda().train()
        params += list(feat.parameters())
    opt = torch.optim.Adam(params, lr=1e-3)
    clip = bb.ClipLoss().cuda().train()
    gen = torch.Generator().manual_seed(1)
    pos = synthetic.normalised_positions(S, C, n_valid, seed=4)
    mask = torch.ones(B, 1, T, dtype=torch.bool, device="cuda")
    out = []
    for _ in range(steps):
        meg = torch.randn(B, C, T, generator=gen).cuda().requires_grad_(meg_grad)
        subj = torch.randint(0, S, (B,), generator=gen)
        batch = synthetic.make_batch(meg, subj.cuda(), pos, subj)
        if deepmel is None:
            cand = torch.randn(B, F, T, generator=gen).cuda()
        else:
            cand = feat(torch.randn(B, deepmel["n_in"], T, generator=gen).cuda())
        side = _busy_side_stream() if perturb else None
        opt.zero_grad(set_to_none=True)
        est = model(dict(meg=meg), batch)
        loss = clip(est, cand, mask)
        loss.backward()
        rec = dict(est=est.detach().clone(), loss=loss.detach().clone())
        rec.update({"grad." + n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None})
        if feat is not None:
            rec.update({"feat.grad." + n: p.grad.clone() for n, p in feat.named_parameters() if p.grad is not None})
        if meg_grad:
            rec["meg.grad"] = meg.grad.clone()
        opt.step()
        if side is not None:
            torch.cuda.current_stream().wait_stream(side[0])
        out.append(rec)
    state = {k: v.clone() for k, v in model.state_dict().items()}          # parameters and BatchNorm running statistics
    if feat is not None:
        state.update({"feat." + k: v.clone() for k, v in feat.state_dict().items()})
    out.append(state)
    if eval_forward:
        model.eval()
        with torch.no_grad():
            out.append(dict(eval=model(dict(meg=meg.detach()), batch)))
    torch.cuda.synchronize()
    BF.check_tc_status()
    return out


def _assert_bitwise(a, b):
    assert len(a) == len(b)
    for i, (ra, rb) in enumerate(zip(a, b)):
        assert ra.keys() == rb.keys()
        for k in ra:
            if ra[k].is_floating_point():
                assert torch.isfinite(ra[k]).all(), (i, k)
            assert torch.equal(ra[k], rb[k]), (i, k, (ra[k].double() - rb[k].double()).abs().max().item())


def _clip_conv(hidden=320, MC=270, IL=270, P=2048, **change):
    kw = dict(hidden=dict(meg=hidden), depth=10, dilation_period=5, kernel_size=3, skip=True, subject_layers=True,
              subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=IL, merger_channels=MC,
              gelu=True, batch_norm=True, merger_pos_dim=P, merger_dropout=0.2)
    kw.update(change)
    return kw


SMALL = dict(hidden=16, MC=12, IL=12, P=32)                  # the FP32-FMA kernels
CASES = {
    "baseline_C208_T360": (_clip_conv(), dict(C=208, T=360, B=64, F=1024, S=27)),
    "baseline_mixed_T343": (_clip_conv(), dict(C=273, T=343, B=64, F=1024, S=8, n_valid=(273, 208, 128, 60))),
    "small_fp32_fma": (_clip_conv(**SMALL), dict(C=10, T=24, B=6, F=8, S=3)),
    "no_merger": (_clip_conv(merger=False), dict(C=208, T=360, B=16, F=1024, S=4)),
    "no_initial_linear": (_clip_conv(initial_linear=0), dict(C=208, T=360, B=16, F=1024, S=4)),
    "no_subject_layers_subject_dim": (_clip_conv(subject_layers=False, subject_dim=16), dict(C=208, T=360, B=16, F=1024, S=4)),
    "subsample_channels": (_clip_conv(subsample_meg_channels=150), dict(C=208, T=360, B=16, F=1024, S=4)),
    "small_no_merger": (_clip_conv(merger=False, **SMALL), dict(C=10, T=24, B=6, F=8, S=3)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_repeated_steps_are_bitwise_identical(case, deterministic):
    kw, dims = CASES[case]
    first = _train(kw, **dims, eval_forward=True)
    second = _train(kw, **dims, perturb=True, eval_forward=True)
    _assert_bitwise(first, second)


@pytest.mark.parametrize("case", ["baseline_C208_T360", "small_fp32_fma"])
def test_meg_grad_is_bitwise_identical(case, deterministic):
    kw, dims = CASES[case]
    _assert_bitwise(_train(kw, **dims, meg_grad=True), _train(kw, **dims, meg_grad=True, perturb=True))


@pytest.mark.parametrize("T,F", [(360, 120), (24, 8)])
def test_deepmel_candidates_are_bitwise_identical(T, F, deterministic):
    from oracle.make_golden import DEEPMEL_CASES
    dm = DEEPMEL_CASES["deepmel_small"]
    kw, dims = CASES["baseline_C208_T360" if T == 360 else "small_fp32_fma"]
    dims = dict(dims, F=F, B=min(dims["B"], 16))
    _assert_bitwise(_train(kw, **dims, deepmel=dm), _train(kw, **dims, deepmel=dm, perturb=True))


@pytest.mark.parametrize("idx", [0, 3])
def test_baseline_shapes_match_oracle_deterministically(idx, deterministic):
    import test_gpu_parity
    test_gpu_parity.test_baseline_shapes_match_oracle(test_gpu_parity.BASELINE_SHAPES[idx])


def test_accuracy_recipe_trains_bitwise_identically(deterministic):
    """The same-recipe leg of test_gpu_zy_accuracy, first 64 Adam steps, twice: identical losses and weights."""
    import json
    import os
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    from oracle import make_accuracy_golden as mg
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "accuracy_full_width.json")
    with open(path) as f:
        spec = json.load(f)["spec"]
    cfg, task, sched, p0 = mg.build(spec)
    recs = [synthetic.SyntheticRecording(s, task["positions"][s]) for s in range(cfg.n_subjects)]
    d = task["train"]
    mask = torch.ones(spec["batch"], 1, spec["T"], dtype=torch.bool, device="cuda")

    def run(perturb):
        model = bb.SimpleConv(
            in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden),
            depth=cfg.depth, dilation_period=5, kernel_size=3, skip=True, subject_layers=True, subject_dim=0,
            complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=cfg.initial_linear,
            merger_channels=cfg.merger_channels, gelu=True, batch_norm=True, merger_pos_dim=cfg.merger_pos_dim,
            n_subjects=cfg.n_subjects)
        model.load_state_dict(p0)
        model = model.cuda().train()
        clip = bb.ClipLoss().cuda().train()
        opt = torch.optim.Adam(model.parameters(), lr=spec["lr"], betas=(0.9, 0.999))
        losses = []
        for step, (idx, ban) in enumerate(sched[:64]):
            meg, feats = d["meg"][idx].cuda(), d["feats"][idx].cuda()
            batch = synthetic.SyntheticBatch(meg, d["subj"][idx].cuda(), [recs[int(s)] for s in d["subj"][idx]])
            model.merger.ban_centre_override = ban
            side = _busy_side_stream() if perturb and step % 8 == 0 else None
            opt.zero_grad(set_to_none=True)
            loss = clip(model(dict(meg=meg), batch), feats, mask)
            loss.backward()
            opt.step()
            if side is not None:
                torch.cuda.current_stream().wait_stream(side[0])
            losses.append(loss.detach())
        return torch.stack(losses), {k: v.clone() for k, v in model.state_dict().items()}

    (l1, s1), (l2, s2) = run(False), run(True)
    assert torch.isfinite(l1).all() and torch.equal(l1, l2)
    for k in s1:
        assert torch.equal(s1[k], s2[k]), k


# ---- the deterministic entry points at their edges: against fp64 and the default forms, and repeated bitwise -------------
def _call(name, *args):
    from brainmagick_b200._lib import call, stream
    call(name, *args, stream())


def _ws(name, *dims):
    from brainmagick_b200 import _lib
    n = int(getattr(_lib.load(), name + "_workspace")(*dims))
    return torch.empty(max(n, 2), device="cuda")


@pytest.mark.parametrize("rows,C", [(1, 7), (343, 320), (16 * 343 + 5, 1024), (97, 33)])
def test_column_reductions_against_fp64(rows, C):
    from brainmagick_b200._lib import ptr
    torch.manual_seed(rows + C)
    y = torch.randn(rows, C, device="cuda") + 0.5
    y64 = y.double()
    for _ in range(2):
        ws = _ws("bm_col_stats_det", rows, C)
        stats = torch.full((2 * C,), float("nan"), device="cuda", dtype=torch.float64)
        _call("bm_col_stats_det", ptr(y), rows, C, ptr(ws), ws.numel(), ptr(stats))
        want = torch.cat([y64.sum(0), (y64 * y64).sum(0)])
        assert rel_err(stats.cpu(), want.cpu()) < 1e-6
        ws = _ws("bm_col_sum_det", rows, C)
        out = torch.full((C,), float("nan"), device="cuda")
        _call("bm_col_sum_det", ptr(y), rows, C, ptr(ws), ws.numel(), ptr(out))
        assert rel_err(out.double().cpu(), y64.sum(0).cpu()) < 1e-5
        if _ == 0:
            first = (stats.clone(), out.clone())
    assert torch.equal(first[0], stats) and torch.equal(first[1], out)


@pytest.mark.parametrize("rows,C", [(1, 8), (343, 320), (16 * 343 + 5, 320), (97, 33)])
def test_batchnorm_backward_reduce_matches_default_form(rows, C):
    from brainmagick_b200._lib import ptr
    torch.manual_seed(C)
    g, y = torch.randn(rows, C, device="cuda"), torch.randn(rows, C, device="cuda")
    mean, invstd = y.mean(0), 1.0 / (y.var(0, unbiased=False) + 1e-5).sqrt()
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.1
    res = {}
    for form in ("bm_bn_gelu_skip_bwd", "bm_bn_gelu_skip_bwd_det", "bm_bn_act_skip_bwd", "bm_bn_act_skip_bwd_det"):
        sums = torch.empty(2 * C, device="cuda", dtype=torch.float64)
        dy, dg, db = torch.empty_like(g), torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        extra = []
        if form.endswith("_det"):
            ws = _ws(form, rows, C)
            extra = [ptr(ws), ws.numel()]
        head = [ptr(g), ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), 1, rows, C]
        if "gelu" in form:
            _call(form, *head, ptr(sums), ptr(dy), ptr(dg), ptr(db), None, *extra)
        else:
            _call(form, *head, 1, 0.1, ptr(sums), ptr(dy), ptr(dg), ptr(db), *extra)
        res[form] = (sums.clone(), dy.clone())
    for base in ("bm_bn_gelu_skip_bwd", "bm_bn_act_skip_bwd"):
        (s0, d0), (s1, d1) = res[base], res[base + "_det"]
        assert rel_err(s1.cpu(), s0.cpu()) < 1e-6 and rel_err(d1.cpu(), d0.cpu()) < 1e-5, base


@pytest.mark.parametrize("rows,H", [(1, 80), (343, 160), (16 * 343 + 5, 80), (97, 7)])
def test_glu_backward_bias_matches_fp64(rows, H):
    from brainmagick_b200._lib import ptr
    torch.manual_seed(H)
    g, h = torch.randn(rows, H, device="cuda"), torch.randn(rows, 2 * H, device="cuda")
    dh, db = torch.empty(rows, 2 * H, device="cuda"), torch.full((2 * H,), float("nan"), device="cuda")
    ws = _ws("bm_glu_bwd_det", rows, H)
    _call("bm_glu_bwd_det", ptr(g), ptr(h), rows, H, ptr(dh), ptr(db), None, ptr(ws), ws.numel())
    assert rel_err(db.double().cpu(), dh.double().sum(0).cpu()) < 1e-5


@pytest.mark.parametrize("Bc,KT", [(1, 20), (7, 343 * 120), (256, 1024 * 360)])
def test_candidate_norms_against_fp64(Bc, KT):
    from brainmagick_b200._lib import ptr
    c = torch.randn(Bc, KT, device="cuda")
    ss, inv = torch.empty(Bc, device="cuda", dtype=torch.float64), torch.empty(Bc, device="cuda")
    _call("bm_candidate_inv_norms_det", ptr(c), Bc, KT, ptr(ss), ptr(inv))
    want = 1.0 / (1e-8 + c.double().norm(dim=1))
    assert rel_err(inv.double().cpu(), want.cpu()) < 1e-6


@pytest.mark.parametrize("B,T,Cin,Cout", [(1, 1, 5, 3), (3, 343, 16, 33), (8, 24, 16, 16)])
def test_fp32_fma_weight_gradients_match_default_form(B, T, Cin, Cout):
    from brainmagick_b200._lib import ptr
    torch.manual_seed(B * T)
    dy, x = torch.randn(B, T, Cout, device="cuda"), torch.randn(B, T, Cin, device="cuda")
    out = {}
    for form in ("bm_conv1d_bwd_weight", "bm_conv1d_bwd_weight_det"):
        dw, db = torch.empty(Cout, Cin, 3, device="cuda"), torch.empty(Cout, device="cuda")
        extra = []
        if form.endswith("_det"):
            ws = _ws(form, B, T, Cin, Cout, 3)
            extra = [ptr(ws), ws.numel()]
        _call(form, ptr(dy), ptr(x), B, T, Cin, Cout, 3, 2, ptr(dw), ptr(db), *extra)
        out[form] = (dw, db)
    (w0, b0), (w1, b1) = out["bm_conv1d_bwd_weight"], out["bm_conv1d_bwd_weight_det"]
    assert rel_err(w1.cpu(), w0.cpu()) < 1e-5 and rel_err(b1.double().cpu(), dy.double().sum((0, 1)).cpu()) < 1e-5
    H, F = Cin, Cout                       # the head: dest [B,F,T], x [B,T,H], h1 = q [B,T,2H]
    dest, h1 = torch.randn(B, F, T, device="cuda"), torch.randn(B, T, 2 * H, device="cuda")
    res = {}
    for form in ("bm_head_bwd_params", "bm_head_bwd_params_det"):
        dq = torch.randn(B, T, 2 * H, device="cuda", generator=torch.Generator("cuda").manual_seed(5))
        grads = [torch.empty(2 * H, H, device="cuda"), torch.empty(2 * H, device="cuda"), torch.empty(2 * H, F, device="cuda"),
                 torch.empty(F, device="cuda")]
        extra = []
        if form.endswith("_det"):
            ws = _ws(form, B, T, H, F)
            extra = [ptr(ws), ws.numel()]
        _call(form, ptr(dest), ptr(x), ptr(h1), ptr(h1), B, T, H, F, ptr(dq), *[ptr(t) for t in grads], *extra)
        res[form] = grads
    for a, b in zip(res["bm_head_bwd_params"], res["bm_head_bwd_params_det"]):
        assert rel_err(b.cpu(), a.cpu()) < 1e-5
