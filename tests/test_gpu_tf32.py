"""PyTorch's TF32 matmul precision on the GPU: every `_tf32` entry point against an fp64 contraction of its tf32-rounded
operands, the BASELINE shapes against the fp64 oracle at the accuracy PyTorch's own TF32 ops reach, retrieval accuracy, and
the composition with torch.use_deterministic_algorithms."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-5          # relative Frobenius error against fp64 on the rounded operands: only fp32 accumulation remains


def rna(t):
    """fp32 -> nearest tf32 (ties away from zero), as fp32: cvt.rna.tf32.f32."""
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


@contextlib.contextmanager
def precision(tf32: bool):
    """PyTorch's float32 matmul precision set to TF32 (or left at "highest"), both forms of the flag restored after."""
    m = torch.backends.cuda.matmul
    saved_new, saved_legacy = m.fp32_precision, torch.get_float32_matmul_precision()
    try:
        torch.set_float32_matmul_precision("high" if tf32 else "highest")
        yield
    finally:
        torch.set_float32_matmul_precision(saved_legacy)
        m.fp32_precision = saved_new


@contextlib.contextmanager
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _call(name, *args):
    from brainmagick_b200._lib import call, stream
    call(name, *args, stream())


def _ptr(t):
    from brainmagick_b200._lib import ptr
    return ptr(t)


def _status():
    return torch.zeros(1, dtype=torch.int32, device="cuda")


def _both(fn):
    """fn(suffix) for the TF32 form and the default form -> (tf32 outputs, default outputs), checking the status word."""
    out = []
    for suffix in ("_tf32", ""):
        st = _status()
        res = fn(suffix, st)
        torch.cuda.synchronize()
        assert int(st.item()) == 0
        out.append([r.clone() for r in res])
    return out


def _check(got, want, default):
    """got (TF32 form) within TOL of the fp64 contraction `want`, and not the default form's bits."""
    e = rel_err(got.double().cpu(), want.cpu())
    assert e < TOL, e
    assert not torch.equal(got, default)
    return e


# ---- (a) every _tf32 entry point at its edges ---------------------------------------------------------------------------
CONV_CASES = [  # B, T, Cin, Ntot, Kw, dilation, sign, glu
    (1, 1, 32, 320, 3, 1, 1, 0),          # one row
    (3, 343, 320, 320, 3, 4, 1, 0),       # 160-wide tiles, a partial time tile
    (2, 200, 64, 1024, 1, 1, 1, 0),       # 128-wide tiles
    (2, 343, 320, 640, 3, 1, 1, 1),       # GLU (80 'a' columns per tile)
    (3, 129, 320, 320, 3, 2, -1, 0),      # data-gradient taps
]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("form", ["persistent", "presplit"])
def test_conv_tf32_against_fp64(case, form):
    B, T, Cin, Ntot, Kw, dil, sign, glu = case
    torch.manual_seed(B * T + Ntot)
    x = torch.randn(B, T, Cin, device="cuda")
    w = torch.randn(Ntot, Cin, Kw, device="cuda") / (Cin * Kw) ** 0.5
    bias = torch.randn(Ntot, device="cuda")
    hi, lo = torch.empty(Kw, Ntot, Cin, device="cuda"), torch.empty(Kw, Ntot, Cin, device="cuda")
    raw = torch.empty(Kw, Ntot, Cin, device="cuda")
    _call("bm_tc_weight_split", _ptr(w), Ntot, Cin, Kw, _ptr(hi), _ptr(lo), None, None)
    _call("bm_tc_weight_split", _ptr(w), Ntot, Cin, Kw, _ptr(raw), None, None, None)
    if form == "presplit" and glu:
        pytest.skip("the pre-split entry point's GLU epilogue is covered by the persistent one")

    def run(suffix, st):
        y = torch.full((B, T, Ntot), float("nan"), device="cuda")
        g = torch.empty(B, T, Ntot // 2, device="cuda") if glu else None
        if form == "persistent":
            _call("bm_tc_conv1d_persistent" + suffix, _ptr(x), _ptr(raw), _ptr(bias), 0, B, T, Cin, Ntot, Kw, dil, sign, glu,
                  0, 0, _ptr(y), None, _ptr(g), None, _ptr(st))
        else:          # the TF32 form reads w_hi alone: w_lo = NULL
            _call("bm_tc_conv1d" + suffix, _ptr(x), _ptr(hi), None if suffix else _ptr(lo), _ptr(bias), None, B, T, Cin,
                  Ntot, Kw, dil, sign, glu, 0, 0, _ptr(y), None, _ptr(g), None, _ptr(st))
        return [y]
    (y,), (y3,) = _both(run)
    wt = rna(w).double()
    if sign < 0:
        wt = wt.flip(2)
    want = F.conv1d(rna(x).double().transpose(1, 2), wt, bias.double(), padding=dil * (Kw // 2), dilation=dil).transpose(1, 2)
    _check(y, want, y3)


def test_pointwise_sel_and_sensor_mix_bwd_tf32_against_fp64():
    S, B, T, Cin, Ntot = 3, 5, 343, 320, 320
    torch.manual_seed(1)
    x, w = torch.randn(B, T, Cin, device="cuda"), torch.randn(S, Ntot, Cin, device="cuda")
    wsel = torch.tensor([2, 0, 1, 2, 2], dtype=torch.int32, device="cuda")

    def run(suffix, st):
        y = torch.empty(B, T, Ntot, device="cuda")
        lo = None if suffix else torch.zeros_like(w)      # w exact in the 3xTF32 form: lo = 0 (hi = w is not split)
        _call("bm_tc_pointwise_sel" + suffix, _ptr(x), _ptr(w), _ptr(lo), _ptr(wsel), S, B, T, Cin, Ntot, _ptr(y), _ptr(st))
        return [y]
    (y,), (y3,) = _both(run)
    want = torch.einsum("btk,bnk->btn", rna(x).double(), rna(w).double()[wsel.long()])
    _check(y, want, y3)

    Op, Cp, C = 320, 256, 201                           # odd live sensor count
    du, wt = torch.randn(B, T, Op, device="cuda"), torch.randn(S, Cp, Op, device="cuda")
    mask = (torch.rand(C, device="cuda") > 0.2).float()

    def run2(suffix, st):
        dmeg = torch.empty(B, C, T, device="cuda")
        lo = None if suffix else torch.zeros_like(wt)
        _call("bm_tc_sensor_mix_bwd_data" + suffix, _ptr(du), _ptr(wt), _ptr(lo), _ptr(wsel), S, _ptr(mask), B, T, Op, Cp,
              C, _ptr(dmeg), _ptr(st))
        return [dmeg]
    (d,), (d3,) = _both(run2)
    want = torch.einsum("bto,bco->bct", rna(du).double(), rna(wt).double()[wsel.long(), :C]) * mask.double()[None, :, None]
    _check(d, want, d3)


def _wgrad_ref(dy, x, Kw, dil, Ntrue):
    T = dy.shape[1]
    pad = (Kw // 2) * dil
    xp = F.pad(rna(x).double(), (0, 0, pad, pad))
    g = rna(dy).double()
    return torch.stack([torch.einsum("btm,btn->mn", g, xp[:, j * dil:j * dil + T])[:, :Ntrue] for j in range(Kw)], dim=2)


@pytest.mark.parametrize("B,T,M,N,Kw,dil", [(1, 1, 32, 320, 1, 1), (4, 343, 320, 320, 3, 2), (16, 130, 640, 320, 1, 1)])
def test_wgrad_tf32_against_fp64(B, T, M, N, Kw, dil):
    from brainmagick_b200 import _lib
    torch.manual_seed(B + T)
    dy, x = torch.randn(B, T, M, device="cuda"), torch.randn(B, T, N, device="cuda")
    ws = torch.empty(int(_lib.load().bm_tc_wgrad_workspace(B, M, N, Kw)) + 2, device="cuda")

    def run(suffix, st):
        dw, db = torch.empty(M, N, Kw, device="cuda"), torch.empty(M, device="cuda")
        _call("bm_tc_wgrad" + suffix, _ptr(dy), _ptr(x), B, T, M, N, N, Kw, dil, _ptr(ws), _ptr(dw), _ptr(db), _ptr(st))
        return [dw, db]
    (dw, db), (dw3, _) = _both(run)
    _check(dw, _wgrad_ref(dy, x, Kw, dil, N), dw3)
    assert rel_err(db.double().cpu(), dy.double().sum((0, 1)).cpu()) < TOL     # the bias gradient sums the fp32 dy


@pytest.mark.parametrize("B,T,M,N,Kw,dil", [(1, 32, 320, 320, 3, 1), (8, 343, 320, 320, 3, 4), (4, 360, 640, 320, 3, 1)])
def test_wgrad_conv_tf32_against_fp64(B, T, M, N, Kw, dil):
    from brainmagick_b200 import _lib
    torch.manual_seed(B * T)
    dy, x = torch.randn(B, T, M, device="cuda"), torch.randn(B, T, N, device="cuda")
    assert _lib.load().bm_tc_wgrad_conv_supported(T, M, N, Kw)
    ws = torch.empty(int(_lib.load().bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)) + 2, device="cuda")

    def run(suffix, st):
        dw = torch.empty(M, N, Kw, device="cuda")
        _call("bm_tc_wgrad_conv" + suffix, _ptr(dy), _ptr(x), B, T, M, N, N, Kw, dil, _ptr(ws), _ptr(dw), _ptr(st))
        return [dw]
    (dw,), (dw3,) = _both(run)
    _check(dw, _wgrad_ref(dy, x, Kw, dil, N), dw3)


def test_wgrad_grouped_tf32_against_fp64():
    G, B, T, M, N = 3, 7, 50, 272, 256
    torch.manual_seed(7)
    dy, x = torch.randn(B, T, M, device="cuda"), torch.randn(B, T, N, device="cuda")
    grp = torch.tensor([2, 0, 2, 1, 0, 2, 2])
    order = torch.argsort(grp, stable=True).to(torch.int32).cuda()
    off = torch.tensor([0, 2, 3, 7], dtype=torch.int32, device="cuda")
    mpad = -(-M // 128) * 128

    def run(suffix, st):
        out = torch.empty(G, mpad, N, device="cuda")
        _call("bm_tc_wgrad_grouped" + suffix, _ptr(dy), _ptr(x), _ptr(order), _ptr(off), G, B, T, M, N, _ptr(out), _ptr(st))
        return [out[:, :M]]
    (o,), (o3,) = _both(run)
    per = torch.einsum("btm,btn->bmn", rna(dy).double(), rna(x).double())
    want = torch.stack([per[grp == g].sum(0) for g in range(G)])
    _check(o, want, o3)


# ---- CLIP: split-K scores at the real K, the loss with a target offset, the three backward GEMMs ----------------------
def _clip_ws(Bn, Bc, KT):
    from brainmagick_b200 import _lib
    return torch.empty(int(_lib.load().bm_clip_workspace(Bn, Bc, KT)) + 2, device="cuda")


@pytest.mark.parametrize("Bn,Bc,KT,off", [(1, 3, 32, 0), (64, 64, 1024 * 360, 0), (48, 64, 272 * 343, 10)])
def test_clip_forward_tf32_against_fp64(Bn, Bc, KT, off):
    torch.manual_seed(Bn + KT)
    est, cand = torch.randn(Bn, KT, device="cuda"), torch.randn(Bc, KT, device="cuda")
    ws = _clip_ws(Bn, Bc, KT)
    inv_want = 1.0 / (1e-8 + cand.double().norm(dim=1))                 # the norms read the fp32 candidates
    sc_want = (rna(est).double() @ rna(cand).double().t()) * inv_want
    lse = torch.logsumexp(sc_want, 1)
    loss_want = (lse - sc_want[torch.arange(Bn), torch.arange(Bn) + off]).mean()
    for det in ("", "_det"):
        def run(suffix, st):
            inv, sc, pr = torch.empty(Bc, device="cuda"), torch.empty(Bn, Bc, device="cuda"), torch.empty(Bn, Bc, device="cuda")
            rl, loss = torch.empty(Bn, device="cuda"), torch.empty(1, device="cuda")
            _call("bm_clip_loss_fwd" + det + suffix, _ptr(est), _ptr(cand), Bn, Bc, KT, off, _ptr(inv), _ptr(sc), _ptr(pr),
                  _ptr(rl), _ptr(loss), _ptr(ws), ws.numel(), _ptr(st))
            sc2 = torch.empty(Bn, Bc, device="cuda")
            _call("bm_clip_scores" + det + suffix, _ptr(est), _ptr(cand), Bn, Bc, KT, 1, _ptr(inv), _ptr(sc2), None, _ptr(ws),
                  ws.numel(), _ptr(st))
            return [inv, sc, loss, sc2]
        (inv, sc, loss, sc2), (_, sc3, _, _) = _both(run)
        assert rel_err(inv.double().cpu(), inv_want.cpu()) < 1e-6
        _check(sc, sc_want, sc3)
        assert rel_err(sc2.double().cpu(), sc_want.cpu()) < TOL
        assert abs(loss.item() - loss_want.item()) < TOL * max(1.0, abs(loss_want.item()))
        if det:
            (again,), _ = _both(lambda suffix, st: run(suffix, st)[1:2])
            assert torch.equal(again, sc)


@pytest.mark.parametrize("Bn,Bc,KT", [(64, 96, 120 * 360), (256, 256, 120 * 360)])   # dest: weight-gradient / NT form
def test_clip_backward_tf32_against_fp64(Bn, Bc, KT):
    torch.manual_seed(Bn)
    est, cand = torch.randn(Bn, KT, device="cuda"), torch.randn(Bc, KT, device="cuda")
    inv = (1.0 / (1e-8 + cand.double().norm(dim=1))).float()
    scores = ((est.double() @ cand.double().t()) * inv.double()).float()
    probs = torch.softmax(scores, 1)
    gout = torch.tensor([0.7], device="cuda")
    dscores = torch.randn(Bn, Bc, device="cuda")
    off = Bc - Bn

    def run(suffix, st):
        G, coef = torch.empty(Bn, Bc, device="cuda"), torch.empty(Bc, device="cuda")
        dest, dcand = torch.empty(Bn, KT, device="cuda"), torch.empty(Bc, KT, device="cuda")
        _call("bm_clip_loss_bwd" + suffix, _ptr(probs), _ptr(inv), _ptr(cand), _ptr(gout), Bn, Bc, KT, off, _ptr(G),
              _ptr(dest), _ptr(st))
        _call("bm_clip_loss_bwd_cand" + suffix, _ptr(probs), _ptr(scores), _ptr(inv), _ptr(est), _ptr(cand), _ptr(gout), Bn,
              Bc, KT, off, _ptr(G), _ptr(coef), _ptr(dcand), _ptr(st))
        sdest, sdcand = torch.empty(Bn, KT, device="cuda"), torch.empty(Bc, KT, device="cuda")
        _call("bm_clip_scores_bwd" + suffix, _ptr(dscores), _ptr(scores), _ptr(inv), _ptr(est), _ptr(cand), Bn, Bc, KT,
              _ptr(G), _ptr(coef), _ptr(sdest), _ptr(sdcand), _ptr(st))
        return [dest, dcand, sdest, sdcand]
    got, ref3 = _both(run)
    norm = 1.0 / inv.double() - 1e-8
    p = probs.clone()
    p[torch.arange(Bn), torch.arange(Bn) + off] -= 1
    for i, g32 in enumerate((p * (gout[0] / Bn) * inv, dscores * inv)):
        g = rna(g32).double()
        coef = (g32.double() * scores.double()).sum(0) / norm
        dest_want = g @ rna(cand).double()
        dcand_want = g.t() @ rna(est).double() - coef[:, None] * cand.double()
        _check(got[2 * i], dest_want, ref3[2 * i])
        _check(got[2 * i + 1], dcand_want, ref3[2 * i + 1])


# ---- (b) the BASELINE shapes against the fp64 oracle, at the accuracy of PyTorch's own TF32 ops ---------------------------
def _oracle(params, cfg, d, dtype, device):
    """The oracle's training step (oracle/bm_oracle.py) in `dtype` on `device`, with the gradient of meg."""
    from oracle import bm_oracle
    cast = lambda t: t.to(device=device, dtype=dtype) if t.is_floating_point() else t.to(device)   # noqa: E731
    p = {k: (cast(v).requires_grad_(True) if v.is_floating_point() and not k.endswith(("running_mean", "running_var"))
             else cast(v)) for k, v in params.items()}
    meg = cast(d["meg"]).requires_grad_(True)
    est = bm_oracle.simpleconv_forward(p, cfg, meg, cast(d["rec_positions"]), d["rec_of_sample"].to(device),
                                       d["subject_index"].to(device), True, cast(d["ban_centre"]), {})
    scores = bm_oracle.clip_scores(est, cast(d["candidates"]))
    loss = F.cross_entropy(scores, torch.arange(len(scores), device=device))
    names = [k for k, v in p.items() if v.requires_grad]
    grads = torch.autograd.grad(loss, [p[k] for k in names] + [meg], allow_unused=True)
    out = dict(estimate=est.detach(), loss=loss.detach().reshape(1), meg=grads[-1])
    out.update({"grad." + k: g for k, g in zip(names, grads[:-1])})
    return {k: v.double().cpu() for k, v in out.items()}


@pytest.mark.parametrize("idx", [0, 3], ids=["cfg2", "cfg5"])
def test_baseline_shapes_match_oracle_in_tf32(idx):
    import test_gpu_parity
    from oracle import bm_oracle
    from brainmagick_b200 import synthetic
    case = test_gpu_parity.BASELINE_SHAPES[idx]
    cfg = bm_oracle.Config(in_channels=case["C"], out_channels=case["F"], n_subjects=case["S"])
    params = bm_oracle.init_state_dict(cfg, seed=21)
    d = bm_oracle.synthetic_batch(cfg, batch=case["B"], T=case["T"], seed=9, n_valid=case["n_valid"])
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, case["n_valid"], seed=4)
    ref64 = _oracle(params, cfg, d, torch.float64, "cpu")
    with precision(True):
        torch_tf32 = _oracle(params, cfg, d, torch.float32, "cuda")     # the oracle's own torch ops, TF32 on this GPU
        model = test_gpu_parity._build_model(cfg, params)
        meg = d["meg"].cuda().requires_grad_(True)
        batch = synthetic.make_batch(meg, d["subject_index"].cuda(), d["rec_positions"], d["rec_of_sample"])
        model.train()
        model.merger.ban_centre_override = d["ban_centre"]
        import brainmagick_b200 as bb
        est = model(dict(meg=meg), batch)
        loss = bb.ClipLoss().cuda().train()(est, d["candidates"].cuda(),
                                             torch.ones(case["B"], 1, case["T"], dtype=torch.bool, device="cuda"))
        loss.backward()
        torch.cuda.synchronize()
    mine = dict(estimate=est.detach(), loss=loss.detach().reshape(1), meg=meg.grad)
    mine.update({"grad." + n: p.grad for n, p in model.named_parameters()})
    wscale = max(v.norm().item() for k, v in ref64.items() if k.startswith("grad.") and k.endswith("weight"))
    report = []
    for k, want in ref64.items():
        got, tt = mine[k].double().cpu(), torch_tf32[k]
        if "sequence" in k and k.endswith(".0.bias"):          # exactly zero in truth (training-mode BatchNorm follows)
            e, e_t = got.abs().max().item() / wscale, tt.abs().max().item() / wscale
        else:
            e, e_t = rel_err(got, want), rel_err(tt, want)
        report.append((k, e, e_t))
        assert e <= max(2 * e_t, 2e-3), (k, e, e_t)
    worst = max(report, key=lambda r: r[1])
    print(f"\n[{case['name']} TF32] worst {worst[0]}: library {worst[1]:.2e}, torch TF32 ops {worst[2]:.2e}; "
          + ", ".join(f"{k} {e:.1e}/{e_t:.1e}" for k, e, e_t in report if k in ("estimate", "loss", "meg")))


# ---- (c) accuracy: the same weights evaluated with the flag on and off, and a model trained with it on ------------------
def test_tf32_training_learns_and_evaluates_like_the_default():
    import json
    import os
    import brainmagick_b200 as bb
    from brainmagick_b200 import functional as BF, retrieval, synthetic
    from oracle import make_accuracy_golden as mg
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "accuracy_full_width.json")
    with open(path) as f:
        spec = json.load(f)["spec"]
    cfg, task, sched, p0 = mg.build(spec)
    model = bb.SimpleConv(
        in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden), depth=cfg.depth,
        dilation_period=5, kernel_size=3, skip=True, subject_layers=True, subject_dim=0, complex_out=True, glu=2,
        glu_context=1, merger=True, initial_linear=cfg.initial_linear, merger_channels=cfg.merger_channels, gelu=True,
        batch_norm=True, merger_pos_dim=cfg.merger_pos_dim, n_subjects=cfg.n_subjects)
    model.load_state_dict(p0)
    model = model.cuda().train()
    clip = bb.ClipLoss().cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=spec["lr"], betas=(0.9, 0.999))
    recs = [synthetic.SyntheticRecording(s, task["positions"][s]) for s in range(cfg.n_subjects)]
    d = task["train"]
    mask = torch.ones(spec["batch"], 1, spec["T"], dtype=torch.bool, device="cuda")
    losses = []
    with precision(True):
        for idx, ban in sched:
            meg, feats, subj = d["meg"][idx].cuda(), d["feats"][idx].cuda(), d["subj"][idx].cuda()
            batch = synthetic.SyntheticBatch(meg, subj, [recs[int(s)] for s in d["subj"][idx]])
            model.merger.ban_centre_override = ban
            opt.zero_grad(set_to_none=True)
            loss = clip(model(dict(meg=meg), batch), feats, mask)
            loss.backward()
            opt.step()
            losses.append(loss.detach())
    BF.check_tc_status()
    model.eval()
    clip.eval()
    e = task["eval"]
    n_eval = len(e["meg"])
    labels = torch.arange(n_eval)
    acc = {}
    for tf32 in (True, False):
        with precision(tf32), torch.no_grad():
            ests = []
            for i in range(0, n_eval, 256):
                sl = slice(i, i + 256)
                meg, subj = e["meg"][sl].cuda(), e["subj"][sl].cuda()
                ests.append(model(dict(meg=meg), synthetic.SyntheticBatch(meg, subj, [recs[int(s)] for s in e["subj"][sl]])))
            acc[tf32] = retrieval.retrieval_accuracy(clip, torch.cat(ests), e["feats"], labels, labels, topk=(1, 10),
                                                     batch_size=256)
    losses = [float(v) for v in torch.stack(losses).cpu()]
    print(f"\n[TF32 accuracy] trained with TF32: top-10 {acc[True][10]:.4f} (TF32 eval) / {acc[False][10]:.4f} (default "
          f"eval), top-1 {acc[True][1]:.4f} / {acc[False][1]:.4f}; loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert abs(acc[True][10] - acc[False][10]) <= 0.005 and abs(acc[True][1] - acc[False][1]) <= 0.005, acc
    assert acc[True][10] > 0.05, "trained with TF32, the model must have learnt the task (chance: 0.01)"


# ---- (d) with the determinism flag, (e) no state left behind --------------------------------------------------------------
@pytest.mark.parametrize("case", ["baseline_C208_T360", "baseline_mixed_T343", "small_fp32_fma"])
def test_tf32_steps_are_bitwise_repeatable_with_determinism(case):
    import test_gpu_deterministic as gd
    kw, dims = gd.CASES[case]
    with deterministic(), precision(True):
        first = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
        second = gd._train(kw, **dims, meg_grad=True, perturb=True, eval_forward=True)
    gd._assert_bitwise(first, second)


def test_turning_tf32_off_leaves_no_state():
    import test_gpu_deterministic as gd
    kw, dims = gd.CASES["baseline_C208_T360"]
    dims = dict(dims, B=16)
    with deterministic():
        never = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
        with precision(True):
            on = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
        after = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
    gd._assert_bitwise(never, after)
    assert not torch.equal(on[0]["est"], never[0]["est"])
