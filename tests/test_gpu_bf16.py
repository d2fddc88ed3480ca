"""torch.autocast(dtype=torch.bfloat16) on the GPU: every `_bf16` entry point against an fp64 contraction of its
bf16-rounded operands, element by element, the rounding mode itself, the BASELINE shapes against the fp64 oracle at the
accuracy PyTorch's own bf16 autocast reaches, training accuracy, determinism, state and CUDA graph capture."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                # unit roundoff of fp32


def rn(t):
    """fp32 -> nearest bf16 (ties to even), as fp32: cvt.rn.bf16x2.f32."""
    return t.to(torch.bfloat16).float()


def autocast(enabled=True, dtype=torch.bfloat16):
    return torch.autocast("cuda", dtype=dtype, enabled=enabled)


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


def _forms(fn):
    """fn(suffix, status) for the bf16 form and the TF32 form -> (bf16 outputs, TF32 outputs), checking the status word."""
    out = []
    for suffix in ("_bf16", "_tf32"):
        st = _status()
        res = fn(suffix, st)
        torch.cuda.synchronize()
        assert int(st.item()) == 0
        out.append([r.clone() for r in res])
    return out


def _check(got, want, mag, K, other=None, extra=None):
    """Per element: |got - want| <= 2 (K + 2) u mag (+ extra), with want the fp64 contraction of the bf16-rounded operands
    and mag the same contraction of their magnitudes: only the fp32 accumulation of exact products remains.  `other` (the
    TF32 form's output) must differ: the bf16 rounding is visible."""
    got, want, mag = got.double().cpu(), want.double().cpu(), mag.double().cpu()
    bound = 2 * (K + 2) * U * mag + 2 * U * want.abs() + 2.0 ** -140
    if extra is not None:
        bound = bound + extra.double().cpu()
    excess = (got - want).abs() - bound
    assert torch.isfinite(got).all()
    assert excess.max().item() <= 0, (excess.argmax().item(), excess.max().item())
    if other is not None:
        assert not torch.equal(got, other.double().cpu())
    return ((got - want).abs() / bound.clamp_min(1e-300)).max().item()


# ---- (a) the rounding mode: outputs that are single bf16-rounded operand elements ------------------------------------
def _tie_cases(n):
    """fp32 values around bf16 ties: exact ties (RNE goes to even, ties-away / truncation do not), values just above and
    below a tie, and values that a tf32 rounding first would carry onto a tie (a double rounding)."""
    ulp = 2.0 ** -7
    base = torch.tensor([1.0 + 0.5 * ulp, 1.0 + 1.5 * ulp, 1.0 + 0.5 * ulp + 2.0 ** -20, 1.0 + 1.5 * ulp - 2.0 ** -20,
                         1.0 + (1.5 - 1.0 / 32) * ulp, 1.0 + (0.5 + 1.0 / 32) * ulp, 1.0 + 0.75 * ulp, 1.0 + 0.25 * ulp])
    scale = 2.0 ** torch.arange(-6, 6).double()
    vals = (base.double()[:, None] * scale[None, :]).flatten().float()
    vals = torch.cat([vals, -vals])
    return vals.repeat((n + len(vals) - 1) // len(vals))[:n]


def test_rounding_is_to_nearest_even_on_both_operands():
    """y = x W with one-hot W (or one-hot x) is one rounded operand element per output: the kernels' bf16 values are
    exactly torch's round-to-nearest-even, for the activation side (A) and the weight side (B) of the conv kernel, and
    for both operands of the register-staged and the TMA-fed weight-gradient kernels."""
    B, T, Cin, Ntot = 1, 8, 32, 64
    v = _tie_cases(B * T * Cin).reshape(B, T, Cin).cuda()
    assert not torch.equal(rn(v), v)
    onehot = torch.zeros(Ntot, Cin, device="cuda")
    onehot[torch.arange(Ntot), torch.arange(Ntot) % Cin] = 1.0
    wsel = torch.zeros(B, dtype=torch.int32, device="cuda")
    st = _status()
    y = torch.empty(B, T, Ntot, device="cuda")
    _call("bm_tc_pointwise_sel_bf16", _ptr(v), _ptr(onehot), None, _ptr(wsel), 1, B, T, Cin, Ntot, _ptr(y), _ptr(st))
    assert torch.equal(y, rn(v)[:, :, torch.arange(Ntot) % Cin])                     # A rounded in the consumers
    w = _tie_cases(Ntot * Cin).reshape(Ntot, Cin).cuda()
    x1 = torch.zeros(B, T, Cin, device="cuda")
    x1[:, torch.arange(T), torch.arange(T)] = 1.0
    _call("bm_tc_pointwise_sel_bf16", _ptr(x1), _ptr(w), None, _ptr(wsel), 1, B, T, Cin, Ntot, _ptr(y), _ptr(st))
    assert torch.equal(y[0], rn(w)[:, :T].t())                                       # B rounded by the producer
    # weight gradients: out[m][n] = sum_t dy[t][m] x[t][n] with a single live row t
    M, N = 128, 128
    a, b = _tie_cases(M).cuda(), _tie_cases(N).flip(0).cuda()
    dy, x = torch.zeros(1, 32, M, device="cuda"), torch.zeros(1, 32, N, device="cuda")
    dy[0, 5], x[0, 5] = a, 1.0
    off = torch.tensor([0, 1], dtype=torch.int32, device="cuda")
    order = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.empty(1, M, N, device="cuda")
    _call("bm_tc_wgrad_grouped_bf16", _ptr(dy), _ptr(x), _ptr(order), _ptr(off), 1, 1, 32, M, N, _ptr(out), _ptr(st))
    assert torch.equal(out[0], rn(a)[:, None].expand(M, N))
    dy[0, 5], x[0, 5] = 1.0, b
    _call("bm_tc_wgrad_grouped_bf16", _ptr(dy), _ptr(x), _ptr(order), _ptr(off), 1, 1, 32, M, N, _ptr(out), _ptr(st))
    assert torch.equal(out[0], rn(b)[None, :].expand(M, N))
    from brainmagick_b200 import _lib
    T2, M2, N2 = 64, 320, 320
    assert _lib.load().bm_tc_wgrad_conv_supported(T2, M2, N2, 1)
    ws = torch.empty(int(_lib.load().bm_tc_wgrad_conv_workspace(1, T2, M2, N2, 1)) + 2, device="cuda")
    for side in ("dy", "x"):
        dy2, x2 = torch.zeros(1, T2, M2, device="cuda"), torch.zeros(1, T2, N2, device="cuda")
        if side == "dy":
            dy2[0, 37], x2[0, 37] = _tie_cases(M2).cuda(), 1.0
            want = rn(dy2[0, 37])[:, None].expand(M2, N2)
        else:
            dy2[0, 37], x2[0, 37] = 1.0, _tie_cases(N2).cuda()
            want = rn(x2[0, 37])[None, :].expand(M2, N2)
        dw = torch.empty(M2, N2, 1, device="cuda")
        _call("bm_tc_wgrad_conv_bf16", _ptr(dy2), _ptr(x2), 1, T2, M2, N2, N2, 1, 1, _ptr(ws), _ptr(dw), _ptr(st))
        torch.cuda.synchronize()
        assert torch.equal(dw[:, :, 0], want), side
    assert int(st.item()) == 0


# ---- (b) every _bf16 entry point at its edges, element by element ----------------------------------------------------
CONV_CASES = [  # B, T, Cin, Ntot, Kw, dilation, sign, glu
    (1, 1, 32, 320, 3, 1, 1, 0),          # one row, one K block per tap
    (3, 343, 320, 320, 3, 4, 1, 0),       # 160-wide tiles, a partial time tile
    (2, 200, 64, 1024, 1, 1, 1, 0),       # 128-wide tiles
    (2, 343, 320, 640, 3, 1, 1, 1),       # GLU (80 'a' columns per tile)
    (3, 129, 320, 320, 3, 2, -1, 0),      # data-gradient taps
]


def _conv_ref(x, w, bias, dil, sign):
    Kw = w.shape[2]
    if sign < 0:
        w = w.flip(2)
    return F.conv1d(x.transpose(1, 2), w, bias, padding=dil * (Kw // 2), dilation=dil).transpose(1, 2)


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("form", ["persistent", "presplit"])
def test_conv_bf16_against_fp64(case, form):
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
        else:          # the bf16 form rounds hi + lo of the pre-split weights
            _call("bm_tc_conv1d" + suffix, _ptr(x), _ptr(hi), _ptr(lo), _ptr(bias), None, B, T, Cin, Ntot, Kw, dil, sign,
                  glu, 0, 0, _ptr(y), None, _ptr(g), None, _ptr(st))
        return [y]
    (y,), (yt,) = _forms(run)
    wr = rn(w if form == "persistent" else (hi + lo).permute(1, 2, 0)).double()
    want = _conv_ref(rn(x).double(), wr, bias.double(), dil, sign)
    mag = _conv_ref(rn(x).double().abs(), wr.abs(), bias.double().abs(), dil, sign)
    _check(y, want, mag, Cin * Kw, yt)


def test_pointwise_sel_and_sensor_mix_bwd_bf16_against_fp64():
    S, B, T, Cin, Ntot = 3, 5, 343, 320, 320
    torch.manual_seed(1)
    x, w = torch.randn(B, T, Cin, device="cuda"), torch.randn(S, Ntot, Cin, device="cuda")
    wsel = torch.tensor([2, 0, 1, 2, 2], dtype=torch.int32, device="cuda")

    def run(suffix, st):
        y = torch.empty(B, T, Ntot, device="cuda")
        _call("bm_tc_pointwise_sel" + suffix, _ptr(x), _ptr(w), None, _ptr(wsel), S, B, T, Cin, Ntot, _ptr(y), _ptr(st))
        return [y]
    (y,), (yt,) = _forms(run)
    xr, wr = rn(x).double(), rn(w).double()[wsel.long()]
    _check(y, torch.einsum("btk,bnk->btn", xr, wr), torch.einsum("btk,bnk->btn", xr.abs(), wr.abs()), Cin, yt)

    Op, Cp, C = 320, 256, 201                           # odd live sensor count
    du, wt = torch.randn(B, T, Op, device="cuda"), torch.randn(S, Cp, Op, device="cuda")
    mask = (torch.rand(C, device="cuda") > 0.2).float()

    def run2(suffix, st):
        dmeg = torch.empty(B, C, T, device="cuda")
        _call("bm_tc_sensor_mix_bwd_data" + suffix, _ptr(du), _ptr(wt), None, _ptr(wsel), S, _ptr(mask), B, T, Op, Cp,
              C, _ptr(dmeg), _ptr(st))
        return [dmeg]
    (d,), (dt,) = _forms(run2)
    dr, wr = rn(du).double(), rn(wt).double()[wsel.long(), :C]
    m = mask.double()[None, :, None]
    _check(d, torch.einsum("bto,bco->bct", dr, wr) * m, torch.einsum("bto,bco->bct", dr.abs(), wr.abs()) * m, Op, dt)


def _wgrad_ref(dy, x, Kw, dil, Ntrue):
    T = dy.shape[1]
    pad = (Kw // 2) * dil
    xp = F.pad(x, (0, 0, pad, pad))
    return torch.stack([torch.einsum("btm,btn->mn", dy, xp[:, j * dil:j * dil + T])[:, :Ntrue] for j in range(Kw)], dim=2)


@pytest.mark.parametrize("B,T,M,N,Kw,dil", [(1, 1, 32, 320, 1, 1), (4, 343, 320, 320, 3, 2), (16, 130, 640, 320, 1, 1)])
def test_wgrad_bf16_against_fp64(B, T, M, N, Kw, dil):
    from brainmagick_b200 import _lib
    torch.manual_seed(B + T)
    dy, x = torch.randn(B, T, M, device="cuda"), torch.randn(B, T, N, device="cuda")
    ws = torch.empty(int(_lib.load().bm_tc_wgrad_workspace(B, M, N, Kw)) + 2, device="cuda")

    def run(suffix, st):
        dw, db = torch.empty(M, N, Kw, device="cuda"), torch.empty(M, device="cuda")
        _call("bm_tc_wgrad" + suffix, _ptr(dy), _ptr(x), B, T, M, N, N, Kw, dil, _ptr(ws), _ptr(dw), _ptr(db), _ptr(st))
        return [dw, db]
    (dw, db), (dwt, _) = _forms(run)
    d, xr = rn(dy).double(), rn(x).double()
    _check(dw, _wgrad_ref(d, xr, Kw, dil, N), _wgrad_ref(d.abs(), xr.abs(), Kw, dil, N), B * T, dwt)
    _check(db, dy.double().sum((0, 1)), dy.double().abs().sum((0, 1)), B * T)        # the bias gradient sums fp32 dy


@pytest.mark.parametrize("B,T,M,N,Kw,dil", [(1, 32, 320, 320, 3, 1), (8, 343, 320, 320, 3, 4), (4, 360, 640, 320, 3, 1)])
def test_wgrad_conv_bf16_against_fp64(B, T, M, N, Kw, dil):
    from brainmagick_b200 import _lib
    torch.manual_seed(B * T)
    dy, x = torch.randn(B, T, M, device="cuda"), torch.randn(B, T, N, device="cuda")
    assert _lib.load().bm_tc_wgrad_conv_supported(T, M, N, Kw)
    ws = torch.empty(int(_lib.load().bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)) + 2, device="cuda")

    def run(suffix, st):
        dw = torch.empty(M, N, Kw, device="cuda")
        _call("bm_tc_wgrad_conv" + suffix, _ptr(dy), _ptr(x), B, T, M, N, N, Kw, dil, _ptr(ws), _ptr(dw), _ptr(st))
        return [dw]
    (dw,), (dwt,) = _forms(run)
    d, xr = rn(dy).double(), rn(x).double()
    _check(dw, _wgrad_ref(d, xr, Kw, dil, N), _wgrad_ref(d.abs(), xr.abs(), Kw, dil, N), B * T, dwt)


def test_wgrad_grouped_bf16_against_fp64():
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
    (o,), (ot,) = _forms(run)
    d, xr = rn(dy).double(), rn(x).double()
    per, per_abs = torch.einsum("btm,btn->bmn", d, xr), torch.einsum("btm,btn->bmn", d.abs(), xr.abs())
    want = torch.stack([per[grp == g].sum(0) for g in range(G)])
    mag = torch.stack([per_abs[grp == g].sum(0) for g in range(G)])
    _check(o, want, mag, 4 * T, ot)


# ---- CLIP: split-K scores at the real K, the loss with a target offset, the three backward GEMMs ----------------------
def _clip_ws(Bn, Bc, KT):
    from brainmagick_b200 import _lib
    return torch.empty(int(_lib.load().bm_clip_workspace(Bn, Bc, KT)) + 2, device="cuda")


@pytest.mark.parametrize("Bn,Bc,KT,off", [(1, 3, 32, 0), (64, 64, 1024 * 360, 0), (48, 64, 272 * 343, 10)])
def test_clip_forward_bf16_against_fp64(Bn, Bc, KT, off):
    torch.manual_seed(Bn + KT)
    est, cand = torch.randn(Bn, KT, device="cuda"), torch.randn(Bc, KT, device="cuda")
    ws = _clip_ws(Bn, Bc, KT)
    inv_want = 1.0 / (1e-8 + cand.double().norm(dim=1))                 # the norms read the fp32 candidates
    er, cr = rn(est).double(), rn(cand).double()
    sc_want = (er @ cr.t()) * inv_want
    sc_mag = (er.abs() @ cr.abs().t()) * inv_want
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
        (inv, sc, loss, sc2), (_, sct, _, _) = _forms(run)
        assert rel_err(inv.double().cpu(), inv_want.cpu()) < 1e-6
        extra = 2 * U * sc_mag         # the norm's own fp32 rounding, applied to the dot product
        _check(sc, sc_want, sc_mag, KT, sct, extra)
        _check(sc2, sc_want, sc_mag, KT, None, extra)
        assert abs(loss.item() - loss_want.item()) < 1e-5 * max(1.0, abs(loss_want.item()))
        if det:
            (again,), _ = _forms(lambda suffix, st: run(suffix, st)[1:2])
            assert torch.equal(again, sc)


@pytest.mark.parametrize("Bn,Bc,KT", [(64, 96, 120 * 360), (256, 256, 120 * 360)])   # dest: weight-gradient / NT form
def test_clip_backward_bf16_against_fp64(Bn, Bc, KT):
    """inv_norm = 1 and gout = Bn make the G each entry point forms in fp32 exactly the one restated here."""
    torch.manual_seed(Bn)
    est, cand = torch.randn(Bn, KT, device="cuda"), torch.randn(Bc, KT, device="cuda")
    inv = torch.ones(Bc, device="cuda")
    scores = (est.double() @ cand.double().t()).float() / KT ** 0.5
    probs = torch.softmax(scores, 1)
    gout = torch.tensor([float(Bn)], device="cuda")
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
    got, tf = _forms(run)
    norm = 1.0 / inv.double() - 1e-8
    p = probs.clone()
    p[torch.arange(Bn), torch.arange(Bn) + off] -= 1
    for i, g32 in enumerate((p, dscores)):
        g = rn(g32).double()
        coef = (g32.double() * scores.double()).sum(0) / norm
        cr, er = rn(cand).double(), rn(est).double()
        _check(got[2 * i], g @ cr, g.abs() @ cr.abs(), Bc, tf[2 * i])
        corr = coef.abs()[:, None] * cand.double().abs()
        # the correction term coef * cand: coef is an fp32 sum over Bn terms, then one product and one subtraction
        _check(got[2 * i + 1], g.t() @ er - coef[:, None] * cand.double(), g.abs().t() @ er.abs(), Bn, tf[2 * i + 1],
               extra=2 * (Bn + 4) * U * corr + 2 * (Bn + 2) * U * ((g32.double() * scores.double()).abs().sum(0) / norm)[
                   :, None] * cand.double().abs())


# ---- (c) the BASELINE shapes against the fp64 oracle, at the accuracy of PyTorch's own bf16 autocast ------------------
FLOOR = 1e-2        # bf16 keeps 8 significant bits: 2^-9 = 2e-3 per rounding, a few roundings deep


@pytest.mark.parametrize("idx", [0, 3], ids=["cfg2", "cfg5"])
def test_baseline_shapes_match_oracle_in_bf16(idx):
    import brainmagick_b200 as bb
    import test_gpu_parity
    import test_gpu_tf32 as gt
    from oracle import bm_oracle
    from brainmagick_b200 import synthetic
    case = test_gpu_parity.BASELINE_SHAPES[idx]
    cfg = bm_oracle.Config(in_channels=case["C"], out_channels=case["F"], n_subjects=case["S"])
    params = bm_oracle.init_state_dict(cfg, seed=21)
    d = bm_oracle.synthetic_batch(cfg, batch=case["B"], T=case["T"], seed=9, n_valid=case["n_valid"])
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, case["n_valid"], seed=4)
    ref64 = gt._oracle(params, cfg, d, torch.float64, "cpu")
    with autocast():
        torch_bf16 = gt._oracle(params, cfg, d, torch.float32, "cuda")   # the oracle's own torch ops under bf16 autocast
    model = test_gpu_parity._build_model(cfg, params)
    meg = d["meg"].cuda().requires_grad_(True)
    batch = synthetic.make_batch(meg, d["subject_index"].cuda(), d["rec_positions"], d["rec_of_sample"])
    model.train()
    model.merger.ban_centre_override = d["ban_centre"]
    with autocast():
        est = model(dict(meg=meg), batch)
        loss = bb.ClipLoss().cuda().train()(est, d["candidates"].cuda(),
                                             torch.ones(case["B"], 1, case["T"], dtype=torch.bool, device="cuda"))
    loss.backward()
    torch.cuda.synchronize()
    assert est.dtype == torch.float32 and all(p.grad.dtype == torch.float32 for p in model.parameters())
    mine = dict(estimate=est.detach(), loss=loss.detach().reshape(1), meg=meg.grad)
    mine.update({"grad." + n: p.grad for n, p in model.named_parameters()})
    wscale = max(v.norm().item() for k, v in ref64.items() if k.startswith("grad.") and k.endswith("weight"))
    report = []
    for k, want in ref64.items():
        got, tt = mine[k].double().cpu(), torch_bf16[k]
        if "sequence" in k and k.endswith(".0.bias"):          # exactly zero in truth (training-mode BatchNorm follows)
            e, e_t = got.abs().max().item() / wscale, tt.abs().max().item() / wscale
        else:
            e, e_t = rel_err(got, want), rel_err(tt, want)
        report.append((k, e, e_t))
    worst = max(report, key=lambda r: r[1] / max(2 * r[2], FLOOR))
    print(f"\n[{case['name']} bf16, floor {FLOOR:.0e}] worst {worst[0]}: library {worst[1]:.2e}, torch bf16 autocast "
          f"{worst[2]:.2e}; " + ", ".join(f"{k} {e:.1e}/{e_t:.1e}" for k, e, e_t in report
                                          if k in ("estimate", "loss", "meg")))
    for k, e, e_t in report:
        assert e <= max(2 * e_t, FLOOR), (k, e, e_t)


# ---- (d) accuracy: a model trained under bf16 autocast, evaluated with and without it ----------------------------------
def test_bf16_training_learns_and_evaluates_like_fp32():
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
    for idx, ban in sched:
        meg, feats, subj = d["meg"][idx].cuda(), d["feats"][idx].cuda(), d["subj"][idx].cuda()
        batch = synthetic.SyntheticBatch(meg, subj, [recs[int(s)] for s in d["subj"][idx]])
        model.merger.ban_centre_override = ban
        opt.zero_grad(set_to_none=True)
        with autocast():
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
    for bf16 in (True, False):
        with autocast(bf16), torch.no_grad():
            ests = []
            for i in range(0, n_eval, 256):
                sl = slice(i, i + 256)
                meg, subj = e["meg"][sl].cuda(), e["subj"][sl].cuda()
                ests.append(model(dict(meg=meg), synthetic.SyntheticBatch(meg, subj, [recs[int(s)] for s in e["subj"][sl]])))
            acc[bf16] = retrieval.retrieval_accuracy(clip, torch.cat(ests), e["feats"], labels, labels, topk=(1, 10),
                                                     batch_size=256)
    losses = [float(v) for v in torch.stack(losses).cpu()]
    print(f"\n[bf16 accuracy] trained under bf16 autocast: top-10 {acc[True][10]:.4f} (bf16 eval) / {acc[False][10]:.4f} "
          f"(fp32 eval), top-1 {acc[True][1]:.4f} / {acc[False][1]:.4f}; loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert abs(acc[True][10] - acc[False][10]) <= 0.01 and abs(acc[True][1] - acc[False][1]) <= 0.01, acc
    assert acc[True][10] > 0.05, "trained under bf16 autocast, the model must have learnt the task (chance: 0.01)"


# ---- (e) with the determinism flag, (f) no state left behind, (g) CUDA graph capture -----------------------------------
@pytest.mark.parametrize("case", ["baseline_C208_T360", "baseline_mixed_T343", "small_fp32_fma"])
def test_bf16_steps_are_bitwise_repeatable_with_determinism(case):
    import test_gpu_deterministic as gd
    kw, dims = gd.CASES[case]
    with deterministic(), autocast():
        first = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
        second = gd._train(kw, **dims, meg_grad=True, perturb=True, eval_forward=True)
    gd._assert_bitwise(first, second)


def test_leaving_bf16_autocast_leaves_no_state():
    import test_gpu_deterministic as gd
    kw, dims = gd.CASES["baseline_C208_T360"]
    dims = dict(dims, B=16)
    with deterministic():
        never = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
        with autocast():
            on = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
        after = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
        with autocast(dtype=torch.float16):
            fp16 = gd._train(kw, **dims, meg_grad=True, eval_forward=True)
    gd._assert_bitwise(never, after)
    gd._assert_bitwise(never, fp16)                   # fp16 autocast is not honoured: the default forms run
    assert not torch.equal(on[0]["est"], never[0]["est"])


def test_captured_training_step_under_bf16_autocast():
    import test_gpu_cuda_graph as gg
    with deterministic(), autocast():
        gg._graph_vs_eager(*gg.CASES["clip_conv"])
