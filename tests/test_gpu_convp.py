"""GPU: the conv entry points -- fp32 weights (bm_tc_conv1d_persistent) and fp16-piece weights (bm_tc_conv1d_f16), both
on the 3xTF32 wgmma engine of csrc/tc_conv.cuh -- in every epilogue mode against torch's fp64 conv (test-only
reference), at the real layer shapes, incl. the flattened-row tiling across sample edges (odd batch sizes, T not a multiple
of anything) and the BatchNorm statistics out of the epilogue."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 3e-5
DEV = "cuda"


def _abi():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream


def _raw_operands(w):
    """w [Cout,Cin,Kw] -> forward operand [Kw,Cout,Cin] and data-gradient operand [Kw,Cin,Cout], raw fp32."""
    call, ptr, stream = _abi()
    Cout, Cin, Kw = w.shape
    f = torch.empty(Kw, Cout, Cin, device=DEV)
    g = torch.empty(Kw, Cin, Cout, device=DEV)
    call("bm_tc_weight_split", ptr(w), Cout, Cin, Kw, ptr(f), None, ptr(g), None, stream())
    return f, g


def _ref_conv(x, w, bias, dilation):
    y = torch.nn.functional.conv1d(x.double().permute(0, 2, 1), w.double(), None if bias is None else bias.double(),
                                   padding=(w.shape[2] // 2) * dilation, dilation=dilation)
    return y.permute(0, 2, 1).contiguous()


PIPE = "tf32"


@pytest.fixture(params=["tf32", "f16"], autouse=True)
def pipe(request):
    global PIPE
    PIPE = request.param
    yield request.param
    PIPE = "tf32"


def _f16_operands(x, w_op):
    """What the host path prepares for bm_tc_conv1d_f16: amax of x, amax + fp16 pieces of the (re-laid) weights."""
    call, ptr, stream = _abi()
    amax = torch.empty(2, device=DEV)
    call("bm_amax", ptr(x), x.numel(), ptr(amax[0:1]), stream())
    call("bm_amax", ptr(w_op), w_op.numel(), ptr(amax[1:2]), stream())
    hi = torch.empty(w_op.shape, device=DEV, dtype=torch.float16)
    lo = torch.empty(w_op.shape, device=DEV, dtype=torch.float16)
    call("bm_f16_split", ptr(w_op), w_op.numel(), ptr(amax[1:2]), ptr(hi), ptr(lo), stream())
    return amax, hi, lo


def _run(x, w_op, bias, accumulate, B, T, Cin, Ntot, Kw, dil, sign, glu, act, tmajor, y, aux, glu_out, stats):
    call, ptr, stream = _abi()
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    if PIPE == "f16":
        amax, hi, lo = _f16_operands(x, w_op)
        # the epilogues another conv consumes (GLU out, GELU out) also report max |output| for that conv's scale
        out_amax = torch.full((1,), float("nan"), device=DEV) if (glu or act) and not tmajor else None
        call("bm_tc_conv1d_f16", ptr(x), ptr(amax[0:1]), ptr(hi), ptr(lo), ptr(amax[1:2]), ptr(bias), accumulate, B, T, Cin,
             Ntot, Kw, dil, sign, glu, act, tmajor, ptr(y), ptr(aux), ptr(glu_out), ptr(stats), ptr(out_amax), ptr(status),
             stream())
        if out_amax is not None:
            produced = glu_out if glu else y
            assert float(out_amax) == float(produced.abs().max()), (float(out_amax), float(produced.abs().max()))
    else:
        call("bm_tc_conv1d_persistent", ptr(x), ptr(w_op), ptr(bias), accumulate, B, T, Cin, Ntot, Kw, dil, sign, glu, act,
             tmajor, ptr(y), ptr(aux), ptr(glu_out), ptr(stats), ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"tensor-core kernel timed out at barrier code {int(status.item())}"


@pytest.mark.parametrize("xs,ws,spread", [(1e-6, 1e-3, 0), (3e4, 50.0, 0), (1.0, 1.0, 12), (1e-30, 1e30, 6)])
def test_operand_ranges(xs, ws, spread):
    """Operand magnitudes far from 1 and a wide dynamic range inside one tensor (per-channel factors 2^-spread .. 2^spread):
    the fp16 pieces rely on the per-tensor power-of-two scale, the tf32 pieces on nothing."""
    torch.manual_seed(11)
    B, T, Cin, Cout, Kw = 3, 200, 320, 320, 3
    fac = torch.exp2((torch.rand(Cin, device=DEV) * 2 - 1) * spread)
    x = torch.randn(B, T, Cin, device=DEV) * fac * xs
    w = torch.randn(Cout, Cin, Kw, device=DEV) / (Cin * Kw) ** 0.5 * ws
    f, _ = _raw_operands(w)
    y = torch.full((B, T, Cout), float("nan"), device=DEV)
    _run(x, f, None, 0, B, T, Cin, Cout, Kw, 2, 1, 0, 0, 0, y, None, None, None)
    ref = _ref_conv(x, w, None, 2)
    e = rel_err(y.cpu(), ref.cpu())
    print(f"[conv {PIPE} x*{xs:g} w*{ws:g} spread 2^+-{spread}] rel_err vs fp64 = {e:.2e}")
    assert e < TOL


@pytest.mark.parametrize("B,T,dilation", [(3, 360, 1), (3, 360, 16), (5, 343, 2), (2, 100, 4), (1, 40, 8), (7, 361, 16),
                                          (160, 360, 4)])
def test_forward_with_statistics(B, T, dilation):
    torch.manual_seed(B * 1000 + T + dilation)
    Cin, Cout, Kw = 320, 320, 3
    x = torch.randn(B, T, Cin, device=DEV)
    w = torch.randn(Cout, Cin, Kw, device=DEV) / (Cin * Kw) ** 0.5
    bias = torch.randn(Cout, device=DEV)
    f, _ = _raw_operands(w)
    y = torch.full((B, T, Cout), float("nan"), device=DEV)
    stats = torch.full((2 * Cout,), float("nan"), device=DEV, dtype=torch.float64)
    _run(x, f, bias, 0, B, T, Cin, Cout, Kw, dilation, 1, 0, 0, 0, y, None, None, stats)
    ref = _ref_conv(x, w, bias, dilation)
    e = rel_err(y.cpu(), ref.cpu())
    print(f"[convp fwd B={B} T={T} d={dilation}] rel_err vs fp64 = {e:.2e}")
    assert e < TOL
    yd = y.double().reshape(-1, Cout)
    assert rel_err(stats[:Cout].cpu(), yd.sum(0).cpu()) < 1e-6
    assert rel_err(stats[Cout:].cpu(), (yd * yd).sum(0).cpu()) < 1e-6


@pytest.mark.parametrize("B,T", [(2, 360), (3, 343), (5, 77)])
@pytest.mark.parametrize("save_h", [True, False])
def test_glu_and_data_gradient(B, T, save_h):
    torch.manual_seed(7 + B)
    H, Kw = 320, 3
    x = torch.randn(B, T, H, device=DEV)
    w = torch.randn(2 * H, H, Kw, device=DEV) / (H * Kw) ** 0.5
    bias = torch.randn(2 * H, device=DEV)
    f, g = _raw_operands(w)
    h = torch.full((B, T, 2 * H), float("nan"), device=DEV) if save_h else None
    out = torch.full((B, T, H), float("nan"), device=DEV)
    _run(x, f, bias, 0, B, T, H, 2 * H, Kw, 1, 1, 1, 0, 0, h, None, out, None)
    ref_h = _ref_conv(x, w, bias, 1)
    if save_h:
        assert rel_err(h.cpu(), ref_h.cpu()) < TOL
    ref_out = ref_h[..., :H] * torch.sigmoid(ref_h[..., H:])
    assert rel_err(out.cpu(), ref_out.cpu()) < TOL
    # data gradient dx[b,t,i] = sum_{o,j} w[o,i,j] dy[b,t-(j-1)d,o], plain store and in-place accumulation (K = 1920)
    dy = torch.randn(B, T, 2 * H, device=DEV)
    ref_dx = torch.nn.functional.conv_transpose1d(dy.double().permute(0, 2, 1), w.double(), padding=1).permute(0, 2, 1)
    dx = torch.full((B, T, H), float("nan"), device=DEV)
    _run(dy, g, None, 0, B, T, 2 * H, H, Kw, 1, -1, 0, 0, 0, dx, None, None, None)
    e = rel_err(dx.cpu(), ref_dx.cpu())
    print(f"[convp dgrad K=1920 B={B} T={T}] rel_err vs fp64 = {e:.2e}")
    assert e < TOL
    acc0 = torch.randn(B, T, H, device=DEV)
    acc = acc0.clone()
    _run(dy, g, None, 1, B, T, 2 * H, H, Kw, 1, -1, 0, 0, 0, acc, None, None, None)
    assert rel_err(acc.cpu(), (ref_dx + acc0.double()).cpu()) < TOL


@pytest.mark.parametrize("B,T", [(2, 360), (3, 101)])
def test_head_modes(B, T):
    """K5: 1x1 320->640 with GELU + saved pre-activation, then 1x1 640->1024 stored channel-major (the estimate)."""
    torch.manual_seed(3)
    H, F = 320, 1024
    x = torch.randn(B, T, H, device=DEV)
    w0 = torch.randn(2 * H, H, 1, device=DEV) / H ** 0.5
    b0 = torch.randn(2 * H, device=DEV)
    f0, _ = _raw_operands(w0)
    q = torch.full((B, T, 2 * H), float("nan"), device=DEV)
    h1 = torch.full((B, T, 2 * H), float("nan"), device=DEV)
    _run(x, f0, b0, 0, B, T, H, 2 * H, 1, 1, 1, 0, 1, 0, q, h1, None, None)
    ref_h1 = _ref_conv(x, w0, b0, 1)
    assert rel_err(h1.cpu(), ref_h1.cpu()) < TOL
    assert rel_err(q.cpu(), torch.nn.functional.gelu(ref_h1).cpu()) < TOL
    q2 = torch.full((B, T, 2 * H), float("nan"), device=DEV)
    _run(x, f0, b0, 0, B, T, H, 2 * H, 1, 1, 1, 0, 1, 0, q2, None, None, None)      # pre-activation not wanted (eval)
    assert torch.equal(q, q2)
    w2 = torch.randn(F, 2 * H, 1, device=DEV) / (2 * H) ** 0.5
    b2 = torch.randn(F, device=DEV)
    f2, _ = _raw_operands(w2)
    est = torch.full((B, F, T), float("nan"), device=DEV)
    _run(q, f2, b2, 0, B, T, 2 * H, F, 1, 1, 1, 0, 0, 1, est, None, None, None)
    ref = _ref_conv(q, w2, b2, 1).permute(0, 2, 1)
    assert rel_err(est.cpu(), ref.cpu()) < TOL


def test_fused_weight_split_matches_two_steps(pipe):
    """bm_tc_weight_split_f16 (one launch) == bm_tc_weight_split (re-layout) + bm_f16_split, bit for bit."""
    if pipe != "f16":
        pytest.skip("one run is enough")
    call, ptr, stream = _abi()
    torch.manual_seed(3)
    for Cout, Cin, Kw in ((320, 320, 3), (640, 320, 3), (1024, 640, 1)):
        w = torch.randn(Cout, Cin, Kw, device=DEV) * 0.02
        f, g = _raw_operands(w)
        amax = torch.empty(1, device=DEV)
        call("bm_amax", ptr(w), w.numel(), ptr(amax), stream())
        outs = [torch.empty(t.shape, device=DEV, dtype=torch.float16) for t in (f, f, g, g)]
        call("bm_f16_split", ptr(f), f.numel(), ptr(amax), ptr(outs[0]), ptr(outs[1]), stream())
        call("bm_f16_split", ptr(g), g.numel(), ptr(amax), ptr(outs[2]), ptr(outs[3]), stream())
        fused = [torch.full(t.shape, float("nan"), device=DEV, dtype=torch.float16) for t in (f, f, g, g)]
        call("bm_tc_weight_split_f16", ptr(w), ptr(amax), Cout, Cin, Kw, ptr(fused[0]), ptr(fused[1]), ptr(fused[2]),
             ptr(fused[3]), stream())
        for a, b in zip(outs, fused):
            assert torch.equal(a, b)


def test_producers_report_amax(pipe):
    """The elementwise kernels in front of a conv leave max |output| in `amax_out` (no separate pass over the tensor)."""
    if pipe != "f16":
        pytest.skip("one run is enough")
    call, ptr, stream = _abi()
    torch.manual_seed(5)
    for rows, C in ((360 * 7 + 13, 320), (97, 64), (1000, 100)):             # column-stationary kernels and the generic ones
        y, x_old = torch.randn(rows, C, device=DEV) * 3, torch.randn(rows, C, device=DEV)
        mean, invstd = torch.randn(C, device=DEV) * 0.1, torch.rand(C, device=DEV) + 0.5
        gamma, beta = torch.randn(C, device=DEV), torch.randn(C, device=DEV) * 0.1
        x_new = torch.empty(rows, C, device=DEV)
        cell = torch.full((1,), float("nan"), device=DEV)
        call("bm_bn_gelu_skip_fwd", ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), ptr(x_old), ptr(x_new), rows, C,
             ptr(cell), stream())
        assert float(cell) == float(x_new.abs().max())
        g = torch.randn(rows, C, device=DEV) * 1e-3
        sums = torch.empty(2 * C, device=DEV, dtype=torch.float64)
        dy, dgamma, dbeta = torch.empty(rows, C, device=DEV), torch.empty(C, device=DEV), torch.empty(C, device=DEV)
        call("bm_bn_gelu_skip_bwd", ptr(g), ptr(y), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta), 1, rows, C, ptr(sums),
             ptr(dy), ptr(dgamma), ptr(dbeta), ptr(cell), stream())
        assert float(cell) == float(dy.abs().max())
        if C % 2 == 0:
            H = C // 2
            gg = torch.randn(rows, H, device=DEV)
            dh, dbias = torch.empty(rows, C, device=DEV), torch.empty(C, device=DEV)
            call("bm_glu_bwd", ptr(gg), ptr(y), rows, H, ptr(dh), ptr(dbias), ptr(cell), stream())
            assert float(cell) == float(dh.abs().max())
    z = torch.zeros(64, 320, device=DEV)                                      # an all-zero tensor reports 0 (scale 1)
    cell = torch.full((1,), float("nan"), device=DEV)
    call("bm_amax", ptr(z), z.numel(), ptr(cell), stream())
    assert float(cell) == 0.0


def test_speed_report(capsys):
    """Not a pass/fail on speed: per-launch times at the BASELINE shape (B=256, T=360), L2 flushed between launches."""
    call, ptr, stream = _abi()
    B, T, C, Kw = 256, 360, 320, 3
    x = torch.randn(B, T, C, device=DEV)
    w = torch.randn(C, C, Kw, device=DEV) / (C * Kw) ** 0.5
    wg = torch.randn(2 * C, C, Kw, device=DEV) / (C * Kw) ** 0.5
    f, g = _raw_operands(w)
    fg, gg = _raw_operands(wg)
    y = torch.empty(B, T, C, device=DEV)
    h = torch.empty(B, T, 2 * C, device=DEV)
    stats = torch.empty(2 * C, device=DEV, dtype=torch.float64)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=DEV)
    st = stream()

    def launcher(xt, w_op, acc, Cin, Ntot, dil, sign, glu, yt, glu_out, stats_t, Bn=B, Tn=T):
        """A closure that launches ONLY the conv kernel (f16: the operand preparation is done here, once)."""
        if PIPE == "f16":
            amax, hi, lo = _f16_operands(xt, w_op)
            out_cell = torch.empty(1, device=DEV)
            return lambda: call("bm_tc_conv1d_f16", ptr(xt), ptr(amax[0:1]), ptr(hi), ptr(lo), ptr(amax[1:2]), None, acc, Bn,
                                Tn, Cin, Ntot, Kw, dil, sign, glu, 0, 0, ptr(yt), None, ptr(glu_out), ptr(stats_t),
                                ptr(out_cell) if glu else None, ptr(status), st)
        return lambda: call("bm_tc_conv1d_persistent", ptr(xt), ptr(w_op), None, acc, Bn, Tn, Cin, Ntot, Kw, dil, sign, glu,
                            0, 0, ptr(yt), None, ptr(glu_out), ptr(stats_t), ptr(status), st)

    k3 = launcher(x, f, 0, C, C, 4, 1, 0, y, None, stats)
    k3_acc = launcher(x, g, 1, C, C, 4, -1, 0, y, None, None)
    k4 = launcher(x, fg, 0, C, 2 * C, 1, 1, 1, h, y, None)
    k4_dgrad = launcher(h, gg, 0, 2 * C, C, 1, -1, 0, y, None, None)
    amax_cell = torch.empty(1, device=DEV)

    def amax_pass():
        call("bm_amax", ptr(x), x.numel(), ptr(amax_cell), st)

    lines = []
    for name, fn, flops in [(f"{PIPE} K3 persistent +stats", k3, 2.0 * C * C * Kw * T * B),
                            ("K3 dgrad accumulate", k3_acc, 2.0 * C * C * Kw * T * B),
                            ("K4 GLU (h saved)", k4, 4.0 * C * C * Kw * T * B),
                            ("K4 dgrad (K=1920)", k4_dgrad, 4.0 * C * C * Kw * T * B),
                            ("bm_amax over one activation tensor (118 MB)", amax_pass, 0.0)]:
        times = []
        for i in range(13):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                times.append(e0.elapsed_time(e1))
        ms = sum(times) / len(times)
        lines.append(f"[{name}] {ms:.4f} ms/launch = {flops / ms / 1e9:.1f} algorithmic TFLOP/s (min {min(times):.4f} ms)")
    # time = fixed + per-tile work: T = 256 makes two 128-row tiles per sample, so the tile count grows linearly with B
    Tt = 256
    xs = torch.randn(370, Tt, C, device=DEV)
    ys = torch.empty(370, Tt, C, device=DEV)
    fit = []
    for k in (1, 2, 3, 4, 5):
        Bk = 74 * k
        fn_k = launcher(xs, f, 0, C, C, 4, 1, 0, ys, None, None, Bn=Bk, Tn=Tt)
        times = []
        for i in range(9):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn_k()
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                times.append(e0.elapsed_time(e1))
        fit.append((k, min(times) * 1e3))
    per_tile = (fit[-1][1] - fit[0][1]) / 4
    lines.append("[K3 persistent, k tiles per pair -> us] " + ", ".join(f"{k}: {t:.1f}" for k, t in fit) +
                 f"  => per tile {per_tile:.2f} us, fixed {fit[0][1] - per_tile:.1f} us "
                 f"(57 600 MMA cycles per tile: {57600 / per_tile / 1e3:.2f} GHz-equivalent)")
    assert int(status.item()) == 0
    with capsys.disabled():
        print("\n" + "\n".join(lines))
