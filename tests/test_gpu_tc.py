"""GPU: the tensor-core (3xTF32) conv kernels against the FP32-FMA kernels of the same library and against torch's
fp64 conv (test-only reference), at the real layer shapes.  Tolerance 3e-5 relative to fp64: the 3xTF32 scheme
must stay fp32-faithful, inside the 1e-4 parity bar (measured ~1e-5 at K=1920: the tensor-core fp32 accumulator
truncates, so the error grows with the accumulation length)."""
TOL = 3e-5
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _reset_debug_flags():
    yield
    from brainmagick_b200 import _lib
    _lib.load().bm_set_debug_flags(0)


def _call():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream


_FN = {1: "bm_tc_conv1d"}


def _gen_flags(gen):
    """generation 1 = the pre-split-weight entry point (bm_tc_conv1d, still used with per-sample weight sets); the raw-weight
    entry point has its own file, tests/test_gpu_convp.py."""
    from brainmagick_b200 import _lib
    _lib.load().bm_set_debug_flags(0)


def _ref_conv(x, w, bias, dilation):
    """x [B,T,Cin] channels-last, w [Cout,Cin,Kw] -> y [B,T,Cout] in fp64 (torch, test-only)."""
    y = torch.nn.functional.conv1d(x.double().permute(0, 2, 1), w.double(), None if bias is None else bias.double(),
                                   padding=(w.shape[2] // 2) * dilation, dilation=dilation)
    return y.permute(0, 2, 1).contiguous()


@pytest.mark.parametrize("gen", [1])
@pytest.mark.parametrize("dilation", [1, 2, 16])
@pytest.mark.parametrize("T", [360, 343, 100])
def test_tc_conv_forward(dilation, T, gen):
    call, ptr, stream = _call()
    _gen_flags(gen)
    torch.manual_seed(dilation * 1000 + T)
    B, Cin, Cout, Kw = 3, 320, 320, 3
    dev = "cuda"
    x = torch.randn(B, T, Cin, device=dev)
    w = torch.randn(Cout, Cin, Kw, device=dev) / (Cin * Kw) ** 0.5
    bias = torch.randn(Cout, device=dev)
    fh = torch.empty(Kw, Cout, Cin, device=dev)
    fl = torch.empty(Kw, Cout, Cin, device=dev)
    call("bm_tc_weight_split", ptr(w), Cout, Cin, Kw, ptr(fh), ptr(fl), None, None, stream())
    y = torch.full((B, T, Cout), float("nan"), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    call(_FN[gen], ptr(x), ptr(fh), ptr(fl), ptr(bias), None, B, T, Cin, Cout, Kw, dilation, 1, 0, 0, 0, ptr(y), None, None,
         None, ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"tensor-core kernel timed out at barrier code {int(status.item())}"
    ref = _ref_conv(x, w, bias, dilation)
    err = rel_err(y.cpu(), ref.cpu())
    print(f'[tc gen{gen} fwd d={dilation} T={T}] rel_err vs fp64 = {err:.2e}')
    assert err < TOL, err


@pytest.mark.parametrize("gen", [1])
def test_tc_conv_glu_and_data_gradient(gen):
    call, ptr, stream = _call()
    _gen_flags(gen)
    torch.manual_seed(7)
    B, T, H, Kw = 2, 360, 320, 3
    dev = "cuda"
    x = torch.randn(B, T, H, device=dev)
    w = torch.randn(2 * H, H, Kw, device=dev) / (H * Kw) ** 0.5
    bias = torch.randn(2 * H, device=dev)
    fh, gh = torch.empty(Kw, 2 * H, H, device=dev), torch.empty(Kw, H, 2 * H, device=dev)
    fl = torch.empty(Kw, 2 * H, H, device=dev)
    gl = torch.empty(Kw, H, 2 * H, device=dev)
    call("bm_tc_weight_split", ptr(w), 2 * H, H, Kw, ptr(fh), ptr(fl), ptr(gh), ptr(gl), stream())
    h = torch.empty(B, T, 2 * H, device=dev)
    out = torch.empty(B, T, H, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    call(_FN[gen], ptr(x), ptr(fh), ptr(fl), ptr(bias), None, B, T, H, 2 * H, Kw, 1, 1, 1, 0, 0, ptr(h), None, ptr(out),
         None, ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    ref_h = _ref_conv(x, w, bias, 1)
    assert rel_err(h.cpu(), ref_h.cpu()) < TOL
    ref_out = ref_h[..., :H] * torch.sigmoid(ref_h[..., H:])
    assert rel_err(out.cpu(), ref_out.cpu()) < TOL
    # data gradient: dx[b,t,i] = sum_{o,j} w[o,i,j] dy[b,t-(j-1)d,o] (+ addend)
    dy = torch.randn(B, T, 2 * H, device=dev)
    addend = torch.randn(B, T, H, device=dev)
    dx = torch.empty(B, T, H, device=dev)
    call(_FN[gen], ptr(dy), ptr(gh), ptr(gl), None, ptr(addend), B, T, 2 * H, H, Kw, 1, -1, 0, 0, 0, ptr(dx), None, None,
         None, ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    ref_dx = torch.nn.functional.conv_transpose1d(dy.double().permute(0, 2, 1), w.double(), padding=1).permute(0, 2, 1)
    ref_dx = ref_dx + addend.double()
    e = rel_err(dx.cpu(), ref_dx.cpu())
    print(f'[tc dgrad K=1920] rel_err vs fp64 = {e:.2e}')
    assert e < TOL
    # in-place skip-gradient accumulation (addend == output): the epilogue reads each element before it overwrites it
    acc = addend.clone()
    call(_FN[gen], ptr(dy), ptr(gh), ptr(gl), None, ptr(acc), B, T, 2 * H, H, Kw, 1, -1, 0, 0, 0, ptr(acc), None, None,
         None, ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    assert rel_err(acc.cpu(), ref_dx.cpu()) < TOL


@pytest.mark.parametrize("gen", [1])
def test_tc_conv_speed_report(capsys, gen):
    """Not a pass/fail on speed: prints the per-launch time at the BASELINE shape for the log."""
    call, ptr, stream = _call()
    _gen_flags(gen)
    B, T, C, Kw = 256, 360, 320, 3
    dev = "cuda"
    x = torch.randn(B, T, C, device=dev)
    w = torch.randn(C, C, Kw, device=dev) / (C * Kw) ** 0.5
    fh = torch.empty(Kw, C, C, device=dev)
    fl = torch.empty(Kw, C, C, device=dev)
    call("bm_tc_weight_split", ptr(w), C, C, Kw, ptr(fh), ptr(fl), None, None, stream())
    y = torch.empty(B, T, C, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    for _ in range(3):
        call(_FN[gen], ptr(x), ptr(fh), ptr(fl), None, None, B, T, C, C, Kw, 4, 1, 0, 0, 0, ptr(y), None, None, None, ptr(status), stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        call(_FN[gen], ptr(x), ptr(fh), ptr(fl), None, None, B, T, C, C, Kw, 4, 1, 0, 0, 0, ptr(y), None, None, None, ptr(status), stream())
    e1.record()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    ms = e0.elapsed_time(e1) / 10
    tf = 2.0 * C * C * Kw * T * B / (ms * 1e-3) / 1e12
    with capsys.disabled():
        print(f"\n[tc gen{gen} conv 320->320 k3 B=256 T=360] {ms:.3f} ms/launch = {tf:.1f} algorithmic TFLOP/s")


# `trunc` sets bm_set_debug_flags, which the ABI still accepts and no kernel reads any more: both settings must give the
# same, correct result.
@pytest.mark.parametrize("trunc", [0, 1])
@pytest.mark.parametrize("case", [
    dict(B=5, T=360, M=320, N=320, Kw=3, dil=1),
    dict(B=3, T=343, M=320, N=320, Kw=3, dil=16),
    dict(B=4, T=100, M=640, N=320, Kw=3, dil=2),
    dict(B=3, T=360, M=640, N=1024, Kw=1, dil=1),
])
def test_tc_wgrad(case, trunc):
    call, ptr, stream = _call()
    from brainmagick_b200 import _lib
    _lib.load().bm_set_debug_flags(trunc)
    torch.manual_seed(11)
    B, T, M, N, Kw, dil = (case[k] for k in ("B", "T", "M", "N", "Kw", "dil"))
    dev = "cuda"
    dy = torch.randn(B, T, M, device=dev)
    x = torch.randn(B, T, N, device=dev)
    ws = torch.empty(_lib.load().bm_tc_wgrad_workspace(B, M, N, Kw), device=dev)
    dw = torch.full((M, N, Kw), float("nan"), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    db = torch.full((M,), float("nan"), device=dev)
    call("bm_tc_wgrad", ptr(dy), ptr(x), B, T, M, N, N, Kw, dil, ptr(ws), ptr(dw), ptr(db), ptr(status), stream())
    torch.cuda.synchronize()
    _lib.load().bm_set_debug_flags(0)
    assert rel_err(db.cpu(), dy.double().sum(dim=(0, 1)).cpu()) < 1e-5
    assert int(status.item()) == 0, f"tensor-core kernel timed out at barrier code {int(status.item())}"
    # fp64 reference: dw[m,n,j] = sum_{b,t} dy[b,t,m] x[b,t+(j-Kw//2)*dil,n]
    ref = torch.zeros(M, N, Kw, dtype=torch.float64, device=dev)
    xd, dyd = x.double(), dy.double()
    for j in range(Kw):
        s = (j - Kw // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        ref[:, :, j] = torch.einsum("btm,btn->mn", dyd[:, lo:hi], xd[:, lo + s:hi + s])
    e = rel_err(dw.cpu(), ref.cpu())
    print(f"[tc wgrad rna_split={trunc} {case}] rel_err vs fp64 = {e:.2e}")
    assert e < TOL


@pytest.mark.parametrize("trunc", [0, 1])
def test_tc_wgrad_speed_report(capsys, trunc):
    call, ptr, stream = _call()
    from brainmagick_b200 import _lib
    _lib.load().bm_set_debug_flags(trunc)
    B, T, M, N, Kw = 256, 360, 320, 320, 3
    dev = "cuda"
    dy = torch.randn(B, T, M, device=dev)
    x = torch.randn(B, T, N, device=dev)
    ws = torch.empty(_lib.load().bm_tc_wgrad_workspace(B, M, N, Kw), device=dev)
    dw = torch.empty(M, N, Kw, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    for _ in range(3):
        call("bm_tc_wgrad", ptr(dy), ptr(x), B, T, M, N, N, Kw, 4, ptr(ws), ptr(dw), None, ptr(status), stream())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        call("bm_tc_wgrad", ptr(dy), ptr(x), B, T, M, N, N, Kw, 4, ptr(ws), ptr(dw), None, ptr(status), stream())
    e1.record()
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    ms = e0.elapsed_time(e1) / 10
    tf = 2.0 * M * N * Kw * T * B / (ms * 1e-3) / 1e12
    with capsys.disabled():
        _lib.load().bm_set_debug_flags(0)
        print(f"\n[tc wgrad rna_split={trunc} 320x320 k3 B=256 T=360] {ms:.3f} ms/launch = {tf:.1f} algorithmic TFLOP/s")


@pytest.mark.parametrize("case", [
    dict(B=5, T=360, M=320, N=320, Kw=3, dil=1),
    dict(B=3, T=343, M=320, N=320, Kw=3, dil=16),
    dict(B=4, T=100, M=640, N=320, Kw=3, dil=2),
    dict(B=7, T=77, M=320, N=320, Kw=3, dil=4),
    dict(B=3, T=360, M=1024, N=640, Kw=1, dil=1),
    dict(B=2, T=64, M=192, N=96, Kw=3, dil=1),
    dict(B=40, T=360, M=320, N=320, Kw=3, dil=8),
])
@pytest.mark.parametrize("pipe", ["tf32", "f16"])
def test_tc_wgrad_pair_kernel(case, pipe):
    """bm_tc_wgrad_conv and bm_tc_wgrad_conv_f16 (the entry point that also takes the operands' amax; csrc/tc_wgradp.cuh):
    rows = (tap, x channel), flattened reduction."""
    call, ptr, stream = _call()
    from brainmagick_b200 import _lib
    torch.manual_seed(11)
    B, T, M, N, Kw, dil = (case[k] for k in ("B", "T", "M", "N", "Kw", "dil"))
    dev = "cuda"
    assert _lib.load().bm_tc_wgrad_conv_supported(T, M, N, Kw)
    dy = torch.randn(B, T, M, device=dev)
    x = torch.randn(B, T, N, device=dev)
    ws = torch.full((int(_lib.load().bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)),), float("nan"), device=dev)
    dw = torch.full((M, N, Kw), float("nan"), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    if pipe == "f16":
        dy *= 3e-4                                                    # gradients are small: the per-tensor scales matter
        amax = torch.empty(2, device=dev)
        call("bm_amax", ptr(dy), dy.numel(), ptr(amax[0:1]), stream())
        call("bm_amax", ptr(x), x.numel(), ptr(amax[1:2]), stream())

        def run(out):
            call("bm_tc_wgrad_conv_f16", ptr(dy), ptr(amax[0:1]), ptr(x), ptr(amax[1:2]), B, T, M, N, N, Kw, dil, ptr(ws),
                 ptr(out), ptr(status), stream())
    else:
        def run(out):
            call("bm_tc_wgrad_conv", ptr(dy), ptr(x), B, T, M, N, N, Kw, dil, ptr(ws), ptr(out), ptr(status), stream())
    run(dw)
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"tensor-core kernel timed out at barrier code {int(status.item())}"
    ref = torch.zeros(M, N, Kw, dtype=torch.float64, device=dev)
    xd, dyd = x.double(), dy.double()
    for j in range(Kw):
        s = (j - Kw // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        ref[:, :, j] = torch.einsum("btm,btn->mn", dyd[:, lo:hi], xd[:, lo + s:hi + s])
    e = rel_err(dw.cpu(), ref.cpu())
    print(f"[tc wgrad pair {pipe} {case}] rel_err vs fp64 = {e:.2e}")
    assert e < TOL
    dw2 = torch.empty_like(dw)
    run(dw2)
    torch.cuda.synchronize()
    assert torch.equal(dw, dw2)                                   # fixed-order reduction


def test_tc_wgrad_pair_speed_report(capsys):
    call, ptr, stream = _call()
    from brainmagick_b200 import _lib
    dev = "cuda"
    B, T, Kw = 256, 360, 3
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    lines = []
    for M, N in ((320, 320), (640, 320)):
        dy = torch.randn(B, T, M, device=dev)
        x = torch.randn(B, T, N, device=dev)
        dw = torch.empty(M, N, Kw, device=dev)
        ws_new = torch.empty(int(_lib.load().bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)), device=dev)
        ws_old = torch.empty(int(_lib.load().bm_tc_wgrad_workspace(B, M, N, Kw)), device=dev)
        amax = torch.empty(2, device=dev)
        call("bm_amax", ptr(dy), dy.numel(), ptr(amax[0:1]), stream())
        call("bm_amax", ptr(x), x.numel(), ptr(amax[1:2]), stream())
        for name, fn in (("fp16-piece entry", lambda: call("bm_tc_wgrad_conv_f16", ptr(dy), ptr(amax[0:1]), ptr(x),
                                                            ptr(amax[1:2]), B, T, M, N, N, Kw, 4, ptr(ws_new), ptr(dw),
                                                            ptr(status), stream())),
                         ("fp32 entry", lambda: call("bm_tc_wgrad_conv", ptr(dy), ptr(x), B, T, M, N, N, Kw, 4, ptr(ws_new),
                                                      ptr(dw), ptr(status), stream())),
                         ("per-tap kernel", lambda: call("bm_tc_wgrad", ptr(dy), ptr(x), B, T, M, N, N, Kw, 4, ptr(ws_old),
                                                          ptr(dw), None, ptr(status), stream()))):
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
            tf = 2.0 * M * N * Kw * T * B / (ms * 1e-3) / 1e12
            lines.append(f"[wgrad {M}x{N} k3 B=256 T=360, {name}] {ms:.4f} ms/launch = {tf:.1f} algorithmic TFLOP/s")
    assert int(status.item()) == 0
    with capsys.disabled():
        print("\n" + "\n".join(lines))
