"""GPU: the edges of the conv epilogue (csrc/tc_conv.cuh ConvOp::epilogue), which loads a column group's bias and addend
before its first store, stores adjacent column pairs as float2 and sums the BatchNorm statistics per warp before one fp64
add per column.  In both pass counts (3xTF32 and the `_tf32` form):

  * a partial last column tile (Ntot = 448 on 160-wide tiles: 2 full tiles and 128 of 160 columns), through
    bm_tc_conv1d, in every row-major epilogue mode and channel-major, against torch's fp64 conv;
  * the BatchNorm statistics of bm_tc_conv1d_persistent against the kernel's own y at T = 343, summed as the kernel
    sums them: the fp32 sum of each thread's two rows, the fp32 shuffle tree over a warp's 8 row lanes, then fp64;
  * in-place accumulation (and a separate skip addend) holding NaN and +-Inf: each reaches exactly the element it sits on.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {3: 1e-5, 1: 3e-3}          # 3xTF32 ~ fp32; TF32: each operand rounded to 11 significant bits


def _abi():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream


def _suffix(passes):
    return "" if passes == 3 else "_tf32"


def _ref(x, wop, dil, sign):
    """fp64 conv of x [B,T,Cin] with wop [K,N,Cin] (tap shift sign*(tap-K//2)*dil), and the same over |x| |w|"""
    B, T, _ = x.shape
    K, N, _ = wop.shape
    xd, wd = x.double(), wop.double()
    y = torch.zeros(B, T, N, dtype=torch.float64, device=DEV)
    a = torch.zeros_like(y)
    for tap in range(K):
        s = sign * (tap - K // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        if lo < hi:
            y[:, lo:hi] += xd[:, lo + s:hi + s] @ wd[tap].T
            a[:, lo:hi] += xd[:, lo + s:hi + s].abs() @ wd[tap].abs().T
    return y, a


def _close(got, ref, scale, tol, what):
    bad = (got.double() - ref).abs() > tol * scale + 1e-30
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at {bad.nonzero()[0].tolist()}"


def _split(wop):
    """tf32 pieces [K][N][Cin] of the nn.Conv1d weight whose K-major re-layout is wop"""
    call, ptr, stream = _abi()
    K, N, Cin = wop.shape
    hi, lo = torch.empty_like(wop), torch.empty_like(wop)
    call("bm_tc_weight_split", ptr(wop.permute(1, 2, 0).contiguous()), N, Cin, K, ptr(hi), ptr(lo), None, None, stream())
    return hi, lo


def _with_specials(y0):
    """y0 with NaN, +Inf and -Inf scattered over rows and columns (including the last column and the partial tile)"""
    y0 = y0.clone()
    flat = y0.view(-1)
    idx = torch.randperm(flat.numel(), device=DEV)[:3 * 97]
    flat[idx[:97]] = float("nan")
    flat[idx[97:194]] = float("inf")
    flat[idx[194:]] = -float("inf")
    y0[:, :, -1] = float("nan")
    y0[-1, -1, :] = float("inf")
    return y0


def _check_specials(got, addend, what):
    assert torch.equal(torch.isnan(got), torch.isnan(addend)), f"{what}: NaN where the addend has none, or lost"
    for s in (1, -1):
        assert torch.equal(got == s * float("inf"), addend == s * float("inf")), f"{what}: {s:+d} Inf misplaced"


# (mode, T, dil, sign): Ntot = 448 on 160-wide column tiles, the last one partial
PARTIAL = [("plain", 343, 2, 1), ("skip", 200, 1, -1), ("gelu", 130, 1, 1), ("tmajor", 100, 1, 1)]


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("case", PARTIAL, ids=[c[0] for c in PARTIAL])
def test_partial_column_tile(passes, case):
    call, ptr, stream = _abi()
    mode, T, dil, sign = case
    B, Cin, Ntot, Kw = 3, 64, 448, 3 if mode != "gelu" else 1
    torch.manual_seed(41)
    x = torch.randn(B, T, Cin, device=DEV)
    wop = torch.randn(Kw, Ntot, Cin, device=DEV) * 0.05
    bias = torch.randn(Ntot, device=DEV)
    hi, lo = _split(wop)
    addend = _with_specials(torch.randn(B, T, Ntot, device=DEV)) if mode == "skip" else None
    act, tmaj = int(mode == "gelu"), int(mode == "tmajor")
    y = torch.full((B, Ntot, T) if tmaj else (B, T, Ntot), float("nan"), device=DEV)
    aux = torch.full((B, T, Ntot), float("nan"), device=DEV) if act else None
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    call("bm_tc_conv1d" + _suffix(passes), ptr(x), ptr(hi), ptr(lo), ptr(bias), ptr(addend), B, T, Cin, Ntot, Kw, dil,
         sign, 0, act, tmaj, ptr(y), ptr(aux), None, None, ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    ref, scale = _ref(x, wop, dil, sign)
    ref, scale = ref + bias.double(), scale + bias.double().abs()
    tol = TOL[passes]
    if mode == "skip":
        _check_specials(y, addend, "skip addend")
        fin = torch.isfinite(addend)
        _close(y[fin], (ref + addend.double())[fin], (scale + addend.double().abs())[fin], tol, "y + addend")
    elif mode == "gelu":
        _close(aux, ref, scale, tol, "pre-activation")
        _close(y, torch.nn.functional.gelu(ref), 1.2 * scale, tol, "GELU output")
    elif mode == "tmajor":
        _close(y.permute(0, 2, 1), ref, scale, tol, "channel-major y")
    else:
        _close(y, ref, scale, tol, "y")


def _persistent(passes, x, wop, bias, acc, T, Ntot, Kw, dil, sign, y, stats):
    call, ptr, stream = _abi()
    B, _, Cin = x.shape
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    call("bm_tc_conv1d_persistent" + _suffix(passes), ptr(x), ptr(wop), ptr(bias), acc, B, T, Cin, Ntot, Kw, dil, sign,
         0, 0, 0, ptr(y), None, None, ptr(stats), ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"status {int(status.item())}"


def _kernel_order_stats(y, bias):
    """column sum and sum of squares of y [B,T,N] in the kernel's order: d = y - bias in fp32, per thread (0 + d_r) + d_r+8
    and fma(d_r+8, d_r+8, fma(d_r, d_r, 0)) in fp32, a fp32 tree over the 8 row lanes of a warp (lane groups 1, 2, 4
    apart), fp64 over the warps; then per time tile of n rows, sum = n b + d1 and sum of squares = d2 + b (n b + 2 d1) in
    fp64; rows past T are zeros of d, which change no sum"""
    B, T, N = y.shape
    tt = (T + 127) // 128
    yp = torch.zeros(B, tt * 128, N, device=DEV)
    yp[:, :T] = y - bias
    v = yp.view(B, tt, 8, 2, 8, N)                             # [b][time tile][warp][row half h][row lane][n]
    v0, v1 = v[:, :, :, 0], v[:, :, :, 1]
    s1 = v0 + v1
    sq0 = (v0.double() * v0.double()).float()                  # fma(v, v, 0): the exact square, rounded once
    s2 = (v1.double() * v1.double() + sq0.double()).float()    # fma(v, v, s): exact in fp64 but for rare ties
    d = []
    for s in (s1, s2):
        s = s[:, :, :, 0::2] + s[:, :, :, 1::2]                # lanes 4 apart: row lanes k, k ^ 1
        s = s[:, :, :, 0::2] + s[:, :, :, 1::2]
        s = s[:, :, :, 0] + s[:, :, :, 1]                      # [b][tile][warp][n]
        d.append(s.double().sum(dim=2))                        # [b][tile][n]
    rows = torch.tensor([min(128, T - 128 * i) for i in range(tt)], device=DEV, dtype=torch.float64)[None, :, None]
    b = bias.double()
    tile_sum = rows * b + d[0]
    tile_sq = d[1] + b * (rows * b + 2 * d[0])
    want = torch.cat([tile_sum.sum(dim=(0, 1)), tile_sq.sum(dim=(0, 1))])
    yd = y.double()
    return want, torch.cat([yd.abs().sum(dim=(0, 1)), (yd ** 2).sum(dim=(0, 1))])


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("Ntot", [320, 256])
@pytest.mark.parametrize("bias_scale", [1.0, 1e3, None])
def test_batchnorm_statistics_bias_shifted_match_own_output(passes, Ntot, bias_scale):
    """the fused statistics are the bias-shifted sums of the kernel's own y, in its order, to fp64 rounding; with no bias,
    with a unit one and with one 1e3 times the conv's spread (where unshifted fp32 sums of y^2 would lose the variance)"""
    torch.manual_seed(43)
    B, T, Cin, Kw = 23, 343, 320, 3
    x = torch.randn(B, T, Cin, device=DEV)
    wop = torch.randn(Kw, Ntot, Cin, device=DEV) * 0.05
    bias = None if bias_scale is None else torch.randn(Ntot, device=DEV) * bias_scale
    y = torch.full((B, T, Ntot), float("nan"), device=DEV)
    stats = torch.full((2 * Ntot,), float("nan"), device=DEV, dtype=torch.float64)
    _persistent(passes, x, wop, bias, 0, T, Ntot, Kw, 2, 1, y, stats)
    assert torch.isfinite(y).all()
    want, scale = _kernel_order_stats(y, torch.zeros(Ntot, device=DEV) if bias is None else bias)
    bad = (stats - want).abs() > 1e-10 * scale
    assert not bad.any(), f"columns {bad.nonzero().flatten().tolist()[:8]} off by {(stats - want).abs().max().item()}"


@pytest.mark.parametrize("passes", [3, 1])
def test_in_place_accumulate_with_nan_and_inf(passes):
    torch.manual_seed(47)
    B, T, Cin, Ntot, Kw = 5, 343, 320, 320, 3
    x = torch.randn(B, T, Cin, device=DEV)
    wop = torch.randn(Kw, Ntot, Cin, device=DEV) * 0.05
    y0 = _with_specials(torch.randn(B, T, Ntot, device=DEV))
    y = y0.clone()
    _persistent(passes, x, wop, None, 1, T, Ntot, Kw, 1, -1, y, None)
    _check_specials(y, y0, "in-place accumulate")
    ref, scale = _ref(x, wop, 1, -1)
    fin = torch.isfinite(y0)
    _close(y[fin], (ref + y0.double())[fin], (scale + y0.double().abs())[fin], TOL[passes], "y += conv")
