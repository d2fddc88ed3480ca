"""GPU: the conv engine (csrc/tc_common.cuh hc_conv_kernel: activations by TMA, split into tf32 pieces in registers) at the
edges of its tiles, for all three weight formats (raw fp32: bm_tc_conv1d_persistent; pre-split tf32 hi + lo: bm_tc_conv1d,
bm_tc_pointwise_sel, bm_tc_sensor_mix_bwd_data; fp16 pieces: bm_tc_conv1d_f16).  Every output element is checked against
torch's fp64 conv (test-only reference), scaled by the fp64 sum of |products| that forms it.

The edges: 160-wide tiles (320 columns: 2 exact tiles; 288: a partial last tile; GLU 80 'a' columns + their gates) and
128-wide ones (1024 columns, GLU with H = 128); T = 360 (a 104-row last time tile), 50 and 1; a dilation above 128, so that
whole shifted tap tiles fall outside the sample and arrive as TMA's zero fill; the data gradient (sign -1); per-sample
weight sets including an out-of-range set index; every epilogue mode, including the BatchNorm statistics of 160-wide tiles
and the channel-major store."""
import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-5
DEV = "cuda"


def _abi():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream


def _ref(x, wop, dil, sign):
    """y[b,t,n] = sum_tap sum_k x[b, t + sign*(tap - K//2)*dil, k] wop[tap,n,k] in fp64, and the same over |x| |w|."""
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


def _close(got, ref, scale, what):
    bad = (got.double() - ref).abs() > TOL * scale + 1e-30
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at {bad.nonzero()[0].tolist()}"


def _weights(fmt, Ntot, Cin, Kw):
    """K-major operand wop [Kw][Ntot][Cin] and what the entry point of `fmt` takes for it."""
    call, ptr, stream = _abi()
    w = torch.randn(Ntot, Cin, Kw, device=DEV) * 0.05                     # nn.Conv1d layout
    wop = w.permute(2, 0, 1).contiguous()
    if fmt == "raw":
        return wop, (wop,)
    if fmt == "split":
        hi, lo = torch.empty_like(wop), torch.empty_like(wop)
        call("bm_tc_weight_split", ptr(w), Ntot, Cin, Kw, ptr(hi), ptr(lo), None, None, stream())
        return wop, (hi, lo)
    amax = torch.empty(1, device=DEV)
    hi = torch.empty(wop.shape, device=DEV, dtype=torch.float16)
    lo = torch.empty(wop.shape, device=DEV, dtype=torch.float16)
    call("bm_amax", ptr(wop), wop.numel(), ptr(amax), stream())
    call("bm_f16_split", ptr(wop), wop.numel(), ptr(amax), ptr(hi), ptr(lo), stream())
    return wop, (hi, lo, amax)


def _conv(fmt, ops, x, bias, addend, B, T, Cin, Ntot, Kw, dil, sign, glu, act, tmajor, y, aux, glu_out, stats):
    call, ptr, stream = _abi()
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    acc = int(addend is not None)
    if fmt == "raw":
        call("bm_tc_conv1d_persistent", ptr(x), ptr(ops[0]), ptr(bias), acc, B, T, Cin, Ntot, Kw, dil, sign, glu, act, tmajor,
             ptr(y), ptr(aux), ptr(glu_out), ptr(stats), ptr(status), stream())
    elif fmt == "split":
        call("bm_tc_conv1d", ptr(x), ptr(ops[0]), ptr(ops[1]), ptr(bias), ptr(addend), B, T, Cin, Ntot, Kw, dil, sign, glu,
             act, tmajor, ptr(y), ptr(aux), ptr(glu_out), None, ptr(status), stream())
    else:
        xa = torch.empty(1, device=DEV)
        call("bm_amax", ptr(x), x.numel(), ptr(xa), stream())
        call("bm_tc_conv1d_f16", ptr(x), ptr(xa), ptr(ops[0]), ptr(ops[1]), ptr(ops[2]), ptr(bias), acc, B, T, Cin, Ntot,
             Kw, dil, sign, glu, act, tmajor, ptr(y), ptr(aux), ptr(glu_out), ptr(stats), None, ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"status {int(status.item())}"


# (B, T, Cin, Ntot, Kw, dil, sign, mode); the raw and fp16 entry points take widths that are multiples of 256 or 320
# (GLU: H a multiple of 128 or 160), the pre-split one multiples of 16 with a divisor in [64, 160] (GLU: H of 80)
PAIR_CASES = [
    (3, 360, 320, 320, 3, 4, 1, "stats"),
    (2, 50, 320, 320, 3, 200, -1, "accumulate"),
    (4, 1, 64, 320, 3, 1, 1, "gelu"),
    (3, 360, 320, 640, 3, 2, 1, "glu"),
    (2, 50, 96, 256, 3, 1, -1, "glu"),
    (2, 50, 320, 1024, 1, 1, 1, "tmajor"),
]
SPLIT_CASES = [
    (3, 360, 320, 288, 3, 2, -1, "addend"),
    (2, 50, 64, 160, 3, 1, 1, "glu"),
    (2, 1, 96, 1024, 3, 130, 1, "gelu"),
    (3, 360, 320, 320, 3, 1, 1, "tmajor"),
]


@pytest.mark.parametrize("fmt,case", [(f, c) for f in ("raw", "f16") for c in PAIR_CASES] +
                         [("split", c) for c in SPLIT_CASES])
def test_conv_edges(fmt, case):
    B, T, Cin, Ntot, Kw, dil, sign, mode = case
    torch.manual_seed(len(fmt) + B * T + Ntot + dil)
    x = torch.randn(B, T, Cin, device=DEV)
    wop, ops = _weights(fmt, Ntot, Cin, Kw)
    ref, absref = _ref(x, wop, dil, sign)
    glu = int(mode == "glu")
    act = int(mode == "gelu")
    tmajor = int(mode == "tmajor")
    bias = None if mode == "accumulate" else torch.randn(Ntot, device=DEV)
    if bias is not None:
        ref, absref = ref + bias.double(), absref + bias.double().abs()
    addend = None
    y = torch.full((B, T, Ntot), float("nan"), device=DEV)
    if mode in ("accumulate", "addend"):
        addend = torch.randn(B, T, Ntot, device=DEV)
        ref, absref = ref + addend.double(), absref + addend.double().abs()
        if mode == "accumulate":
            y = addend.clone()              # y += conv, in place
        else:
            y = torch.full_like(addend, float("nan"))
    aux = torch.full((B, T, Ntot), float("nan"), device=DEV) if act else None
    glu_out = torch.full((B, T, Ntot // 2), float("nan"), device=DEV) if glu else None
    stats = torch.full((2 * Ntot,), float("nan"), device=DEV, dtype=torch.float64) if mode == "stats" else None
    if tmajor:
        y = torch.full((B, Ntot, T), float("nan"), device=DEV)
    _conv(fmt, ops, x, bias, addend if mode == "addend" else (y if mode == "accumulate" else None), B, T, Cin, Ntot, Kw,
          dil, sign, glu, act, tmajor, y, aux, glu_out, stats)
    if glu:
        H = Ntot // 2
        _close(y, ref, absref, "h")
        a, g = ref[..., :H], ref[..., H:]
        o = a * torch.sigmoid(g)
        _close(glu_out, o, absref[..., :H] + a.abs() * absref[..., H:], "GLU output")
    elif act:
        _close(aux, ref, absref, "pre-activation")
        _close(y, torch.nn.functional.gelu(ref), 1.2 * absref, "GELU output")
    elif tmajor:
        _close(y.permute(0, 2, 1), ref, absref, "channel-major y")
    else:
        _close(y, ref, absref, "y")
    if stats is not None:
        yd = y.double().reshape(-1, Ntot)
        s = torch.cat([yd.sum(0), (yd * yd).sum(0)])
        # the epilogue sums 16 values per column in fp32 before its fp64 atomics
        bad = (stats - s).abs() > 2e-6 * torch.cat([yd.abs().sum(0), (yd * yd).sum(0)])
        assert not bad.any(), f"BatchNorm statistics: columns {bad.nonzero().flatten().tolist()[:8]} off"


def _set_weights(S, Ntot, Cin):
    """S weight sets [S][Ntot][Cin] and their tf32 pieces."""
    call, ptr, stream = _abi()
    w = torch.randn(S, Ntot, Cin, 1, device=DEV) * 0.05
    hi, lo = torch.empty(S, Ntot, Cin, device=DEV), torch.empty(S, Ntot, Cin, device=DEV)
    for s in range(S):
        call("bm_tc_weight_split", ptr(w[s]), Ntot, Cin, 1, ptr(hi[s]), ptr(lo[s]), None, None, stream())
    return w[..., 0], hi, lo


@pytest.mark.parametrize("T,Ntot", [(360, 320), (50, 288), (1, 1024)])
def test_pointwise_weight_sets(T, Ntot):
    """bm_tc_pointwise_sel: y[b] = x[b] W[wsel[b]]^T; an index outside the sets reports 900."""
    call, ptr, stream = _abi()
    torch.manual_seed(T + Ntot)
    B, Cin, S = 5, 256, 3
    w, hi, lo = _set_weights(S, Ntot, Cin)
    x = torch.randn(B, T, Cin, device=DEV)
    wsel = torch.tensor([2, 0, 1, 2, 0], dtype=torch.int32, device=DEV)
    y = torch.full((B, T, Ntot), float("nan"), device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    call("bm_tc_pointwise_sel", ptr(x), ptr(hi), ptr(lo), ptr(wsel), S, B, T, Cin, Ntot, ptr(y), ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    wd = w.double()[wsel.long()]
    _close(y, torch.einsum("btk,bnk->btn", x.double(), wd), torch.einsum("btk,bnk->btn", x.double().abs(), wd.abs()), "y")
    wsel[3] = S
    call("bm_tc_pointwise_sel", ptr(x), ptr(hi), ptr(lo), ptr(wsel), S, B, T, Cin, Ntot, ptr(y), ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 900


def test_sensor_mix_bwd_data_partial_tile():
    """bm_tc_sensor_mix_bwd_data with Cp = 288 (a partial 160-wide tile): dmeg[b,c,t] = mask[c] sum_o du[b,t,o] W[rec][c][o]."""
    call, ptr, stream = _abi()
    torch.manual_seed(11)
    B, T, Op, Cp, C, S = 3, 360, 320, 288, 273, 2
    w, hi, lo = _set_weights(S, Cp, Op)
    du = torch.randn(B, T, Op, device=DEV)
    wsel = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
    mask = (torch.rand(C, device=DEV) > 0.2).float()
    dmeg = torch.full((B, C, T), float("nan"), device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    call("bm_tc_sensor_mix_bwd_data", ptr(du), ptr(hi), ptr(lo), ptr(wsel), S, ptr(mask), B, T, Op, Cp, C, ptr(dmeg),
         ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    wd = w.double()[wsel.long()][:, :C]
    ref = torch.einsum("bto,bco->bct", du.double(), wd) * mask.double()[None, :, None]
    scale = torch.einsum("bto,bco->bct", du.double().abs(), wd.abs())
    _close(dmeg, ref, scale, "dmeg")
