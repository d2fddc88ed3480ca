"""GPU: the persistent tile walk of the conv engine (csrc/tc_common.cuh hc_conv_kernel: min(tiles, SMs) CTAs, CTA i computing
tiles i, i + grid, ...; the stage ring and barrier phases run on across tiles).  Every output element is checked against
torch's fp64 conv (test-only reference), scaled by the fp64 sum of |products| that forms it, in both pass counts (3xTF32
and the `_tf32` form), and a second launch must reproduce the first bit for bit.

Covered: tile counts below, equal to and not a multiple of the SM count, and many tiles per CTA; B = 1; T = 343 and T < 128;
GLU, BatchNorm statistics, in-place accumulate, GELU with its pre-activation copy, channel-major output; the sensor-mix
data gradient; per-sample weight sets that change between consecutive tiles of one CTA, including an out-of-range set
(status 900, the other samples still computed); NaN-filled output buffers."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {3: 1e-5, 1: 3e-3}          # 3xTF32 ~ fp32; TF32: each operand rounded to 11 significant bits


def _abi():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _suffix(passes):
    return "" if passes == 3 else "_tf32"


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


def _close(got, ref, scale, tol, what):
    bad = (got.double() - ref).abs() > tol * scale + 1e-30
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at {bad.nonzero()[0].tolist()}"


def _run_conv(passes, x, wop, bias, B, T, Cin, Ntot, Kw, dil, sign, mode, y0):
    """bm_tc_conv1d_persistent into NaN-filled buffers (accumulate: into a copy of y0); returns the outputs"""
    call, ptr, stream = _abi()
    glu, act, tmaj, acc = int(mode == "glu"), int(mode == "gelu"), int(mode == "tmajor"), int(mode == "accumulate")
    nan = float("nan")
    y = y0.clone() if acc else torch.full((B, Ntot, T) if tmaj else (B, T, Ntot), nan, device=DEV)
    aux = torch.full((B, T, Ntot), nan, device=DEV) if act else None
    glu_out = torch.full((B, T, Ntot // 2), nan, device=DEV) if glu else None
    stats = torch.full((2 * Ntot,), nan, device=DEV, dtype=torch.float64) if mode == "stats" else None
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    call("bm_tc_conv1d_persistent" + _suffix(passes), ptr(x), ptr(wop), ptr(bias), acc, B, T, Cin, Ntot, Kw, dil, sign,
         glu, act, tmaj, ptr(y), ptr(aux), ptr(glu_out), ptr(stats), ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0, f"status {int(status.item())}"
    return dict(y=y, aux=aux, glu_out=glu_out, stats=stats)


# (B, T, Cin, Ntot, Kw, dil, sign, mode); tiles = B * ceil(T / 128) * column tiles (160 wide; GLU: 80 'a' columns + gates)
def _cases():
    sms = _sms()
    return [
        (2, 360, 320, 320, 3, 2, 1, "stats"),                  # 12 tiles: fewer than the SMs
        (sms // 2, 100, 320, 320, 3, 1, -1, "plain"),         # exactly one tile per SM (T < 128)
        (23, 343, 320, 320, 3, 4, 1, "accumulate"),           # 138 tiles: not a multiple of the SM count, T = 343
        (1, 343, 320, 640, 3, 1, 1, "glu"),                   # B = 1
        (40, 360, 320, 640, 1, 1, 1, "gelu"),                 # 480 tiles: several per CTA
        (37, 50, 640, 1024, 1, 1, 1, "tmajor"),               # 128-wide tiles, T < 128
        (64, 360, 320, 320, 3, 2, 1, "stats"),                # 384 tiles, statistics summed over several tiles per CTA
    ]


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("idx", range(7))
def test_tile_walk(passes, idx):
    B, T, Cin, Ntot, Kw, dil, sign, mode = _cases()[idx]
    torch.manual_seed(100 + idx)
    x = torch.randn(B, T, Cin, device=DEV)
    wop = torch.randn(Kw, Ntot, Cin, device=DEV) * 0.05
    bias = None if mode == "accumulate" else torch.randn(Ntot, device=DEV)
    y0 = torch.randn(B, T, Ntot, device=DEV) if mode == "accumulate" else None
    out = _run_conv(passes, x, wop, bias, B, T, Cin, Ntot, Kw, dil, sign, mode, y0)
    again = _run_conv(passes, x, wop, bias, B, T, Cin, Ntot, Kw, dil, sign, mode, y0)
    for k in ("y", "aux", "glu_out"):
        if out[k] is not None:
            assert torch.equal(out[k], again[k]), f"{k}: a second launch differs"
    tol = TOL[passes]
    ref, scale = _ref(x, wop, dil, sign)
    if bias is not None:
        ref, scale = ref + bias.double(), scale + bias.double().abs()
    if y0 is not None:
        ref, scale = ref + y0.double(), scale + y0.double().abs()
    if mode == "glu":
        H = Ntot // 2
        _close(out["y"], ref, scale, tol, "h")
        a, g = ref[..., :H], ref[..., H:]
        _close(out["glu_out"], a * torch.sigmoid(g), scale[..., :H] + a.abs() * scale[..., H:], tol, "GLU output")
    elif mode == "gelu":
        _close(out["aux"], ref, scale, tol, "pre-activation")
        _close(out["y"], torch.nn.functional.gelu(ref), 1.2 * scale, tol, "GELU output")
    elif mode == "tmajor":
        _close(out["y"].permute(0, 2, 1), ref, scale, tol, "channel-major y")
    else:
        _close(out["y"], ref, scale, tol, "y")
    if mode == "stats":
        yd = out["y"].double().reshape(-1, Ntot)
        s = torch.cat([yd.sum(0), (yd * yd).sum(0)])
        bad = (out["stats"] - s).abs() > 2e-6 * torch.cat([yd.abs().sum(0), (yd * yd).sum(0)])
        assert not bad.any(), f"BatchNorm statistics: columns {bad.nonzero().flatten().tolist()[:8]} off"
        assert torch.allclose(out["stats"], again["stats"], rtol=1e-12, atol=0)


def _set_weights(S, Ntot, Cin):
    call, ptr, stream = _abi()
    w = torch.randn(S, Ntot, Cin, device=DEV) * 0.05
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    call("bm_tc_weight_split", ptr(w), S * Ntot, Cin, 1, ptr(hi), ptr(lo), None, None, stream())
    return w, hi, lo


@pytest.mark.parametrize("passes", [3, 1])
def test_weight_sets_change_between_tiles_of_a_cta(passes):
    """bm_tc_pointwise_sel with 3 times as many tiles as SMs: each CTA's consecutive tiles belong to samples with different
    weight sets.  An out-of-range set reports 900 and the other samples are still computed."""
    call, ptr, stream = _abi()
    torch.manual_seed(7)
    S, Cin, Ntot, T = 3, 256, 320, 50
    B = 3 * _sms() // 2                                       # 2 column tiles per sample: 3 tiles per CTA
    w, hi, lo = _set_weights(S, Ntot, Cin)
    x = torch.randn(B, T, Cin, device=DEV)
    # CTA i's tiles are i, i + SMs, i + 2 SMs: samples s, s + SMs/2, s + SMs: one set after another
    wsel = ((torch.arange(B, device=DEV) // (_sms() // 2)) % S).to(torch.int32)
    ref = torch.einsum("btk,bnk->btn", x.double(), w.double()[wsel.long()])
    scale = torch.einsum("btk,bnk->btn", x.double().abs(), w.double().abs()[wsel.long()])
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    outs = []
    for _ in range(2):
        y = torch.full((B, T, Ntot), float("nan"), device=DEV)
        call("bm_tc_pointwise_sel" + _suffix(passes), ptr(x), ptr(hi), ptr(lo), ptr(wsel), S, B, T, Cin, Ntot, ptr(y),
             ptr(status), stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        outs.append(y)
    assert torch.equal(outs[0], outs[1])
    _close(outs[0], ref, scale, TOL[passes], "y")
    bad = B // 2 + 1
    wsel[bad] = S
    y = torch.full((B, T, Ntot), float("nan"), device=DEV)
    call("bm_tc_pointwise_sel" + _suffix(passes), ptr(x), ptr(hi), ptr(lo), ptr(wsel), S, B, T, Cin, Ntot, ptr(y),
         ptr(status), stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 900
    keep = torch.arange(B, device=DEV) != bad
    _close(y[keep], ref[keep], scale[keep], TOL[passes], "y beside the out-of-range sample")
    assert torch.isfinite(y[bad]).all()


@pytest.mark.parametrize("passes", [3, 1])
def test_sensor_mix_bwd_many_tiles(passes):
    """bm_tc_sensor_mix_bwd_data over several tiles per CTA: dmeg[b,c,t] = mask[c] sum_o du[b,t,o] W[rec_b][c][o]."""
    call, ptr, stream = _abi()
    torch.manual_seed(12)
    Op, Cp, C, R, T = 320, 288, 273, 4, 200
    B = _sms() // 2 + 5
    w, hi, lo = _set_weights(R, Cp, Op)
    du = torch.randn(B, T, Op, device=DEV)
    wsel = torch.arange(B, device=DEV, dtype=torch.int32) % R
    mask = (torch.rand(C, device=DEV) > 0.2).float()
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    outs = []
    for _ in range(2):
        dmeg = torch.full((B, C, T), float("nan"), device=DEV)
        call("bm_tc_sensor_mix_bwd_data" + _suffix(passes), ptr(du), ptr(hi), ptr(lo), ptr(wsel), R, ptr(mask), B, T, Op,
             Cp, C, ptr(dmeg), ptr(status), stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        outs.append(dmeg)
    assert torch.equal(outs[0], outs[1])
    wd = w.double()[wsel.long()][:, :C]
    ref = torch.einsum("bto,bco->bct", du.double(), wd) * mask.double()[None, :, None]
    scale = torch.einsum("bto,bco->bct", du.double().abs(), wd.abs())
    _close(outs[0], ref, scale, TOL[passes], "dmeg")
