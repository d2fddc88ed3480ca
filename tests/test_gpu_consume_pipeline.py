"""GPU: the consumer K loop of the warp-specialised tensor-core kernels (csrc/tc_common.cuh hc_consume_block in
hc_conv_kernel and hw_wgrad_kernel: the per-block A split, MMAs, stage release and `acc += part`, and the stage ring it
walks) at its edges, in both pass counts:

  * tiles of 1, 2, 3, 4 and 7 K blocks (Cin 32 .. 224 at kernel size 1) and of 3, 6 and 9 (Cin 32, 64, 96 at kernel
    size 3), so that the 3-stage ring wraps at odd and even points of a tile;
  * persistent CTAs with more tiles than SMs, whose consecutive tiles start at different ring positions;
  * 160- and 128-wide column tiles, and per-sample weight sets whose last column tile has dead columns;
  * the GLU epilogue (its 'a' columns and their gates sit in different column halves of a tile), in-place accumulate,
    channel-major output and BatchNorm statistics;
  * conv weight gradients with K slices of a single block and sample edges inside a block.

Every output is checked against fp64 (relative Frobenius error, and element by element against the fp64 sum of |products|
as test_gpu_conv_persistent.py does), and a second launch under torch.use_deterministic_algorithms(True) must reproduce
the first bit for bit (the fused BatchNorm statistics, fp64 atomics across tiles, to 1e-12)."""
import pytest
import torch

from conftest import rel_err
from test_gpu_conv_persistent import TOL, _close, _ref, _run_conv, _set_weights, _sms, _suffix
from test_gpu_wgrad_pipeline import TOL1, TOL3, _ref as _wgrad_ref, _rna

pytestmark = pytest.mark.gpu
DEV = "cuda"
FRO = {3: 1e-4, 1: 3e-3}        # relative Frobenius error against fp64 (TF32: each operand rounded to 11 bits)


def _deterministic(run):
    """run() twice under torch.use_deterministic_algorithms(True)"""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        return run(), run()
    finally:
        torch.use_deterministic_algorithms(prev)


def _check_conv(case, passes, seed):
    B, T, Cin, Ntot, Kw, dil, sign, mode = case
    torch.manual_seed(seed)
    x = torch.randn(B, T, Cin, device=DEV)
    wop = torch.randn(Kw, Ntot, Cin, device=DEV) * 0.05
    bias = None if mode == "accumulate" else torch.randn(Ntot, device=DEV)
    y0 = torch.randn(B, T, Ntot, device=DEV) if mode == "accumulate" else None
    out, again = _deterministic(lambda: _run_conv(passes, x, wop, bias, B, T, Cin, Ntot, Kw, dil, sign, mode, y0))
    for k in ("y", "aux", "glu_out"):
        if out[k] is not None:
            assert torch.equal(out[k], again[k]), f"{k}: a second launch differs"
    if out["stats"] is not None:                # fp64 atomics across tiles: summed in a run-dependent order
        assert torch.allclose(out["stats"], again["stats"], rtol=1e-12, atol=0)
    ref, scale = _ref(x, wop, dil, sign)
    if bias is not None:
        ref, scale = ref + bias.double(), scale + bias.double().abs()
    if y0 is not None:
        ref, scale = ref + y0.double(), scale + y0.double().abs()
    got = out["y"].permute(0, 2, 1) if mode == "tmajor" else out["y"]
    assert rel_err(got.double(), ref) < FRO[passes]
    _close(got, ref, scale, TOL[passes], "y")
    if mode == "glu":
        H = Ntot // 2
        a, g = ref[..., :H], ref[..., H:]
        _close(out["glu_out"], a * torch.sigmoid(g), scale[..., :H] + a.abs() * scale[..., H:], TOL[passes], "GLU output")
    if mode == "stats":
        yd = out["y"].double().reshape(-1, Ntot)
        s = torch.cat([yd.sum(0), (yd * yd).sum(0)])
        bad = (out["stats"] - s).abs() > 2e-6 * torch.cat([yd.abs().sum(0), (yd * yd).sum(0)])
        assert not bad.any(), f"BatchNorm statistics: columns {bad.nonzero().flatten().tolist()[:8]} off"


# (B, T, Cin, Ntot, Kw, dil, sign, mode): K blocks per tile = Kw * Cin / 32
KBLOCK_CASES = [(3, 300, cin, 320, 1, 1, 1, "plain") for cin in (32, 64, 96, 128, 224)] + \
               [(3, 300, cin, 320, 3, 2, -1, "plain") for cin in (32, 64, 96)]


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("case", KBLOCK_CASES, ids=lambda c: f"cin{c[2]}_k{c[4]}")
def test_kblock_counts(case, passes):
    _check_conv(case, passes, seed=case[2] + case[4])


def _tile_cases():
    sms = _sms()
    return {
        "7_blocks_many_tiles": (sms // 2 + 7, 360, 224, 320, 1, 1, 1, "plain"),   # > 3 tiles per SM, 7-block tiles
        "9_blocks_stats": (sms // 3 + 1, 360, 96, 320, 3, 1, 1, "stats"),
        "bn128": (5, 200, 64, 256, 3, 1, 1, "plain"),                            # 2 tiles of 128 columns
        "glu": (7, 250, 96, 640, 3, 1, 1, "glu"),
        "accumulate": (9, 150, 64, 320, 3, 3, -1, "accumulate"),
        "channel_major": (11, 90, 224, 1024, 1, 1, 1, "tmajor"),
    }


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("name", ["7_blocks_many_tiles", "9_blocks_stats", "bn128", "glu", "accumulate",
                                  "channel_major"])
def test_tiles_and_epilogues(name, passes):
    _check_conv(_tile_cases()[name], passes, seed=len(name))


@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("Ntot", [288, 192])
def test_weight_sets_dead_columns(Ntot, passes):
    """bm_tc_pointwise_sel, 3-block tiles, per-sample weight sets, more tiles than SMs; 288 columns: 2 tiles of 160, the
    last with 32 dead columns; 192: 2 tiles of 128, the last with 64"""
    from brainmagick_b200 import _lib
    call, ptr, stream = _lib.call, _lib.ptr, _lib.stream
    torch.manual_seed(31)
    S, Cin, T = 4, 96, 200
    B = _sms() + 3
    w, hi, lo = _set_weights(S, Ntot, Cin)
    x = torch.randn(B, T, Cin, device=DEV)
    wsel = (torch.arange(B, device=DEV) % S).to(torch.int32)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)

    def run():
        y = torch.full((B, T, Ntot), float("nan"), device=DEV)
        call("bm_tc_pointwise_sel" + _suffix(passes), ptr(x), ptr(hi), ptr(lo), ptr(wsel), S, B, T, Cin, Ntot, ptr(y),
             ptr(status), stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        return y

    y, again = _deterministic(run)
    assert torch.equal(y, again)
    ref = torch.einsum("btk,bnk->btn", x.double(), w.double()[wsel.long()])
    scale = torch.einsum("btk,bnk->btn", x.double().abs(), w.double().abs()[wsel.long()])
    assert rel_err(y.double(), ref) < FRO[passes]
    _close(y, ref, scale, TOL[passes], "y")


WGRAD_CASES = [  # B, T, Mdy, Nx, Ntrue, Kw, dilation
    (3, 100, 64, 96, 96, 3, 1),          # every K slice a single block
    (4, 320, 320, 32, 32, 1, 1),         # single-block slices, 160-wide column tiles
    (5, 33, 192, 160, 160, 3, 2),        # a sample edge inside almost every block
    (6, 70, 320, 64, 64, 3, 1),          # sample edges inside blocks, 160-wide
]


@pytest.mark.parametrize("form", ["", "_tf32"])
@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_wgrad(case, form):
    from brainmagick_b200 import _lib
    call, ptr, stream = _lib.call, _lib.ptr, _lib.stream
    lib = _lib.load()
    B, T, M, N, Ntrue, Kw, dil = case
    assert lib.bm_tc_wgrad_conv_supported(T, M, N, Kw)
    torch.manual_seed(B + T + M)
    dy = torch.randn(B, T, M, device=DEV)
    x = torch.randn(B, T, N, device=DEV)
    ws = torch.full((int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)),), float("nan"), device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)

    def run():
        dw = torch.full((M, Ntrue, Kw), float("nan"), device=DEV)
        call("bm_tc_wgrad_conv" + form, ptr(dy), ptr(x), B, T, M, N, Ntrue, Kw, dil, ptr(ws), ptr(dw), ptr(status),
             stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0, f"pipeline status {int(status.item())}"
        return dw

    dw, again = _deterministic(run)
    assert torch.equal(dw, again)
    if form == "_tf32":
        assert rel_err(dw.double().cpu(), _wgrad_ref(_rna(dy), _rna(x), Kw, dil, Ntrue).cpu()) < TOL1
    else:
        ref = _wgrad_ref(dy, x, Kw, dil, Ntrue)
        assert rel_err(dw.double().cpu(), ref.cpu()) < TOL3
        # element by element, against the fp64 sum of |products|
        scale = _wgrad_ref(dy.abs(), x.abs(), Kw, dil, Ntrue)
        _close(dw, ref, scale, TOL[3], "dW")
