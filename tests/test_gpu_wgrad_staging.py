"""GPU: the conv weight gradient's dY staging (hw_wgrad_kernel in csrc/tc_common.cuh: dY boxes by TMA into a ring of 2
slots, transposed in shared memory) at the edges of that ring: K slices whose block count is a multiple of neither the
ring's 2 slots nor the 3 pipeline stages, slices of a single K block, flattened rows that end inside the last dY box (zero
filled by TMA), column tiles whose last dY boxes lie past Mdy, and dy widths 64, 192 and 1024 (128-wide column tiles) and
320, 640 and 960 (160-wide).  The slice counts in the comments are those of a 132-SM H100.  Checked as
test_gpu_wgrad_pipeline.py checks: against fp64, with NaN-filled workspace and output, a second run bitwise equal,
status 0."""
import pytest
import torch

from conftest import rel_err
from test_gpu_wgrad_pipeline import TOL1, TOL3, _ref, _rna

pytestmark = pytest.mark.gpu

CASES = [  # B, T, Mdy, Nx, Ntrue, Kw, dilation
    (9, 233, 192, 96, 96, 3, 2),         # 5 blocks per slice, the last slice 1; boxes m >= 192 of column tile 1: all zeros
    (17, 161, 1024, 64, 64, 3, 1),       # 11 blocks per slice, the last 9; 8 column tiles
    (3, 100, 64, 96, 96, 3, 1),          # every slice a single block; 64 columns: boxes 2-3 of the tile are all zeros
    (4, 320, 64, 32, 32, 1, 1),          # single-block slices, rows an exact multiple of 32
    (9, 233, 320, 96, 80, 3, 4),         # 160-wide: 5 blocks per slice, the last slice 1; Ntrue < Nx
    (13, 161, 640, 64, 64, 3, 2),        # 160-wide, 5 blocks per slice
    (9, 161, 960, 64, 64, 3, 1),         # 160-wide, 6 column tiles
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("form", ["", "_tf32", "_f16"])
def test_wgrad_dy_staging(case, form):
    from brainmagick_b200 import _lib
    call, ptr, stream = _lib.call, _lib.ptr, _lib.stream
    lib = _lib.load()
    B, T, M, N, Ntrue, Kw, dil = case
    assert lib.bm_tc_wgrad_conv_supported(T, M, N, Kw)
    torch.manual_seed(B * T + M + N + Kw)
    dev = "cuda"
    dy = torch.randn(B, T, M, device=dev)
    x = torch.randn(B, T, N, device=dev)
    ws = torch.full((int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)),), float("nan"), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    amax = torch.empty(2, device=dev)
    call("bm_amax", ptr(dy), dy.numel(), ptr(amax[0:1]), stream())
    call("bm_amax", ptr(x), x.numel(), ptr(amax[1:2]), stream())

    def run():
        dw = torch.full((M, Ntrue, Kw), float("nan"), device=dev)
        if form == "_f16":
            call("bm_tc_wgrad_conv_f16", ptr(dy), ptr(amax[0:1]), ptr(x), ptr(amax[1:2]), B, T, M, N, Ntrue, Kw, dil,
                 ptr(ws), ptr(dw), ptr(status), stream())
        else:
            call("bm_tc_wgrad_conv" + form, ptr(dy), ptr(x), B, T, M, N, Ntrue, Kw, dil, ptr(ws), ptr(dw), ptr(status),
                 stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0, f"pipeline status {int(status.item())}"
        return dw

    dw = run()
    if form == "_tf32":
        e = rel_err(dw.double().cpu(), _ref(_rna(dy), _rna(x), Kw, dil, Ntrue).cpu())
        assert e < TOL1, e
    else:
        e = rel_err(dw.double().cpu(), _ref(dy, x, Kw, dil, Ntrue).cpu())
        assert e < TOL3, e
    assert torch.equal(dw, run())
