"""GPU: the conv weight gradient (bm_tc_wgrad_conv, its `_tf32` form and bm_tc_wgrad_conv_f16; hw_wgrad_kernel in
csrc/tc_common.cuh) at the edges of its pipeline: flattened rows that end inside a K block and a K slice, sample edges
inside a block, taps that change inside a 128-row tile and inside a warpgroup's 64 rows, a tap made of padding alone,
x channels past Ntrue, every dy width the column tiles take.  3 passes against fp64 (the tolerance of test_gpu_tc.py),
1 pass against fp64 on tf32-rounded operands (the tolerance of test_gpu_tf32.py); NaN-filled workspace and output, a
second run bitwise equal, status 0."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL3, TOL1 = 3e-5, 1e-5

CASES = [  # B, T, Mdy, Nx, Ntrue, Kw, dilation
    (3, 32, 64, 96, 96, 3, 1),           # T = one K block; taps change at rows 96, 192 (inside warpgroup 1 of tile 0)
    (5, 33, 192, 160, 160, 3, 2),        # a sample edge in almost every block; tap change at 160 (warpgroup 0 of tile 1)
    (2, 361, 576, 224, 224, 3, 4),       # taps change at 224 (warpgroup 1 of tile 1), 448 (tile 3)
    (3, 40, 192, 96, 96, 3, 50),         # shift 50 >= T: taps 0 and 2 are all padding
    (3, 77, 320, 320, 270, 3, 1),        # Ntrue < Nx, 160-wide column tiles
    (2, 45, 1024, 96, 96, 1, 1),         # one tap, 8 column tiles
    (7, 361, 64, 224, 200, 1, 1),
    (9, 33, 576, 160, 150, 3, 16),
]


def _rna(t):
    """fp32 -> nearest tf32 (ties away from zero), as fp32."""
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def _ref(dy, x, Kw, dil, Ntrue):
    """dW [M][Ntrue][Kw] in fp64: dW[m][n][j] = sum_{b,t} dy[b,t,m] x[b,t+s_j,n], zero outside the sample."""
    B, T, M = dy.shape
    ref = torch.zeros(M, Ntrue, Kw, dtype=torch.float64, device=dy.device)
    xd, dyd = x.double()[:, :, :Ntrue], dy.double()
    for j in range(Kw):
        s = (j - Kw // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        if lo < hi:
            ref[:, :, j] = torch.einsum("btm,btn->mn", dyd[:, lo:hi], xd[:, lo + s:hi + s])
    return ref


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("form", ["", "_tf32", "_f16"])
def test_wgrad_pipeline_edges(case, form):
    from brainmagick_b200 import _lib
    call, ptr, stream = _lib.call, _lib.ptr, _lib.stream
    lib = _lib.load()
    B, T, M, N, Ntrue, Kw, dil = case
    assert (B * T) % 32 != 0 or T == 32                 # the last K block is partial (T = 32: exact blocks)
    assert lib.bm_tc_wgrad_conv_supported(T, M, N, Kw)
    torch.manual_seed(B * T + M + N)
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
    if Kw == 3 and dil >= T:                            # a tap of padding alone is exactly zero
        assert torch.count_nonzero(dw[:, :, 0]) == 0 and torch.count_nonzero(dw[:, :, 2]) == 0
    assert torch.equal(dw, run())                       # fixed-order reduction: the same bits again
