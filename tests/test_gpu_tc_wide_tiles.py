"""GPU: the weight gradients on 160-column engine tiles with a partial last tile.  576 output columns run as three full
160-wide tiles and one with 96 live columns, so the zero-filled operand columns and the bounded store of that tile are
exercised; checked against torch's fp64 contraction (test-only reference) at the tolerance of tests/test_gpu_tc.py."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 3e-5


def _ref(dy, x, Kw, dil):
    """dw[m,n,j] = sum_{b,t} dy[b,t,m] x[b,t+(j-Kw//2)*dil,n] in fp64."""
    B, T, M = dy.shape
    N = x.shape[2]
    ref = torch.zeros(M, N, Kw, dtype=torch.float64, device=dy.device)
    xd, dyd = x.double(), dy.double()
    for j in range(Kw):
        s = (j - Kw // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        ref[:, :, j] = torch.einsum("btm,btn->mn", dyd[:, lo:hi], xd[:, lo + s:hi + s])
    return ref


@pytest.mark.parametrize("B,T,M,N,Kw,dil", [(3, 100, 320, 576, 3, 2), (2, 77, 96, 576, 1, 1)])
def test_tc_wgrad_partial_wide_tile(B, T, M, N, Kw, dil):
    """bm_tc_wgrad (per-tap form): N = 576 columns of x."""
    from brainmagick_b200 import _lib
    lib = _lib.load()
    assert lib.bm_tc_wgrad_supported(M, N)
    torch.manual_seed(5)
    dev = "cuda"
    dy = torch.randn(B, T, M, device=dev)
    x = torch.randn(B, T, N, device=dev)
    ws = torch.full((int(lib.bm_tc_wgrad_workspace(B, M, N, Kw)),), float("nan"), device=dev)
    dw = torch.full((M, N, Kw), float("nan"), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    _lib.call("bm_tc_wgrad", _lib.ptr(dy), _lib.ptr(x), B, T, M, N, N, Kw, dil, _lib.ptr(ws), _lib.ptr(dw), None,
              _lib.ptr(status), _lib.stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    e = rel_err(dw.cpu(), _ref(dy, x, Kw, dil).cpu())
    print(f"[tc wgrad B={B} T={T} M={M} N={N} Kw={Kw}] rel_err vs fp64 = {e:.2e}")
    assert e < TOL


@pytest.mark.parametrize("B,T,M,N,Kw,dil", [(3, 100, 576, 320, 3, 2), (4, 64, 576, 96, 3, 1)])
def test_tc_wgrad_conv_partial_wide_tile(B, T, M, N, Kw, dil):
    """bm_tc_wgrad_conv (one GEMM over the flattened rows): Mdy = 576 dy channels are the engine's columns."""
    from brainmagick_b200 import _lib
    lib = _lib.load()
    assert lib.bm_tc_wgrad_conv_supported(T, M, N, Kw)
    torch.manual_seed(6)
    dev = "cuda"
    dy = torch.randn(B, T, M, device=dev)
    x = torch.randn(B, T, N, device=dev)
    ws = torch.full((int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, Kw)),), float("nan"), device=dev)
    dw = torch.full((M, N, Kw), float("nan"), device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    _lib.call("bm_tc_wgrad_conv", _lib.ptr(dy), _lib.ptr(x), B, T, M, N, N, Kw, dil, _lib.ptr(ws), _lib.ptr(dw),
              _lib.ptr(status), _lib.stream())
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    e = rel_err(dw.cpu(), _ref(dy, x, Kw, dil).cpu())
    print(f"[tc wgrad_conv B={B} T={T} M={M} N={N} Kw={Kw}] rel_err vs fp64 = {e:.2e}")
    assert e < TOL
