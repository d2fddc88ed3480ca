"""GPU: the tensor-core contractions that run on every training step and had no per-element check -- the weight gradients
bm_tc_wgrad (hg_gemm_kernel<WgradOp> + wgrad_reduce_kernel, csrc/tc_wgrad.cuh), bm_tc_wgrad_conv (hw_wgrad_kernel +
wgradp_reduce_kernel, csrc/tc_wgradp.cuh) and bm_tc_wgrad_grouped, the CLIP scores and loss (hg_gemm_kernel<ClipOp> +
clip_finalize_kernel, csrc/tc_clip.cuh) and the three GEMMs the CLIP backward picks between (clip_dest_gemm /
clip_dcand_gemm in csrc/clip_api.cu) -- against a plain fp64 reference, element by element, at their tile, K-slice,
batch-slice, sample and dispatch edges, in the default (3xTF32) and the `_tf32` forms.

The reference is fp64 from the fp32 operands the kernel read, and chained stages are checked stage by stage from the fp32
values the kernel wrote: the scores from its own inv_norm, the probabilities and row loss from its own scores, dE and dC
from a G recomputed in fp64 from the probs, inv_norm and gout (or dscores) the test passed in.  With u = 2^-24 and mag the
same contraction over absolute values, every contraction element is held to

    |got - ref| <= (E_SPLIT + E_MMA + nblk + ks + 2) u mag  +  epilogue terms  +  TINY

  - E_SPLIT = 20: tf32_split (tc_common.cuh) sets hi = x rounded to 10 mantissa bits (ties away), so |lo| <= 2^-11 |x|; the
    tensor core reads lo truncated to tf32 (less than 2^-21 |x| lost) and the lo*lo product is dropped: at most
    (2 * 2^-21 + 2^-22) |xy| = 20 u |xy| per product, every product of tf32 pieces being exact in fp32.
  - E_MMA = 48: the 12 chained wgmma.k8 of one 32-wide K block (`part`, fresh in every block), each taken to err by at most
    2 ulp of its 8 products plus the incoming partial (12 * 4 u).  NVIDIA does not document how wgmma rounds inside its
    accumulator, so this is the one constant not derived from a documented rule.  Measured on an H100 80GB HBM3 (SXM,
    700 W power limit), the largest |got - ref| / bound over this file's tensor-core checks is 0.22 for the 3xTF32 forms
    and 0.17 for the `_tf32` forms, both in dC of the CLIP backward (pytest -s prints the figures and where they occur).
  - nblk: the K blocks added with round-to-nearest into one accumulator (the blocks of one K or batch slice); ks: the slice
    partials wgrad_reduce_kernel, wgradp_reduce_kernel or clip_finalize_kernel adds.  Both follow the library's geometry
    rules (wgrad_geometry, wgradp_geometry, clip_geometry) at the device's SM count.
  - epilogue terms, each from the kernel's own arithmetic: inv_norm = 1 / (1e-8f + (float)sqrt(fp64 sum of squares)),
    3 u |inv| (the reference adds the fp32 constant 1e-8f, as the kernel does); the score scale, u |ref|; expf 2 ulp and
    logf 1 ulp in the softmax and row loss (test_gpu_fma_entry_points.py's checks); clip_ce_bwd_kernel's G, 4 u |G|
    (clip_scores_grad_kernel's, u |G|), carried into dE and dC as that many u times mag; clip_cand_coef_kernel's fmaf
    chain over Bn and its division; the final fmaf(-coef, cand, dcand), u |ref|; dbias, fp32 column sums of 256 rows
    added with atomics.
The `_tf32` forms are held to the same bound with E_SPLIT = 0 against a reference of the rna-rounded operands (the bound
test_gpu_bf16.py uses for `_bf16`); there G is the kernel's own fp32 G, reproduced bit for bit and checked against its
scratch, because rounding an fp64 G to tf32 can land one tf32 step away.  The FP32-FMA fallbacks of the CLIP backward are
held to test_gpu_fma_entry_points.py's 2 (K + 2) u mag.

A worst-case bound grows with nblk, so on random data it might not notice a form that silently lost one of its three
passes.  test_lost_pass_is_seen feeds each engine operands x = m (1 + 2^-12), m a positive tf32 value: tf32_split gives
hi = m and lo = m 2^-12 exactly, so 3xTF32 errs by u |xy| per product and a form without hi*lo or lo*hi by 2^-12 |xy|.
There the bound stays below 2^-13 relative, the default form passes it, and the `_tf32` output of the same call (a
one-pass stand-in for a lost pass) fails it at every element.

Every output starts as NaN inside a buffer with sentinel guard zones (an element left unwritten fails, and so does a write
outside the output); every workspace and scratch starts as NaN; the weight gradients, the `_det` CLIP forms and the
backward GEMMs must give the same bits on a second call onto a workspace of other contents; the status word must read 0.
Each CLIP backward case asserts, from the kernel names torch.profiler records, which GEMM ran for dE and for dC
(hg_gemm_kernel<GemmNTOp>, hg_gemm_kernel<WgradOp> in its direct mode, or gemm_simt_kernel), so a shape list that stops
reaching a path fails instead of testing another one.

Out of scope: the pooled CLIP forms (per element in test_gpu_negative_pool.py), the conv forward entry points (per element
in test_gpu_conv_pipeline.py, test_gpu_conv_persistent.py and test_gpu_conv_epilogue.py), and the fp16-piece entry points
bm_tc_conv1d_f16 and bm_tc_wgrad_conv_f16, which are not on the host path and whose error is relative to amax, not |x|.
"""
import os

import numpy as np
import pytest
import torch

from test_gpu_elementwise_entry_points import _kernels
from test_gpu_fma_entry_points import C_BOUND, Out, _by_group, _check, _check_softmax, _gen, _groups, _rand, _sms
from test_gpu_wgrad_pipeline import _rna

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                # unit roundoff of fp32
UD = 2.0 ** -53               # unit roundoff of fp64
E_SPLIT = 20                  # the tf32 split's error per product, in u |xy|
E_MMA = 48                    # the chained wgmma.k8 of one K block, in u mag (the one constant not derived from a rule)
TINY = 2.0 ** -140            # underflow: a few fp32 subnormal steps
EPS = float(np.float32(1e-8))                           # the kernels' 1e-8f
INV_ZERO = float(np.float32(1.0) / np.float32(1e-8))    # 1 / (1e-8f + 0): the inv_norm of an all-zero candidate
FORMS = ["", "_tf32"]
# the largest |got - ref| / bound of the tensor-core checks per form, and where: printed at the end of the module (pytest -s)
WORST = {"": (0.0, None), "_tf32": (0.0, None)}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for form, name in (("", "3xTF32"), ("_tf32", "_tf32")):
        print(f"\nlargest |got - ref| / bound, {name} forms: {WORST[form][0]:.3g} ({WORST[form][1]})")


def _abi():
    from brainmagick_b200 import _lib
    return _lib.call, _lib.ptr, _lib.stream, _lib.load()


def _ops(form, *ts):
    """the operand values the form multiplies, in fp64: as read (3xTF32), or rounded to tf32 (`_tf32`)"""
    return [(t if form == "" else _rna(t)).double() for t in ts]


def _tc_tol(form, mag, nblk, ks, extra=0.0):
    """the bound of the module docstring; nblk may be a tensor broadcastable to mag"""
    e = (E_SPLIT if form == "" else 0) + E_MMA + 2 + ks + torch.as_tensor(nblk, dtype=torch.float64, device=DEV)
    return e * U * mag + extra + TINY


def _check_tc(what, form, got, ref, tol):
    """_check of a tensor-core bound, recording the largest |got - ref| / tol of the form"""
    d = (got.double() - ref).abs() / tol
    if not torch.isnan(d).any() and d.max().item() > WORST[form][0]:
        WORST[form] = (d.max().item(), f"{os.environ.get('PYTEST_CURRENT_TEST', '').split(' ')[0]} {what}")
    _check(what, got, ref, tol)


def _status():
    return torch.zeros(1, dtype=torch.int32, device=DEV)


def _pick_bn(n):
    """tc_common.cuh hg_pick_bn"""
    return 160 if -(-n // 160) * 160 <= -(-n // 128) * 128 else 128


def _wgrad_geometry(B, M, N, taps):
    """(samples per batch slice, slices) of bm_tc_wgrad (tc_wgrad.cuh wgrad_geometry)"""
    tiles = -(-M // 128) * -(-N // _pick_bn(N)) * taps
    want = min(max(1, _sms() // tiles), B)
    bchunk = -(-B // want)
    return bchunk, -(-B // bchunk)


def _wgradp_geometry(B, T, Mdy, Nx, taps):
    """(K blocks per slice, slices) of bm_tc_wgrad_conv (tc_wgradp.cuh wgradp_geometry)"""
    chunks = -(-(B * T) // 32)
    tiles = 2 * -(-(taps * Nx) // 256) * -(-Mdy // _pick_bn(Mdy))
    ks = min(max(1, _sms() // tiles), chunks)
    per = -(-chunks // ks)
    return per, -(-chunks // per)


def _clip_geometry(Bn, Bc, KT):
    """(K blocks per slice, slices) of the CLIP scores GEMM (tc_clip.cuh clip_geometry)"""
    chunks = -(-KT // 32)
    ks = min(max(1, _sms() // (-(-Bc // 128) * -(-Bn // 128))), chunks)
    per = -(-chunks // ks)
    return per, -(-chunks // per)


def _wgrad_ref(dy, x, Kw, dil, Ntrue):
    """dW[m][n][tap] = sum_{b,t} dy[b,t,m] x[b, t + (tap - Kw//2) dil, n] (zero outside the sample) for n < Ntrue, and the
    same over |dy| |x|; dy, x fp64"""
    B, T, M = dy.shape
    ref = torch.zeros(M, Ntrue, Kw, dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(ref)
    for tap in range(Kw):
        s = (tap - Kw // 2) * dil
        lo, hi = max(0, -s), min(T, T - s)
        if lo < hi:
            g, xs = dy[:, lo:hi].reshape(-1, M), x[:, lo + s:hi + s, :Ntrue].reshape(-1, Ntrue)
            ref[:, :, tap] = g.T @ xs
            mag[:, :, tap] = g.abs().T @ xs.abs()
    return ref, mag


def _structured(gen, *shape):
    """x = m (1 + 2^-12) with m a positive tf32 value (module docstring): exact in fp32, hi = m, lo = m 2^-12"""
    return _rna(torch.rand(*shape, generator=gen, device=DEV) + 0.5) * (1.0 + 2.0 ** -12)


# =====================================================================================================================
# bm_tc_wgrad: hg_gemm_kernel<WgradOp>, batch slices + wgrad_reduce_kernel, dbias
# =====================================================================================================================
# (B, T, M, N, Ntrue, Kw, dilation, dbias): M >= 32 and M % 4 == 0; N a multiple of 128, 192, 256 or 320.  M = 132 / 260 /
# 640: a partial last 128-row tile; N = 192 (128-wide tiles) and 576 (160-wide): a partial last column tile; "direct": one
# tap, one slice, Ntrue = N (the output written by the GEMM itself); B = 7 / 33: a ragged last batch slice (132 SMs)
WGRAD = {"direct-B1-T343-M32-N128-Kw1": (1, 343, 32, 128, 128, 1, 1, True),
         "direct-B1-T33-M32-N320-Kw1": (1, 33, 32, 320, 320, 1, 1, False),
         "B7-T31-M132-N192-Kw3": (7, 31, 132, 192, 192, 3, 1, True),
         "B33-T33-M260-N320-Ntrue300-Kw3-d2": (33, 33, 260, 320, 300, 3, 2, False),
         "B7-T1-M640-N576-Kw3-d5": (7, 1, 640, 576, 576, 3, 5, True),                  # taps 0 and 2 entirely padding
         "B33-T343-M132-N128-Ntrue100-Kw3-d343": (33, 343, 132, 128, 100, 3, 343, False),   # the same at dilation = T
         "B1-T343-M260-N576-Ntrue500-Kw2-d7": (1, 343, 260, 576, 500, 2, 7, True)}


def _check_dbias(got, dy):
    """fp32 column sums of up to 256 rows, added into a zeroed output with atomics"""
    r = dy.reshape(-1, dy.shape[-1]).double()
    n = r.shape[0]
    _check("dbias", got, r.sum(0), (min(n, 256) + -(-n // 256) + 2) * U * r.abs().sum(0) + TINY)


@pytest.mark.parametrize("form", FORMS, ids=["bm_tc_wgrad", "bm_tc_wgrad_tf32"])
@pytest.mark.parametrize("case", list(WGRAD))
def test_tc_wgrad(case, form):
    call, ptr, stream, lib = _abi()
    B, T, M, N, Ntrue, Kw, dil, with_bias = WGRAD[case]
    assert lib.bm_tc_wgrad_supported(M, N)
    bchunk, ksplit = _wgrad_geometry(B, M, N, Kw)
    assert (Kw == 1 and ksplit == 1 and Ntrue == N) == case.startswith("direct")
    gen = _gen(61)
    dy, x = _rand(gen, B, T, M), _rand(gen, B, T, N)
    nws = int(lib.bm_tc_wgrad_workspace(B, M, N, Kw))
    ws = torch.full((nws,), float("nan"), device=DEV)
    status = _status()

    def run():
        dw, db = Out(M, Ntrue, Kw), Out(M) if with_bias else None
        call("bm_tc_wgrad" + form, ptr(dy), ptr(x), B, T, M, N, Ntrue, Kw, dil, ptr(ws), ptr(dw.t),
             db and ptr(db.t), ptr(status), stream())
        torch.cuda.synchronize()
        assert status.item() == 0, f"status {status.item()}"
        return dw, db

    dw, db = run()
    ref, mag = _wgrad_ref(*_ops(form, dy, x), Kw, dil, Ntrue)
    _check_tc("dw", form, dw.v, ref, _tc_tol(form, mag, bchunk * -(-T // 32), ksplit))
    dw.untouched("dw")
    if with_bias:
        _check_dbias(db.v, dy)
        db.untouched("dbias")
    ws.copy_(torch.randn(nws, generator=gen, device=DEV))
    assert torch.equal(run()[0].v, dw.v), "dw: a second call differs"


# =====================================================================================================================
# bm_tc_wgrad_conv: hw_wgrad_kernel over flattened rows, K slices + wgradp_reduce_kernel
# =====================================================================================================================
# (B, T, Mdy, Nx, Ntrue, Kw, dilation, slices): T >= 32, Nx % 32 == 0, Mdy % 64 == 0; `slices` = 1 or "many" K slices
WGRAD_CONV = {"B3-T37-M64-N96-Kw3": (3, 37, 64, 96, 96, 3, 1, "many"),   # 288 (tap, n) rows; B T = 111 ends in a block
              "B2-T40-M192-N64-Ntrue50-Kw3-d2": (2, 40, 192, 64, 50, 3, 2, "many"),
              "B5-T77-M320-N96-Kw2-d3": (5, 77, 320, 96, 96, 2, 3, "many"),        # 160-wide column tiles
              "B33-T360-M1024-N32-Kw1": (33, 360, 1024, 32, 32, 1, 1, "many"),
              "B2-T64-M1024-N640-Ntrue600-Kw3": (2, 64, 1024, 640, 600, 3, 1, 1),   # 1920 rows: one slice of 4 blocks
              "B1-T32-M64-N32-Kw3": (1, 32, 64, 32, 32, 3, 1, 1),                    # one block
              "B4-T33-M64-N96-Kw3-d40": (4, 33, 64, 96, 96, 3, 40, "many")}          # taps 0 and 2 entirely padding


@pytest.mark.parametrize("form", FORMS, ids=["bm_tc_wgrad_conv", "bm_tc_wgrad_conv_tf32"])
@pytest.mark.parametrize("case", list(WGRAD_CONV))
def test_tc_wgrad_conv(case, form):
    call, ptr, stream, lib = _abi()
    B, T, M, N, Ntrue, Kw, dil, slices = WGRAD_CONV[case]
    assert lib.bm_tc_wgrad_conv_supported(T, M, N, Kw)
    per, ks = _wgradp_geometry(B, T, M, N, Kw)
    assert (ks == 1) == (slices == 1), f"{ks} K slices"
    gen = _gen(62)
    dy, x = _rand(gen, B, T, M), _rand(gen, B, T, N)
    nws = int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, Kw))
    ws = torch.full((nws,), float("nan"), device=DEV)
    status = _status()

    def run():
        dw = Out(M, Ntrue, Kw)
        call("bm_tc_wgrad_conv" + form, ptr(dy), ptr(x), B, T, M, N, Ntrue, Kw, dil, ptr(ws), ptr(dw.t), ptr(status),
             stream())
        torch.cuda.synchronize()
        assert status.item() == 0, f"status {status.item()}"
        return dw

    dw = run()
    ref, mag = _wgrad_ref(*_ops(form, dy, x), Kw, dil, Ntrue)
    _check_tc("dw", form, dw.v, ref, _tc_tol(form, mag, per, ks))
    dw.untouched("dw")
    ws.copy_(torch.randn(nws, generator=gen, device=DEV))
    assert torch.equal(run().v, dw.v), "dw: a second call differs"


# =====================================================================================================================
# bm_tc_wgrad_grouped: hg_gemm_kernel<WgradOp> over CSR groups, one plane per group
# =====================================================================================================================
# (B, T, M, N, G): G >= 3 has an empty group 0 and a one-sample group 1, each group's samples in shuffled order (_groups);
# M = 272: planes padded to 384 rows; N = 320: a partial last 128-wide column tile
GROUPED = {"G1-B5-T40-M320-N256": (5, 40, 320, 256, 1),
           "G4-B9-T33-M272-N320": (9, 33, 272, 320, 4),
           "G3-B7-T64-M272-N256": (7, 64, 272, 256, 3),
           "G5-B12-T1-M32-N320": (12, 1, 32, 320, 5)}


@pytest.mark.parametrize("form", FORMS, ids=["bm_tc_wgrad_grouped", "bm_tc_wgrad_grouped_tf32"])
@pytest.mark.parametrize("case", list(GROUPED))
def test_tc_wgrad_grouped(case, form):
    call, ptr, stream, lib = _abi()
    B, T, M, N, G = GROUPED[case]
    Mpad = -(-M // 128) * 128
    gen = _gen(63)
    a, order, off = _groups(gen, B, G)
    dy, x = _rand(gen, B, T, M), _rand(gen, B, T, N)
    status = _status()

    def run():
        out = Out(G, Mpad, N)
        call("bm_tc_wgrad_grouped" + form, ptr(dy), ptr(x), ptr(order), ptr(off), G, B, T, M, N, ptr(out.t), ptr(status),
             stream())
        torch.cuda.synchronize()
        assert status.item() == 0, f"status {status.item()}"
        return out

    out = run()
    d, xd = _ops(form, dy, x)
    ref = _by_group(torch.einsum("btm,btn->bmn", d, xd), a, G)
    mag = _by_group(torch.einsum("btm,btn->bmn", d.abs(), xd.abs()), a, G)
    nblk = (torch.bincount(a, minlength=G) * -(-T // 32)).view(G, 1, 1)
    _check_tc("planes", form, out.v[:, :M], ref, _tc_tol(form, mag, nblk, 0))
    assert (out.v[:, M:] == 0).all(), "plane padding rows are not exactly 0"
    out.untouched("planes")
    assert torch.equal(run().v, out.v), "planes: a second call differs"


# =====================================================================================================================
# CLIP forward: split-K scores (hg_gemm_kernel<ClipOp>) + clip_finalize_kernel
# =====================================================================================================================
# (Bn, Bc, KT): KT % 4 == 0 and KT >= 32.  Bc = 2048: each finalize thread loops over 8 columns; KT = 36: one partial
# K block; KT = 36 864 at Bn = 1, Bc = 3: 128 K slices of 9 blocks (132 SMs)
CLIP = {"Bn1-Bc1-KT32": (1, 1, 32), "Bn3-Bc127-KT36": (3, 127, 36), "Bn127-Bc128-KT4100": (127, 128, 4100),
        "Bn128-Bc129-KT36": (128, 129, 36), "Bn129-Bc257-KT4100": (129, 257, 4100), "Bn257-Bc3-KT32": (257, 3, 32),
        "Bn3-Bc2048-KT36": (3, 2048, 36), "Bn1-Bc3-KT36864": (1, 3, 36864), "Bn127-Bc257-KT36864": (127, 257, 36864),
        "real-Bn256-Bc256-KT368640": (256, 256, 368640)}
# (entry point, norms_given); the loss needs Bn <= Bc (target_offset = Bc - Bn)
CLIP_CALLS = [("bm_clip_scores", 0), ("bm_clip_scores", 1), ("bm_clip_scores_det", 0), ("bm_clip_scores_det", 1),
              ("bm_clip_loss_fwd", 0), ("bm_clip_loss_fwd_det", 0)]
CLIP_PARAMS = [pytest.param(c, e, g, id=f"{e}-{'norms_given' if g else 'norms'}-{c}") for c in CLIP
               for e, g in CLIP_CALLS if "loss" not in e or CLIP[c][0] <= CLIP[c][1]]


def _clip_inputs(gen, Bn, Bc, KT):
    """est, cand with candidate Bc // 2 all zero (a padded negative) when Bc >= 3, and that index"""
    est, cand = _rand(gen, Bn, KT), _rand(gen, Bc, KT)
    zero = Bc // 2 if Bc >= 3 else None
    if zero is not None:
        cand[zero] = 0.0
    return est, cand, zero


def _check_inv_norm(inv, cand, zero):
    """fp64 sum of squares (its order's error below KT 2^-53), then (float)sqrt, + 1e-8f and 1 / .: three fp32 roundings"""
    ref = 1.0 / (EPS + cand.double().pow(2).sum(1).sqrt())
    n = 3
    _check("inv_norm", inv, ref, (n * U / (1 - n * U) + cand.shape[1] * UD) * ref)
    if zero is not None:
        assert inv[zero].item() == INV_ZERO, "inv_norm of the all-zero candidate is not 1 / 1e-8f"


@pytest.mark.parametrize("form", FORMS, ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("case,entry,given", CLIP_PARAMS)
def test_clip_fwd(case, entry, given, form):
    call, ptr, stream, lib = _abi()
    Bn, Bc, KT = CLIP[case]
    per, ks = _clip_geometry(Bn, Bc, KT)
    gen = _gen(71)
    est, cand, zero = _clip_inputs(gen, Bn, Bc, KT)
    nws = int(lib.bm_clip_workspace(Bn, Bc, KT))
    ws = torch.full((nws,), float("nan"), device=DEV)
    status = _status()
    loss_fwd = "loss" in entry
    off = Bc - Bn
    inv_given = (1.0 / (1e-8 + cand.double().norm(dim=1))).float()

    def run():
        outs = [Out(Bc), Out(Bn, Bc), Out(Bn, Bc)] + ([Out(Bn), Out(1)] if loss_fwd else [])
        if given:
            outs[0].v.copy_(inv_given)
        p = [ptr(o.t) for o in outs]
        if loss_fwd:
            call(entry + form, ptr(est), ptr(cand), Bn, Bc, KT, off, *p, ptr(ws), nws, ptr(status), stream())
        else:
            call(entry + form, ptr(est), ptr(cand), Bn, Bc, KT, given, *p, ptr(ws), nws, ptr(status), stream())
        torch.cuda.synchronize()
        assert status.item() == 0, f"status {status.item()}"
        return outs

    outs = run()
    inv, scores, probs = (o.v for o in outs[:3])
    if given:
        assert torch.equal(inv, inv_given), "inv_norm (an input) was changed"
    else:
        _check_inv_norm(inv, cand, zero)
    e, c = _ops(form, est, cand)
    i = inv.double()
    ref = (e @ c.T) * i
    mag = (e.abs() @ c.abs().T) * i
    _check_tc("scores", form, scores, ref, _tc_tol(form, mag, per, ks, U * ref.abs()))
    if zero is not None:
        assert (scores[:, zero] == 0).all(), "the all-zero candidate's scores are not exactly 0"
    s = scores.double()
    _check_softmax("probs", probs, s, torch.zeros_like(s), torch.ones_like(s, dtype=torch.bool))
    if loss_fwd:
        # row loss = (logf(sum) + max) - s[target] from the kernel's scores (test_gpu_fma_entry_points.py's bound)
        row_loss, loss = outs[3].v, outs[4].v
        m = s.max(1).values
        lse = torch.logsumexp(s, 1)
        rl = lse - s[torch.arange(Bn, device=DEV), off + torch.arange(Bn, device=DEV)]
        _check("row_loss", row_loss, rl, C_BOUND * U * ((Bc + 4) + 2 * (lse - m).abs() + lse.abs() + rl.abs()) + TINY)
        mean = row_loss.double().mean()        # fp64 sum, one rounding to fp32
        _check("loss", loss, mean.view(1), C_BOUND * U * mean.abs().view(1) + TINY)
    for k, o in enumerate(outs):
        o.untouched(f"output {k}")
    if "_det" in entry:
        ws.copy_(torch.randn(nws, generator=gen, device=DEV))
        again = run()
        assert all(torch.equal(a.v, b.v) for a, b in zip(again, outs)), "det: a second call differs"


# =====================================================================================================================
# CLIP backward: dE = G C and dC = G^T E - coef C, each on the GEMM-NT kernel, the weight-gradient kernel (direct mode,
# G written transposed) or the FP32-FMA GEMM
# =====================================================================================================================
# (Bn, Bc, KT, path of dE, path of dC): clip_dest_gemm takes GEMM-NT for Bn >= 192 and Bc % 4 == 0, else the weight-gradient
# kernel for Bn >= 32, Bn % 4 == 0 and KT a multiple of 128, 192, 256 or 320, else the FMA GEMM; clip_dcand_gemm takes
# GEMM-NT for Bn >= 8 and Bn % 4 == 0, else the weight-gradient kernel (Bc, KT), else the FMA GEMM (KT % 4 == 0 throughout)
CLIP_BWD = {"Bn256-Bc256-KT43200": (256, 256, 43200, "nt", "nt"),
            "Bn192-Bc258-KT43200": (192, 258, 43200, "wgrad", "nt"),
            "Bn191-Bc256-KT43200": (191, 256, 43200, "fma", "wgrad"),
            "Bn64-Bc96-KT43200": (64, 96, 43200, "wgrad", "nt"),
            "Bn100-Bc130-KT36": (100, 130, 36, "fma", "nt"),          # dC: one partial 36-column tile
            "Bn6-Bc9-KT96": (6, 9, 96, "fma", "fma")}
GOUT = 1.7


def _gemm_paths(names):
    """the CLIP backward GEMMs among the kernel names, in launch order"""
    out = []
    for n in names:
        if "hg_gemm_kernel" in n and "GemmNTOp" in n:
            out.append("nt")
        elif "hg_gemm_kernel" in n and "WgradOp" in n:
            out.append("wgrad")
        elif "gemm_simt_kernel" in n:
            out.append("fma")
    return out


def _profiled(run, launched=1):
    """(run(), the GEMM paths it launched); torch.profiler now and then drops kernel records of a session -- all of them,
    or the first ones of a call that launches two GEMMs -- so a session that recorded fewer GEMMs than the `launched` the
    call must run is repeated (run() makes fresh outputs).  What was recorded is asserted by the caller either way."""
    for _ in range(3):
        with _kernels() as names:
            res = run()
        if len(_gemm_paths(names)) >= launched:
            break
    return res, _gemm_paths(names)


def _gemm_tol(form, path, mag, K, gerr):
    """the bound of the GEMM on `path` over a reduction of K, plus G's own error gerr u mag"""
    if path == "fma":
        return 2 * (K + 2) * U * mag + gerr * U * mag + TINY
    return _tc_tol(form, mag, -(-K // 32), 0, gerr * U * mag)


def _bwd_inputs(gen, Bn, Bc, KT):
    est, cand, zero = _clip_inputs(gen, Bn, Bc, KT)
    scores = _rand(gen, Bn, Bc, scale=0.3)
    scores[:, zero] = 0.0                  # as the forward scores an all-zero candidate
    inv = (1.0 / (EPS + cand.double().norm(dim=1))).float()
    inv[zero] = INV_ZERO
    return est, cand, zero, scores, torch.softmax(scores, 1), inv


def _g(kind, Bn, Bc, probs, inv, off, dscores):
    """(G as the kernel computes it in fp32, G in fp64 from the same inputs, G's error in u |G|):
    clip_ce_bwd_kernel: (gout / Bn) (probs - onehot) inv, four roundings; clip_scores_grad_kernel: dscores inv, one"""
    if kind == "ce":
        hot = torch.zeros(Bn, Bc, device=DEV)
        hot[torch.arange(Bn, device=DEV), off + torch.arange(Bn, device=DEV)] = 1.0
        gs = torch.tensor(float(np.float32(GOUT) / np.float32(Bn)), device=DEV)
        g32 = (gs * (probs - hot)) * inv
        g64 = GOUT / Bn * (probs.double() - hot.double()) * inv.double()
        return g32, g64, 4
    return dscores * inv, dscores.double() * inv.double(), 1


def _check_gemm(what, form, path, got, ref, tol):
    """_check_tc where the tensor cores ran, the plain _check on the FMA GEMM (kept out of the tensor-core record)"""
    if path == "fma":
        _check(what, got, ref, tol)
    else:
        _check_tc(what, form, got, ref, tol)


def _gemm_ops(form, path, g32, g64, other):
    """(G, the other operand) of the reference in fp64: G from fp64 for the default form; the kernel's fp32 G for the
    `_tf32` form, rounded to tf32 with the other operand where the tensor cores ran (the FMA GEMM reads them unrounded)"""
    if form == "":
        return g64, other.double()
    if path == "fma":
        return g32.double(), other.double()
    return _ops(form, g32, other)


def _check_dcand(form, path, dcand, coef, g32, g64, gerr, scores, inv, est, cand, zero):
    Bn = est.shape[0]
    # coef = (fmaf chain over Bn of G s) / (1 / inv - 1e-8f), from the fp32 G the kernel read
    gd, sd, invd = g32.double(), scores.double(), inv.double()
    norm = 1.0 / invd - EPS
    live = torch.ones_like(norm, dtype=torch.bool)
    live[zero] = False
    n = torch.where(live, norm, 1.0)
    acc, acc_mag = (gd * sd).sum(0), (gd * sd).abs().sum(0)
    cref = torch.where(live, acc / n, 0.0)
    ctol = C_BOUND * ((Bn + 1) * U * acc_mag / n + cref.abs() * (U / (invd * n) + 2 * U)) + TINY
    _check("coef", coef, cref, torch.where(live, ctol, 0.0))
    assert coef[zero].item() == 0.0, "coef of the all-zero candidate is not 0"
    gg, e = _gemm_ops(form, path, g32, g64, est)
    ref = gg.T @ e - coef.double()[:, None] * cand.double()       # the zero candidate's row: G^T E alone
    mag = gg.abs().T @ e.abs()
    _check_gemm("dcand", form, path, dcand, ref, _gemm_tol(form, path, mag, Bn, gerr) + U * ref.abs())


def _check_dest(form, path, dest, g32, g64, gerr, cand):
    Bc = cand.shape[0]
    gg, c = _gemm_ops(form, path, g32, g64, cand)
    _check_gemm("dest", form, path, dest, gg @ c, _gemm_tol(form, path, gg.abs() @ c.abs(), Bc, gerr))


@pytest.mark.parametrize("form", FORMS, ids=["3xtf32", "tf32"])
@pytest.mark.parametrize("entry", ["bm_clip_loss_bwd", "bm_clip_loss_bwd_cand", "bm_clip_scores_bwd"])
@pytest.mark.parametrize("case", list(CLIP_BWD))
def test_clip_bwd(case, entry, form):
    call, ptr, stream, lib = _abi()
    Bn, Bc, KT, p_dest, p_dcand = CLIP_BWD[case]
    gen = _gen(81)
    est, cand, zero, scores, probs, inv = _bwd_inputs(gen, Bn, Bc, KT)
    off = Bc - Bn
    gout = torch.tensor([GOUT], device=DEV)
    dscores = _rand(gen, Bn, Bc)
    status = _status()
    want_dest, want_dcand = entry != "bm_clip_loss_bwd_cand", entry != "bm_clip_loss_bwd"

    def run():
        G = Out(Bn * Bc)                       # scratch: NaN-filled, guard zones checked
        dest = Out(Bn, KT) if want_dest else None
        dcand, coef = (Out(Bc, KT), Out(Bc)) if want_dcand else (None, None)
        if entry == "bm_clip_loss_bwd":
            call(entry + form, ptr(probs), ptr(inv), ptr(cand), ptr(gout), Bn, Bc, KT, off, ptr(G.t), ptr(dest.t),
                 ptr(status), stream())
        elif entry == "bm_clip_loss_bwd_cand":
            call(entry + form, ptr(probs), ptr(scores), ptr(inv), ptr(est), ptr(cand), ptr(gout), Bn, Bc, KT, off,
                 ptr(G.t), ptr(coef.t), ptr(dcand.t), ptr(status), stream())
        else:
            call(entry + form, ptr(dscores), ptr(scores), ptr(inv), ptr(est), ptr(cand), Bn, Bc, KT, ptr(G.t),
                 ptr(coef.t), ptr(dest.t), ptr(dcand.t), ptr(status), stream())
        torch.cuda.synchronize()
        assert status.item() == 0, f"status {status.item()}"
        return G, dest, dcand, coef

    (G, dest, dcand, coef), paths = _profiled(run, want_dest + want_dcand)
    assert paths == [p_dest] * want_dest + [p_dcand] * want_dcand, f"GEMMs {paths}"
    g32, g64, gerr = _g("scores" if entry == "bm_clip_scores_bwd" else "ce", Bn, Bc, probs, inv, off, dscores)
    if form != "":
        gerr = 0                               # the `_tf32` reference starts from the kernel's own fp32 G
    if want_dest:
        _check_dest(form, p_dest, dest.v, g32, g64, gerr, cand)
        dest.untouched("dest")
    if want_dcand:
        _check_dcand(form, p_dcand, dcand.v, coef.v, g32, g64, gerr, scores, inv, est, cand, zero)
        dcand.untouched("dcand")
        coef.untouched("coef")
    # the scratch holds the last G written, transposed where the last GEMM read it so
    transposed = (want_dcand and p_dcand == "nt") or (not want_dcand and p_dest == "wgrad")
    assert torch.equal(G.v, (g32.T if transposed else g32).reshape(-1)), "G is not the kernel's fp32 G"
    G.untouched("G")
    again = run()
    for a, b, n in ((again[1], dest, "dest"), (again[2], dcand, "dcand"), (again[3], coef, "coef")):
        if b is not None:
            assert torch.equal(a.v, b.v), f"{n}: a second call differs"


# =====================================================================================================================
# A lost pass is seen: structured operands on which 3xTF32 errs by u |xy| per product and one pass by 2^-11 |xy|
# =====================================================================================================================
@pytest.mark.parametrize("engine", ["bm_tc_wgrad", "bm_tc_wgrad_conv", "bm_clip_scores", "gemm_nt"])
def test_lost_pass_is_seen(engine):
    call, ptr, stream, lib = _abi()
    gen = _gen(91)
    status = _status()
    outs = {}
    if engine in ("bm_tc_wgrad", "bm_tc_wgrad_conv"):
        B, T, M, Kw = 4, 64, 128, 3
        N = 96 if engine == "bm_tc_wgrad_conv" else 128
        dy, x = _structured(gen, B, T, M), _structured(gen, B, T, N)
        if engine == "bm_tc_wgrad":
            nws = int(lib.bm_tc_wgrad_workspace(B, M, N, Kw))
            bchunk, ks = _wgrad_geometry(B, M, N, Kw)
            nblk = bchunk * -(-T // 32)
        else:
            nws = int(lib.bm_tc_wgrad_conv_workspace(B, T, M, N, Kw))
            nblk, ks = _wgradp_geometry(B, T, M, N, Kw)
        ws = torch.full((nws,), float("nan"), device=DEV)
        for form in FORMS:
            dw = Out(M, N, Kw)
            extra = [None] if engine == "bm_tc_wgrad" else []            # dbias
            call(engine + form, ptr(dy), ptr(x), B, T, M, N, N, Kw, 1, ptr(ws), ptr(dw.t), *extra, ptr(status), stream())
            outs[form] = dw
        ref, mag = _wgrad_ref(dy.double(), x.double(), Kw, 1, N)
        tol = _tc_tol("", mag, nblk, ks)
    elif engine == "bm_clip_scores":
        Bn, Bc, KT = 128, 128, 4096
        est, cand = _structured(gen, Bn, KT), _structured(gen, Bc, KT)
        nws = int(lib.bm_clip_workspace(Bn, Bc, KT))
        ws = torch.full((nws,), float("nan"), device=DEV)
        inv = torch.ones(Bc, device=DEV)
        for form in FORMS:
            scores, probs = Out(Bn, Bc), Out(Bn, Bc)
            call(engine + form, ptr(est), ptr(cand), Bn, Bc, KT, 1, ptr(inv), ptr(scores.t), ptr(probs.t), ptr(ws), nws,
                 ptr(status), stream())
            outs[form] = scores
        ref = est.double() @ cand.double().T
        per, ks = _clip_geometry(Bn, Bc, KT)
        tol = _tc_tol("", ref.abs(), per, ks, U * ref.abs())
    else:                                      # dE on GEMM-NT: G = dscores * 1 exactly
        Bn, Bc, KT = 192, 256, 4096
        dscores, cand = _structured(gen, Bn, Bc), _structured(gen, Bc, KT)
        inv = torch.ones(Bc, device=DEV)
        G = torch.full((Bn * Bc,), float("nan"), device=DEV)

        def run(form):
            dest = Out(Bn, KT)
            call("bm_clip_scores_bwd" + form, ptr(dscores), None, ptr(inv), None, ptr(cand), Bn, Bc, KT, ptr(G), None,
                 ptr(dest.t), None, ptr(status), stream())
            torch.cuda.synchronize()
            return dest

        outs[""], paths = _profiled(lambda: run(""))
        assert paths == ["nt"], f"GEMMs {paths}"
        outs["_tf32"] = run("_tf32")
        ref = dscores.double() @ cand.double()
        tol = _tc_tol("", ref.abs(), -(-Bc // 32), 0)
    torch.cuda.synchronize()
    assert status.item() == 0, f"status {status.item()}"
    assert (tol < 2.0 ** -13 * ref.abs()).all(), "the bound is too loose to see a lost pass here"
    _check_tc(engine, "", outs[""].v, ref, tol)
    one = outs["_tf32"].v.double()
    assert not torch.isnan(one).any()
    assert ((one - ref).abs() > tol).all(), "the one-pass (`_tf32`) output meets the 3xTF32 bound somewhere"
