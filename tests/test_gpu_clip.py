"""GPU: the ClipLoss kernels (csrc/tc_clip.cuh: split-K score GEMM with per-K-block fp32 accumulation + fused
finalize) against fp64 references (torch, test-only) of bm/losses.py:77-114, through the C ABI.

The case that matters most is the SAME-SIGNED one: the tensor core's fp32 accumulator truncates, so a long accumulation of
positive products (a self dot product, a trained estimate against its own candidate) used to come out 1.1e-4 low at the
BASELINE feature size K = F*T = 368 640 (round 1).  Bound here: 3e-5 relative on every score, north-star tolerance 1e-4."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
K_FULL = 1024 * 360


def _abi():
    from brainmagick_b200 import _lib
    from brainmagick_b200 import functional as BF
    return _lib.call, _lib.ptr, _lib.stream, _lib.load(), BF


def _scores_abi(est, cand, inv_given=None, want_probs=False):
    call, ptr, stream, lib, BF = _abi()
    Bn, Bc, KT = est.shape[0], cand.shape[0], est.shape[1]
    n = max(int(lib.bm_clip_workspace(Bn, Bc, KT)), 2)
    ws = torch.full((n,), float("nan"), device=DEV)          # the library must not depend on the scratch's contents
    inv = inv_given.clone() if inv_given is not None else torch.full((Bc,), float("nan"), device=DEV)
    scores = torch.full((Bn, Bc), float("nan"), device=DEV)
    probs = torch.full((Bn, Bc), float("nan"), device=DEV) if want_probs else None
    status = BF.tc_status_tensor(DEV)
    call("bm_clip_scores", ptr(est), ptr(cand), Bn, Bc, KT, 0 if inv_given is None else 1, ptr(inv), ptr(scores),
         ptr(probs), ptr(ws), n, ptr(status), stream())
    torch.cuda.synchronize()
    BF.check_tc_status()
    return scores, inv, probs


def _ref_scores(est, cand):
    c = cand.double()
    inv = 1.0 / (1e-8 + c.norm(dim=1))
    return (est.double() @ c.t()) * inv, inv


@pytest.mark.parametrize("Bn,Bc,KT", [(256, 256, K_FULL), (64, 512, K_FULL), (128, 1024, 36864), (5, 7, 2560),
                                      (100, 300, 1000), (130, 257, 4100), (3, 2, 32), (33, 40, 36)])
def test_scores_random_sign(Bn, Bc, KT):
    g = torch.Generator(device=DEV).manual_seed(Bn * 7 + Bc)
    est = torch.randn(Bn, KT, device=DEV, generator=g)
    cand = torch.randn(Bc, KT, device=DEV, generator=g)
    scores, inv, probs = _scores_abi(est, cand, want_probs=True)
    ref, ref_inv = _ref_scores(est, cand)
    assert rel_err(inv.cpu(), ref_inv.cpu()) < 2e-7
    e = rel_err(scores.cpu(), ref.cpu())
    print(f"[clip scores {Bn}x{Bc}x{KT}] rel_err vs fp64 = {e:.2e}")
    assert e < 2e-5
    assert rel_err(probs.cpu(), torch.softmax(ref, dim=1).cpu()) < 2e-5


@pytest.mark.parametrize("Bc", [256, 2048])
def test_scores_same_signed_products_at_baseline_feature_size(Bc):
    """est_b = cand_b + small noise (what training converges to): every product of the diagonal dot is positive."""
    g = torch.Generator(device=DEV).manual_seed(3)
    Bn = 256
    cand = torch.randn(Bc, K_FULL, device=DEV, generator=g)
    est = cand[:Bn] + 0.1 * torch.randn(Bn, K_FULL, device=DEV, generator=g)
    scores, inv, _ = _scores_abi(est, cand)
    ref, _ = _ref_scores(est, cand)
    d = torch.arange(Bn, device=DEV)
    diag_err = ((scores[d, d].double() - ref[d, d]) / ref[d, d]).abs().max().item()
    bias = ((scores[d, d].double() - ref[d, d]) / ref[d, d]).mean().item()
    print(f"[clip same-signed Bc={Bc}] worst diagonal rel err {diag_err:.2e}, mean (bias) {bias:.2e}")
    assert diag_err < 3e-5
    assert rel_err(scores.cpu(), ref.cpu()) < 3e-5
    # all-positive operands: EVERY dot product is a same-signed sum
    est_p, cand_p = est[:64].abs().contiguous(), cand[:256].abs().contiguous()
    sp, _, _ = _scores_abi(est_p, cand_p)
    rp, _ = _ref_scores(est_p, cand_p)
    worst = ((sp.double() - rp) / rp).abs().max().item()
    print(f"[clip all-positive] worst rel err {worst:.2e}")
    assert worst < 3e-5


def test_given_norms_and_determinism():
    g = torch.Generator(device=DEV).manual_seed(11)
    est = torch.randn(48, 5120, device=DEV, generator=g)
    cand = torch.randn(96, 5120, device=DEV, generator=g)
    s1, inv, _ = _scores_abi(est, cand)
    s2, inv2, _ = _scores_abi(est, cand)
    assert torch.equal(s1, s2) and torch.equal(inv, inv2)            # fixed-order reductions
    s3, _, _ = _scores_abi(est, cand, inv_given=inv)
    assert torch.equal(s1, s3)


@pytest.mark.parametrize("Bn,Bc,KT,off", [(256, 256, K_FULL, 0), (64, 512, 36864, 128), (6, 9, 96, 2), (7, 7, 250, 0)])
def test_loss_forward_and_gradient(Bn, Bc, KT, off):
    """bm_clip_loss_fwd / bm_clip_loss_bwd vs torch fp64 cross-entropy of the fp64 scores (losses.py:104-114)."""
    _, _, _, _, BF = _abi()
    g = torch.Generator(device=DEV).manual_seed(17 + Bn)
    cand = torch.randn(Bc, KT, device=DEV, generator=g)
    # scaled so that the scores are O(1) (the reference's are ~1e-2 at init, a few units when trained): an unscaled
    # estimate at K = 368 640 saturates the softmax and the gradient underflows in fp32 for the reference as well
    est = ((0.5 * cand[off:off + Bn] + torch.randn(Bn, KT, device=DEV, generator=g)) * (8.0 / KT ** 0.5)).requires_grad_(True)
    loss = BF.clip_loss(est, cand, off)
    loss.backward()
    torch.cuda.synchronize()
    BF.check_tc_status()
    e64 = est.detach().double().requires_grad_(True)
    c64 = cand.double()
    sc = (e64 @ c64.t()) / (1e-8 + c64.norm(dim=1))
    ref = torch.nn.functional.cross_entropy(sc, off + torch.arange(Bn, device=DEV))
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-5 * max(1.0, abs(ref.item()))
    e = rel_err(est.grad.cpu(), e64.grad.cpu())
    print(f"[clip loss {Bn}x{Bc}x{KT}] loss {loss.item():.6f} vs {ref.item():.6f}; dE rel_err {e:.2e}")
    assert e < 3e-5


def test_non_fp32_operands_are_refused():
    _, _, _, _, BF = _abi()
    est = torch.randn(4, 64, device=DEV, dtype=torch.float64, requires_grad=True)
    cand = torch.randn(4, 64, device=DEV)
    with pytest.raises(TypeError):
        BF.clip_loss(est, cand, 0)
