"""The drop-in spectral penalty (bm/svd.py: svd_penalty) on the GPU: bm_svd_penalty_fwd / _bwd against the fp64 oracle
(oracle/svd_oracle.py) fed the same CUDA draws, re-drawn by reseeding, at the algorithm's edges (n = 1, n < q, n = q,
m < n, shapes off the block multiples) and on a BASELINE-width clip_conv SimpleConv.  The tolerance is twice the error of
the reference algorithm itself (torch.svd_lowrank's steps in fp32, with autograd) against the same oracle on the same
inputs, or a few fp32 roundings where that error happens to be smaller.  Also: the draws are torch's bit for bit; repeated
calls are bitwise equal; frozen weights keep their term and get no gradient; TF32 and bf16 autocast change nothing; and a
captured training step with the penalty replays bitwise equal to eager."""
import random

import pytest
import torch

import test_gpu_cuda_graph as G
from oracle import svd_oracle

pytestmark = pytest.mark.gpu

Q, NITER = 16, 2
VALUE_FLOOR, GRAD_FLOOR = 2e-6, 2e-5        # a few fp32 roundings: relative to the value, to the largest gradient element


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _draws(weights, seed):
    torch.manual_seed(seed)
    return [torch.randn(min(w.shape[0], w.numel() // w.shape[0]), Q, device="cuda") for w in weights]


def _penalty(weights, seed, proba=1.0):
    from brainmagick_b200 import functional as BF
    for w in weights:
        w.grad = None
    torch.manual_seed(seed)
    value = BF.svd_penalty(weights, Q, NITER, proba)
    value.backward()
    return value.detach(), [None if w.grad is None else w.grad.clone() for w in weights]


def _reference_errors(weights, draws):
    """the reference algorithm's own fp32 error against the oracle on these inputs: (value, [per-weight gradient])"""
    total_ref, total_oracle, errs = 0.0, 0.0, []
    for w, R in zip(weights, draws):
        p = w.detach().reshape(w.shape[0], -1).clone().requires_grad_(True)
        v = svd_oracle.reference_algorithm(p, R, NITER)
        v.backward()
        s2, g = svd_oracle.estimate(p.detach().cpu(), R.cpu(), NITER)
        total_ref += v.item()
        total_oracle += s2
        errs.append((p.grad.cpu().double() - g).abs().max().item() / g.abs().max().item())
    return abs(total_ref - total_oracle) / total_oracle, errs


def _check(weights, seed, proba=1.0):
    draws = _draws(weights, seed)
    value, grads = _penalty(weights, seed, proba)
    want, gw = svd_oracle.penalty([w.detach().cpu() for w in weights], [r.cpu() for r in draws], NITER, proba)
    e_val, e_grads = _reference_errors(weights, draws)
    assert abs(value.item() - want) <= max(2 * e_val, VALUE_FLOOR) * want, (value.item(), want, e_val)
    for i, (w, g, ref, e) in enumerate(zip(weights, grads, gw, e_grads)):
        if not w.requires_grad:
            assert g is None
            continue
        err = (g.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
        assert err <= max(2 * e, GRAD_FLOOR), (i, tuple(w.shape), err, e)
    return value, grads


SHAPES = {
    "n1": [(300, 1, 1)],                      # post_skip: n = 1
    "n_lt_q": [(40, 5), (9, 12)],             # n < q, and a wide one with m < q
    "n_eq_q": [(70, 16), (16, 16)],           # n = q: the exact rule
    "n_q_plus_1": [(37, 17)],                 # the smallest span-chain shape
    "wide": [(17, 333), (64, 1024, 1)],       # m < n: read transposed
    "off_blocks": [(333, 97), (1000, 65, 1), (95, 33, 3)],
    "clip_conv_shapes": [(320, 270, 3), (640, 320, 3), (640, 1024, 1), (270, 270, 1)],
    "mixed": [(300, 1, 1), (37, 17), (17, 333), (40, 5), (333, 97)],
}


@pytest.mark.parametrize("case", list(SHAPES))
def test_entry_points_match_fp64(case):
    torch.manual_seed(3)
    weights = [torch.randn(*s, device="cuda").requires_grad_(True) for s in SHAPES[case]]
    _check(weights, 11)


def test_proba_scales_value_and_gradient():
    torch.manual_seed(3)
    weights = [torch.randn(*s, device="cuda").requires_grad_(True) for s in [(333, 97), (40, 5)]]
    _check(weights, 12, proba=0.25)


def test_draws_are_torchs():
    from brainmagick_b200 import functional as BF
    torch.manual_seed(3)
    weights = [torch.randn(*s, device="cuda") for s in [(320, 960), (640, 1024, 1), (24, 1, 1), (270, 270)]]
    draws = _draws(weights, 5)
    plan = BF.svd_plan(weights, Q, NITER)
    torch.manual_seed(5)
    R = BF.svd_draws(plan, weights[0])
    assert torch.equal(R, torch.cat([r.reshape(-1) for r in draws]))


def _baseline_model():
    import brainmagick_b200 as bb
    torch.manual_seed(0)
    return bb.SimpleConv(in_channels=dict(meg=208), out_channels=1024, n_subjects=27, **G._clip_conv()).cuda()


def _weights(model):
    return [m.weight for _, m in model.named_modules()
            if isinstance(m, (torch.nn.modules.conv._ConvNd, torch.nn.Linear)) and m.weight.numel() >= 256]


def test_rank_deficient_weights_give_sigma1_and_its_gradient():
    """weights with n > q whose range has fewer than q dimensions (rank 8, 10 nonzero rows, all zero): the span holds A's
    range, so the value is σ₁² and the gradient 2 σ₁ u₁ v₁ᵀ of an fp64 SVD of the fp32 weight -- finite, where an
    unguarded Cholesky QR divides by a vanishing pivot"""
    torch.manual_seed(4)
    rank8 = torch.randn(100, 8, device="cuda") @ torch.randn(8, 40, device="cuda")
    rows10 = torch.cat([torch.randn(10, 40, device="cuda"), torch.zeros(190, 40, device="cuda")])
    weights = [w.requires_grad_(True) for w in (rank8, rows10, torch.zeros(60, 50, device="cuda"), rank8.detach().T.contiguous())]
    for seed in range(7, 12):                                   # several draws: rounding must never become a column
        value, grads = _penalty(weights, seed)
        want = 0.0
        for w, g in zip(weights, grads):
            assert torch.isfinite(g).all()
            U, Sv, Vh = torch.linalg.svd(w.detach().double().cpu())
            want += Sv[0].item() ** 2
            ref = 2 * Sv[0] * torch.outer(U[:, 0], Vh[0])
            if Sv[0] == 0:
                assert torch.equal(g, torch.zeros_like(g))
            else:
                err = (g.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
                assert err <= 1e-4, (seed, tuple(w.shape), err)
        assert abs(value.item() - want) <= 1e-5 * want


def test_baseline_clip_conv_matches_fp64_and_is_bitwise_repeatable(monkeypatch):
    from brainmagick_b200 import svd as S
    model = _baseline_model()
    weights = _weights(model)
    assert len(weights) == 18
    v1, g1 = _check(weights, 21)
    monkeypatch.setattr(S, "penalty_rng", random.Random(1234))
    for w in weights:
        w.grad = None
    torch.manual_seed(21)
    v2 = S.svd_penalty(model)
    v2.backward()
    assert torch.equal(v1, v2.detach())
    for w, g in zip(weights, g1):
        assert torch.equal(w.grad, g)


def test_frozen_weights_keep_their_term_and_get_no_gradient():
    torch.manual_seed(3)
    weights = [torch.randn(*s, device="cuda").requires_grad_(True) for s in [(333, 97), (40, 5), (64, 1024, 1)]]
    v_all, _ = _penalty(weights, 13)
    weights[0].requires_grad_(False)
    weights[1].requires_grad_(False)
    v, grads = _check(weights, 13)
    assert torch.equal(v, v_all) and grads[0] is None and grads[1] is None and grads[2] is not None


def test_tf32_and_autocast_change_nothing():
    model = _baseline_model()
    weights = _weights(model)
    v0, g0 = _penalty(weights, 31)
    was = torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32"
    try:
        v1, g1 = _penalty(weights, 31)
    finally:
        torch.backends.cuda.matmul.fp32_precision = was
    with torch.autocast("cuda", dtype=torch.bfloat16):
        v2, g2 = _penalty(weights, 31)
    assert torch.equal(v0, v1) and torch.equal(v0, v2) and v2.dtype == torch.float32
    for a, b, c in zip(g0, g1, g2):
        assert torch.equal(a, b) and torch.equal(a, c)


def test_launch_count_does_not_grow_with_the_weights():
    from brainmagick_b200 import _lib
    counts = []
    for shapes in ([(333, 97)], [(333, 97)] * 40):
        torch.manual_seed(3)
        weights = [torch.randn(*s, device="cuda").requires_grad_(True) for s in shapes]
        _penalty(weights, 1)
        before = _lib.launch_count()
        _penalty(weights, 1)
        counts.append(_lib.launch_count() - before)
    assert counts[0] == counts[1] == 13 + 12


class _PenaltyTrainer(G._Trainer):
    def step(self):
        from brainmagick_b200 import svd as S
        self.opt.zero_grad(set_to_none=True)
        est = self.model(dict(meg=self.meg), self.sb)
        loss = self.clip(est, self.cand, self.mask) + 0.1 * S.svd_penalty(self.model)
        loss.backward()
        self.opt.step()
        return est, loss


def test_captured_step_with_the_penalty_is_bitwise_equal_to_eager(deterministic, monkeypatch):
    from brainmagick_b200 import svd as S
    monkeypatch.setattr(S, "penalty_rng", random.Random(1234))        # every step draws the coin; leave the module's be
    dims = G.CLIP_DIMS
    warm, fresh = G._items(dims, 2, 1), G._items(dims, 3, 2)
    g, e = _PenaltyTrainer(G._clip_conv(), dims), _PenaltyTrainer(G._clip_conv(), dims)
    # the same draws on both sides: every step, warm-up included, starts from its own seed
    graph, (g_est, g_loss) = G._capture(g.step, [lambda it=it, j=j: (g.load(it), torch.manual_seed(50 + j))
                                                 for j, it in enumerate(warm)])
    for j, it in enumerate(warm):
        e.load(it)
        torch.manual_seed(50 + j)
        e.step()
    for i, it in enumerate(fresh):
        g.load(it)
        torch.manual_seed(100 + i)
        graph.replay()
        e.load(it)
        torch.manual_seed(100 + i)
        e_est, e_loss = e.step()
        torch.cuda.synchronize()
        G._assert_bitwise(g.state(g_est, g_loss), e.state(e_est, e_loss), f"step {i}")
