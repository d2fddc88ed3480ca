"""GPU checks of the negative pool's entry points and of the drop-in NegativePool in training steps:
  (a) bm_clip_loss_fwd_pooled[_det] and bm_clip_loss_bwd_pooled in each operand mode against an fp64 definition, element by
      element, over shuffled and repeated slots, candidate counts either side of the 128-wide tiles and odd ones;
  (b) the pooled forms bitwise equal to the contiguous forms on `materialize()` (the backward where the contiguous form
      also runs its Bn >= 192 GEMM);
  (c) training steps of a small clip_conv SimpleConv with a pool against the same steps fed by the reference's host pool
      (oracle/negative_pool_oracle.py), under torch.use_deterministic_algorithms(True);
  (d) bitwise repeatability of such runs, and (e) one pool allocation."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MODES = ["default", "det", "tf32", "bf16"]
SUFFIX = {"default": "", "det": "_det", "tf32": "_tf32", "bf16": "_bf16"}
TOL = {"default": 2e-5, "det": 2e-5, "tf32": 4e-3, "bf16": 3e-2}
SHAPES = [(1, 127), (64, 128), (64, 129), (191, 255), (192, 256), (256, 257), (192, 195), (1, 1), (256, 256)]


def _lib():
    from brainmagick_b200 import _lib as L
    return L


def _fwd_name(mode, pooled):
    base = "bm_clip_loss_fwd_pooled" if pooled else "bm_clip_loss_fwd"
    if mode == "det":
        return base + "_det"
    return base + SUFFIX[mode]


def _bwd_name(mode, pooled):
    base = "bm_clip_loss_bwd_pooled" if pooled else "bm_clip_loss_bwd"
    return base + ("" if mode == "det" else SUFFIX[mode])


def _operands(Bn, Bc, KT, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    Bb = Bn
    n = Bc - Bb
    cap = max(n, 1) + 7
    est = torch.randn(Bn, KT, device="cuda", generator=g)
    batch = torch.randn(Bb, KT, device="cuda", generator=g)
    arena = torch.randn(cap, KT, device="cuda", generator=g)
    host = np.random.default_rng(seed).integers(0, cap, size=n).astype(np.int32)     # shuffled, with repeats
    if n >= 2:
        host[1] = host[0]
    slots = torch.from_numpy(host).cuda()
    return est, batch, arena, slots


def _pooled_fwd(mode, est, batch, arena, slots, Bc):
    L = _lib()
    from brainmagick_b200 import functional as BF
    Bn, KT = est.shape
    out = {k: torch.empty(s, device="cuda") for k, s in
           (("inv", (Bc,)), ("scores", (Bn, Bc)), ("probs", (Bn, Bc)), ("row_loss", (Bn,)), ("loss", (1,)))}
    ws = torch.empty(max(int(L.load().bm_clip_workspace(Bn, Bc, KT)), 2), device="cuda")
    L.call(_fwd_name(mode, True), L.ptr(est), L.ptr(batch), batch.shape[0], L.ptr(arena), L.ptr(slots), Bn, Bc, KT, 0,
           L.ptr(out["inv"]), L.ptr(out["scores"]), L.ptr(out["probs"]), L.ptr(out["row_loss"]), L.ptr(out["loss"]),
           L.ptr(ws), ws.numel(), L.ptr(BF.tc_status_tensor(est.device)), L.stream())
    return out


def _contig_fwd(mode, est, cand):
    L = _lib()
    from brainmagick_b200 import functional as BF
    Bn, KT = est.shape
    Bc = cand.shape[0]
    out = {k: torch.empty(s, device="cuda") for k, s in
           (("inv", (Bc,)), ("scores", (Bn, Bc)), ("probs", (Bn, Bc)), ("row_loss", (Bn,)), ("loss", (1,)))}
    ws = torch.empty(max(int(L.load().bm_clip_workspace(Bn, Bc, KT)), 2), device="cuda")
    L.call(_fwd_name(mode, False), L.ptr(est), L.ptr(cand), Bn, Bc, KT, 0, L.ptr(out["inv"]), L.ptr(out["scores"]),
           L.ptr(out["probs"]), L.ptr(out["row_loss"]), L.ptr(out["loss"]), L.ptr(ws), ws.numel(),
           L.ptr(BF.tc_status_tensor(est.device)), L.stream())
    return out


def _pooled_bwd(mode, fwd, batch, arena, slots, gout, Bn, Bc, KT):
    L = _lib()
    from brainmagick_b200 import functional as BF
    G = torch.full((Bn, (Bc + 3) // 4 * 4), float("nan"), device="cuda")
    dest = torch.empty(Bn, KT, device="cuda")
    L.call(_bwd_name(mode, True), L.ptr(fwd["probs"]), L.ptr(fwd["inv"]), L.ptr(batch), batch.shape[0], L.ptr(arena),
           L.ptr(slots), L.ptr(gout), Bn, Bc, KT, 0, L.ptr(G), L.ptr(dest), L.ptr(BF.tc_status_tensor(batch.device)),
           L.stream())
    return dest


def _contig_bwd(mode, fwd, cand, gout, Bn, Bc, KT):
    L = _lib()
    from brainmagick_b200 import functional as BF
    G = torch.empty(Bn * Bc, device="cuda")
    dest = torch.empty(Bn, KT, device="cuda")
    L.call(_bwd_name(mode, False), L.ptr(fwd["probs"]), L.ptr(fwd["inv"]), L.ptr(cand), L.ptr(gout), Bn, Bc, KT, 0,
           L.ptr(G), L.ptr(dest), L.ptr(BF.tc_status_tensor(cand.device)), L.stream())
    return dest


def _fp64(est, cand, gout):
    e, c = est.double(), cand.double()
    inv = 1.0 / (1e-8 + c.norm(dim=1))
    s = (e @ c.t()) * inv
    p = torch.softmax(s, dim=1)
    Bn = e.shape[0]
    idx = torch.arange(Bn, device=e.device)
    row = torch.logsumexp(s, dim=1) - s[idx, idx]
    g = p.clone()
    g[idx, idx] -= 1
    dest = (g * inv * (float(gout) / Bn)) @ c
    return dict(inv=inv, scores=s, probs=p, row_loss=row, loss=row.mean().reshape(1)), dest


def _close(got, ref, tol, what, scale=None):
    """|got - ref| <= tol * (scale + |ref|) element by element; scale defaults to max |ref|"""
    ref = ref.to(got.device)
    scale = (ref.abs().max().item() if scale is None else scale) + 1e-30
    err = (got.double() - ref).abs()
    bad = err > tol * scale + tol * ref.abs()
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, max err {err.max().item():.3e} (scale {scale:.3e})"


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Bn,Bc", SHAPES)
def test_pooled_entry_points_against_fp64(mode, Bn, Bc):
    KT = 4 * 97
    est, batch, arena, slots = _operands(Bn, Bc, KT, seed=Bn * 1000 + Bc)
    cand = torch.cat([batch, arena[slots.long()]])
    gout = torch.tensor([0.75], device="cuda")
    fwd = _pooled_fwd(mode, est, batch, arena, slots, Bc)
    dest = _pooled_bwd(mode, fwd, batch, arena, slots, gout, Bn, Bc, KT)
    torch.cuda.synchronize()
    ref, ref_dest = _fp64(est, cand, 0.75)
    tol = TOL[mode]
    _close(fwd["inv"], ref["inv"], 1e-6, "inv_norm")           # fp64 sums of squares in every mode
    # a score is a dot product of est_b with a unit vector: its rounding error scales with ||est_b||, not with the score
    enorm = est.double().norm(dim=1).max().item()
    for k in ("scores", "probs", "row_loss", "loss"):
        _close(fwd[k], ref[k], tol, k, scale=enorm)
    _close(dest, ref_dest, tol, "dest")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Bn,Bc", SHAPES)
def test_pooled_forms_bitwise_equal_contiguous_forms(mode, Bn, Bc):
    KT = 4 * 97
    est, batch, arena, slots = _operands(Bn, Bc, KT, seed=7 + Bn + Bc)
    cand = torch.cat([batch, arena[slots.long()]])
    gout = torch.tensor([1.0], device="cuda")
    a = _pooled_fwd(mode, est, batch, arena, slots, Bc)
    b = _contig_fwd(mode, est, cand)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    if Bn >= 192 and Bc % 4 == 0:          # the contiguous form's GemmNTOp path
        da = _pooled_bwd(mode, a, batch, arena, slots, gout, Bn, Bc, KT)
        db = _contig_bwd(mode, b, cand, gout, Bn, Bc, KT)
        assert torch.equal(da, db)


# ---- training steps -----------------------------------------------------------------------------------------------
B, T, NEG = 32, 60, 80


def _model():
    import brainmagick_b200 as bb
    from oracle import bm_oracle
    cfg = bm_oracle.Config(in_channels=40, out_channels=128, n_subjects=3, hidden=160, merger_channels=48,
                           initial_linear=24, merger_pos_dim=128)
    model = bb.SimpleConv(
        in_channels=dict(meg=cfg.in_channels), out_channels=cfg.out_channels, hidden=dict(meg=cfg.hidden),
        depth=cfg.depth, dilation_period=cfg.dilation_period, kernel_size=3, skip=True, subject_layers=True,
        subject_dim=0, complex_out=True, glu=2, glu_context=1, merger=True, initial_linear=cfg.initial_linear,
        merger_channels=cfg.merger_channels, gelu=True, batch_norm=True, merger_pos_dim=cfg.merger_pos_dim,
        n_subjects=cfg.n_subjects)
    model.load_state_dict(bm_oracle.init_state_dict(cfg, seed=1))
    return cfg, model.cuda()


def _batch(cfg, i):
    from brainmagick_b200 import synthetic
    from oracle import bm_oracle
    d = bm_oracle.synthetic_batch(cfg, batch=B, T=T, seed=100 + i)
    d["rec_positions"] = synthetic.normalised_positions(cfg.n_subjects, cfg.in_channels, seed=3)
    meg = d["meg"].cuda()
    batch = synthetic.make_batch(meg, d["subject_index"].cuda(), d["rec_positions"], d["rec_of_sample"])
    return meg, batch, d["ban_centre"], d["candidates"].cuda()


def _step(model, clip, cfg, i, training, pool):
    meg, batch, centre, output = _batch(cfg, i)
    model.train(training)
    clip.train(training)
    model.merger.ban_centre_override = centre
    model.zero_grad(set_to_none=True)
    est = model(dict(meg=meg), batch)
    cand = pool.complete(output, training)
    loss = clip(est, cand, torch.ones(B, 1, T, dtype=torch.bool, device="cuda"))
    if training:
        loss.backward()
    return loss.detach().clone(), {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}


PHASES = [True, True, True, False, True, True, False, True]


def test_training_steps_match_the_host_pool():
    import brainmagick_b200 as bb
    from oracle.negative_pool_oracle import HostNegativePool
    torch.use_deterministic_algorithms(True)
    try:
        cfg, model = _model()
        clip = bb.ClipLoss().cuda()
        pool, host = bb.NegativePool(NEG), HostNegativePool(NEG)
        opt = torch.optim.SGD(model.parameters(), lr=1e-3)
        torch.manual_seed(5)
        for i, training in enumerate(PHASES):
            rng = torch.get_rng_state()
            loss_a, grads_a = _step(model, clip, cfg, i, training, pool)
            torch.set_rng_state(rng)
            loss_b, grads_b = _step(model, clip, cfg, i, training, host)
            assert torch.equal(loss_a, loss_b), (i, loss_a.item(), loss_b.item())
            assert grads_a.keys() == grads_b.keys()
            for n in grads_a:
                err = (grads_a[n] - grads_b[n]).abs().max().item()
                assert err <= 1e-5 * max(grads_b[n].abs().max().item(), 1.0), (i, n, err)
            for phase in ("train", "valid"):
                want = host.negative_pool[phase]
                got = pool.buffer(phase)
                assert got.shape == want.shape and torch.equal(got.cpu(), want.cpu()), (i, phase)
            if training:
                opt.step()
    finally:
        torch.use_deterministic_algorithms(False)


def _run(steps):
    import brainmagick_b200 as bb
    cfg, model = _model()
    clip = bb.ClipLoss().cuda()
    pool = bb.NegativePool(NEG)
    opt = torch.optim.SGD(model.parameters(), lr=1e-3)
    torch.manual_seed(9)
    losses, mem = [], []
    for i, training in enumerate(PHASES[:steps]):
        loss, grads = _step(model, clip, cfg, i, training, pool)
        if training:
            opt.step()
        losses.append(loss.cpu())
        torch.cuda.synchronize()
        mem.append(torch.cuda.memory_allocated() if training else None)
    return losses, [p.detach().clone() for p in model.parameters()], mem


def test_deterministic_runs_are_bitwise_equal():
    torch.use_deterministic_algorithms(True)
    try:
        la, pa, _ = _run(4)
        lb, pb, _ = _run(4)
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(a, b) for a, b in zip(la, lb))
    assert all(torch.equal(a, b) for a, b in zip(pa, pb))


def test_pool_storage_is_allocated_once():
    _, _, mem = _run(8)
    # both phases have pooled once by step 3 and the candidate count is `negatives` from step 2 on: after that, every
    # training step ends with the same allocation (valid steps hold no gradients and are not compared)
    assert len({m for m in mem[4:] if m is not None}) == 1, mem
