"""CPU checks of the drop-in negative pool (bm/solver.py:152-164, 358-371): on the ABI emulator
(tests/negative_pool_emulator.py), `NegativePool.complete` + the drop-in `ClipLoss` match, step by step, what the reference's
pool fed the verbatim reference ClipLoss (oracle/make_negative_pool_golden.py): the candidates and the pool exactly, the
loss and the estimate gradient to fp32 rounding, and the CPU generator's stream.  Also: no host read in a pooled step, the
pooled entry points only when a pool is used, the slot lease across two forwards before either backward, and the errors."""
import os

import numpy as np
import pytest
import torch

import negative_pool_emulator
from conftest import GOLDEN_DIR

CASES = ["fill", "truncate", "phases", "noop", "ragged", "odd"]


def load_case(name):
    z = np.load(os.path.join(GOLDEN_DIR, f"negative_pool_{name}.npz"))
    f = {k: z[k] for k in z.files}
    negatives, pool_size, seed, steps, F, T = (int(v) for v in f["meta"])
    return f, negatives, (None if pool_size < 0 else pool_size), seed, steps


def _step_inputs(f, i, out_grad):
    out = torch.from_numpy(f[f"out_{i}"]).requires_grad_(out_grad)
    est = torch.from_numpy(f[f"est_{i}"]).requires_grad_(True)
    return bool(f[f"train_{i}"]), out, est


def _check_step(f, i, pool, loss, est, out):
    torch.testing.assert_close(loss.detach().reshape(()), torch.from_numpy(f[f"loss_{i}"]).reshape(()), rtol=1e-5,
                               atol=1e-6)
    torch.testing.assert_close(est.grad, torch.from_numpy(f[f"gest_{i}"]), rtol=1e-4, atol=1e-6)
    if out.requires_grad:
        torch.testing.assert_close(out.grad, torch.from_numpy(f[f"gout_{i}"]), rtol=1e-4, atol=1e-6)
    for phase in ("train", "valid"):
        want = torch.from_numpy(f[f"pool_{phase}_{i}"])
        got = pool.buffer(phase)
        assert got.shape == want.shape and torch.equal(got, want), (i, phase)


@pytest.mark.parametrize("name", CASES)
def test_drop_in_matches_the_reference_fixture(name):
    import brainmagick_b200 as bb
    f, negatives, pool_size, seed, steps = load_case(name)
    with negative_pool_emulator.emulated():
        pool = bb.NegativePool(negatives, pool_size)
        clip = bb.ClipLoss()
        torch.manual_seed(seed)
        for i in range(steps):
            training, out, est = _step_inputs(f, i, name == "noop")
            clip.train(training)
            cand = pool.complete(out, training)
            if int(f[f"ran_{i}"]):
                assert isinstance(cand, bb.PooledCandidates)
                want = torch.from_numpy(f[f"cand_{i}"])
                assert cand.shape == want.shape and cand.size() == want.size() and len(cand) == len(want)
                assert cand.size(0) == want.size(0) and cand.dtype == want.dtype and not cand.requires_grad
                assert torch.equal(cand.materialize(), want)
            else:
                assert cand is out
            loss = clip(est, cand, torch.ones(out.shape[0], 1, out.shape[2], dtype=torch.bool))
            loss.backward()
            _check_step(f, i, pool, loss, est, out)
            if not out.requires_grad:
                assert out.grad is None
        assert torch.equal(torch.rand(4), torch.from_numpy(f["final_rand"]))


def _recorded_names(monkeypatch):
    import brainmagick_b200.functional as BF
    names = []
    call = BF.call

    def record(name, *args):
        names.append(name)
        return call(name, *args)
    monkeypatch.setattr(BF, "call", record)
    return names


POOLED = {"bm_scatter_rows", "bm_clip_loss_fwd_pooled", "bm_clip_loss_bwd_pooled"}


@pytest.mark.parametrize("name", ["fill", "noop"])
def test_pooled_entry_points_only_when_a_pool_is_used(name, monkeypatch):
    import brainmagick_b200 as bb
    f, negatives, pool_size, seed, steps = load_case(name)
    with negative_pool_emulator.emulated():
        names = _recorded_names(monkeypatch)
        pool = bb.NegativePool(negatives, pool_size)
        clip = bb.ClipLoss()
        torch.manual_seed(seed)
        for i in range(steps):
            training, out, est = _step_inputs(f, i, False)
            names.clear()
            clip.train(training)
            cand = pool.complete(out, training)
            clip(est, cand, torch.ones(out.shape[0], 1, out.shape[2], dtype=torch.bool)).backward()
            if int(f[f"ran_{i}"]):
                assert names == ["bm_scatter_rows", "bm_clip_loss_fwd_pooled", "bm_clip_loss_bwd_pooled"]
            else:
                assert names == ["bm_clip_loss_fwd", "bm_clip_loss_bwd"]
    assert bb.NegativePool(None).complete(out, True) is out


def test_pooled_step_reads_nothing_on_the_host(monkeypatch):
    """complete + forward + backward: no Tensor.item / tolist / cpu / bool (or int / float / index) outside the entry
    points, once the mask object has been checked (the reference's `assert mask.all()`, kept per mask object)"""
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    f, negatives, pool_size, seed, steps = load_case("fill")
    with negative_pool_emulator.emulated():
        pool = bb.NegativePool(negatives, pool_size)
        clip = bb.ClipLoss().train()
        mask = torch.ones(3, 1, 10, dtype=torch.bool)
        torch.manual_seed(seed)
        _, out, est = _step_inputs(f, 0, False)
        clip(est, pool.complete(out, True), mask).backward()
        device = [False]

        def guarded(name, original):
            def refuse(self, *a, **k):
                if not device[0]:
                    raise AssertionError(f"host read: Tensor.{name}")
                return original(self, *a, **k)
            return refuse
        for name in ("item", "tolist", "cpu", "__bool__", "__int__", "__float__", "__index__"):
            monkeypatch.setattr(torch.Tensor, name, guarded(name, getattr(torch.Tensor, name)))
        call = BF.call

        def on_device(*args):
            device[0] = True
            try:
                return call(*args)
            finally:
                device[0] = False
        monkeypatch.setattr(BF, "call", on_device)
        for i in range(1, steps):
            _, out, est = _step_inputs(f, i, False)
            cand = pool.complete(out, True)
            loss = clip(est, cand, mask)
            loss.backward()
            monkeypatch.undo()
            _check_step(f, i, pool, loss, est, out)
            for name in ("item", "tolist", "cpu", "__bool__", "__int__", "__float__", "__index__"):
                monkeypatch.setattr(torch.Tensor, name, guarded(name, getattr(torch.Tensor, name)))
            monkeypatch.setattr(BF, "call", on_device)


def test_two_forwards_then_two_backwards_keep_the_drawn_rows():
    """With pool size = negatives the rows a step draws can leave the pool at the next step; while the first step's graph
    is alive, the second step's new rows must not overwrite them (the lease)."""
    import brainmagick_b200 as bb
    f, negatives, pool_size, seed, steps = load_case("truncate")
    with negative_pool_emulator.emulated():
        pool = bb.NegativePool(negatives, pool_size)
        clip = bb.ClipLoss().train()
        torch.manual_seed(seed)
        for i in range(0, steps - 1, 2):
            pending = []
            for j in (i, i + 1):
                _, out, est = _step_inputs(f, j, False)
                cand = pool.complete(out, True)
                pending.append((j, clip(est, cand, torch.ones(3, 1, out.shape[2], dtype=torch.bool)), est, out))
                del cand
            for j, loss, est, out in pending:
                loss.backward()
                torch.testing.assert_close(loss.detach(), torch.from_numpy(f[f"loss_{j}"]).reshape(()), rtol=1e-5,
                                           atol=1e-6)
                torch.testing.assert_close(est.grad, torch.from_numpy(f[f"gest_{j}"]), rtol=1e-4, atol=1e-6)
            assert torch.equal(pool.buffer("train"), torch.from_numpy(f[f"pool_train_{i + 1}"]))


def test_errors(monkeypatch):
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import distrib
    with pytest.raises(AssertionError, match="Pool of negatives should be larger"):
        bb.NegativePool(4, 3)
    assert bb.NegativePool(4).negative_pool_size == 8
    with negative_pool_emulator.emulated():
        pool = bb.NegativePool(4)
        est = torch.randn(2, 4, 8, requires_grad=True)
        cand = pool.complete(torch.randn(2, 4, 8), True)
        mask = torch.ones(2, 1, 8, dtype=torch.bool)
        with pytest.raises(RuntimeError) as want:          # the reference's torch.cat error
            torch.cat([torch.randn(2, 4, 9), torch.randn(1, 4, 8)])
        with pytest.raises(RuntimeError) as got:
            pool.complete(torch.randn(2, 4, 9), True)
        assert str(got.value) == str(want.value)
        monkeypatch.setattr(distrib, "world_size", lambda: 2)
        with pytest.raises(NotImplementedError):
            bb.ClipLoss(global_negatives=True)(est, cand, mask)
        monkeypatch.undo()
        monkeypatch.setattr(BF, "capturing", lambda: True)
        with pytest.raises(RuntimeError, match="CUDA graph"):
            bb.ClipLoss()(est, cand, mask)
        out = torch.randn(2, 4, 8)
        state = torch.get_rng_state()
        with pytest.raises(RuntimeError, match="CUDA graph"):
            pool.complete(out, True)
        assert torch.equal(torch.get_rng_state(), state)    # refused before drawing
