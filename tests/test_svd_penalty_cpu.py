"""CPU checks of the drop-in spectral penalty (bm/svd.py: svd_penalty): the fp64 oracle (oracle/svd_oracle.py) and, on the
ABI emulator (tests/svd_emulator.py), the drop-in match the verbatim reference's fixtures (oracle/make_svd_golden.py) --
value, gradients, the draws bit for bit from the same seed, and penalty_rng's skip pattern; the call stream is the same
two calls for 1 and for 40 weights and, once the weight table is cached, reads nothing on the host; the errors."""
import json
import os
import random

import numpy as np
import pytest
import torch

import svd_emulator
from conftest import GOLDEN_DIR
from oracle import make_svd_golden, svd_oracle
from test_regression_loss_cpu import _host_reads_forbidden

CASES = ["clip_conv", "residual", "layers", "frozen", "proba"]


def load_case(name):
    z = np.load(os.path.join(GOLDEN_DIR, f"svd_{name}.npz"))
    f = {k: z[k] for k in z.files}
    model = make_svd_golden.model_from_spec(json.loads(str(f["model"])))
    weights = make_svd_golden.walk(model)
    with torch.no_grad():
        for i, w in enumerate(weights):
            w.copy_(torch.from_numpy(f[f"w_{i}"]))
    for i in f["frozen"].tolist():
        weights[i].requires_grad_(False)
    return f, model, weights


def _selected(f, weights):
    return [i for i, w in enumerate(weights) if w.numel() / 2**8 >= float(f["min_size"])]


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_the_reference_fixture(name):
    f, _, weights = load_case(name)
    sel = _selected(f, weights)
    for c in range(int(f["calls"])):
        want = float(f[f"value_{c}"])
        if np.isnan(want):
            assert int(f[f"draws_{c}"]) == 0
            continue
        assert int(f[f"draws_{c}"]) == len(sel)
        draws = [torch.from_numpy(f[f"r_{c}_{k}"]) for k in range(len(sel))]
        value, grads = svd_oracle.penalty([weights[i].detach() for i in sel], draws, proba=float(f["proba"]))
        assert abs(value - want) <= 1e-5 * want
        for i, g in zip(sel, grads):
            ref = torch.from_numpy(f[f"g_{c}_{i}"]).double()
            if not weights[i].requires_grad:
                continue
            assert (g - ref).abs().max().item() <= 2e-4 * max(ref.abs().max().item(), 1e-3), (c, i)


@pytest.mark.parametrize("name", CASES)
def test_drop_in_matches_the_reference_fixture(name, monkeypatch):
    from brainmagick_b200 import svd as S
    f, model, weights = load_case(name)
    sel = _selected(f, weights)
    monkeypatch.setattr(S, "penalty_rng", random.Random(1234))
    with svd_emulator.emulated() as emu:
        for c in range(int(f["calls"])):
            for w in weights:
                w.grad = None
            torch.manual_seed(int(f[f"seed_{c}"]))
            n_before = len(emu.draws)
            value = S.svd_penalty(model, min_size=float(f["min_size"]), proba=float(f["proba"]))
            want = float(f[f"value_{c}"])
            if np.isnan(want):                              # the reference's coin skipped this call
                assert value == 0. and isinstance(value, float) and len(emu.draws) == n_before
                continue
            assert isinstance(value, torch.Tensor) and value.dim() == 0 and value.dtype == torch.float32
            assert abs(value.item() - want) <= 1e-5 * want
            # the draws: torch.randn(min(m, n), 16) per selected weight, in order, bit for bit
            R = emu.draws[-1]
            off = 0
            for k, i in enumerate(sel):
                r = torch.from_numpy(f[f"r_{c}_{k}"])
                assert torch.equal(R[off:off + r.numel()].view(r.shape), r), (c, k)
                off += r.numel()
            assert off == R.numel()
            value.backward()
            for i, w in enumerate(weights):
                ref = torch.from_numpy(f[f"g_{c}_{i}"])
                if not w.requires_grad or i not in sel:
                    assert w.grad is None
                    continue
                assert w.grad.shape == w.shape
                assert (w.grad - ref).abs().max().item() <= 2e-4 * max(ref.abs().max().item(), 1e-3), (c, i)


def test_fixture_shapes_cover_the_algorithm_edges():
    """the residual case holds n = 1 < q weights (post_skip), the layers case a wide weight, n = q and skipped weights"""
    f, _, weights = load_case("residual")
    assert any(w.shape[1:] == (1, 1) for w in weights) and len(_selected(f, weights)) == len(weights)
    f, _, weights = load_case("layers")
    shapes = [(w.shape[0], w.numel() // w.shape[0]) for w in weights]
    assert (24, 120) in shapes and (16, 16) in shapes and len(_selected(f, weights)) == len(weights) - 2


def _calls(monkeypatch, model, **kw):
    """the C-ABI calls of one svd_penalty forward and backward after an eager call cached the table, with every host read
    refused"""
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import svd as S
    monkeypatch.setattr(S, "penalty_rng", random.Random(0))
    with svd_emulator.emulated():
        S.svd_penalty(model, **kw).backward()                   # builds and caches the table
        names = []
        inner = BF.call

        def recording(name, *args):
            names.append(name)
            return inner(name, *args)
        monkeypatch.setattr(BF, "call", recording)
        with monkeypatch.context() as m:
            _host_reads_forbidden(m)
            value = S.svd_penalty(model, **kw)
            value.backward()
        return names


@pytest.mark.parametrize("layers", [1, 40])
def test_one_forward_and_one_backward_call_whatever_the_weights(layers, monkeypatch):
    torch.manual_seed(0)
    model = torch.nn.Sequential(*[torch.nn.Linear(24 + k % 3, 20) for k in range(layers)])
    assert _calls(monkeypatch, model, min_size=0.01) == ["bm_svd_penalty_fwd", "bm_svd_penalty_bwd"]


def test_table_is_cached_per_weights_and_shapes_while_they_live():
    import gc

    import brainmagick_b200.functional as BF
    from brainmagick_b200 import svd as S
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(30, 20), torch.nn.Conv1d(4, 40, 3))
    with svd_emulator.emulated():
        S.svd_penalty(model, min_size=0.01)
        S.svd_penalty(model, min_size=0.01)
        assert len(BF._svd_plans) == 1
        model[0].weight.requires_grad_(False)               # another grad flag: another table
        S.svd_penalty(model, min_size=0.01)
        assert len(BF._svd_plans) == 2
        del model
        gc.collect()
        S.svd_penalty(torch.nn.Sequential(torch.nn.Linear(30, 20)), min_size=0.01)
        assert len(BF._svd_plans) == 1                      # the dead model's tables went when the next one was built


def test_table_layout():
    """bm_svd_table: the tall orientation, the exact flag (n <= q), the offsets and the grouped tile counts"""
    from brainmagick_b200 import _lib
    rows, cols, grad = [320, 640, 270, 24, 50], [960, 320, 270, 1, 16], [1, 1, 0, 1, 1]
    W, q = len(rows), 16
    table, sizes = torch.zeros(W, 12, dtype=torch.int64), torch.zeros(7, dtype=torch.int64)
    args = [torch.tensor(v, dtype=torch.int64) for v in ([4096 * (i + 1) for i in range(W)], rows, cols)]
    g = torch.tensor(grad, dtype=torch.int32)
    assert _lib.load().bm_svd_table(W, *(a.data_ptr() for a in args), g.data_ptr(), q, 2, table.data_ptr(),
                                    sizes.data_ptr()) == 0
    t = table.tolist()
    assert [(r[1], r[2], r[3], r[4]) for r in t] == [(960, 320, 1, 0), (640, 320, 0, 0), (270, 270, 0, 0), (24, 1, 0, 1),
                                                     (50, 16, 0, 1)]
    assert [r[7] for r in t] == [0, 320 * q, 640 * q, 910 * q, 911 * q] and sizes[2] == 927 * q
    assert [r[8] for r in t] == [0, 320 * 960, -1, 640 * 320 + 320 * 960, 640 * 320 + 320 * 960 + 24]
    assert sizes[3] == 320 * 960 + 640 * 320 + 24 + 50 * 16
    assert sizes[4] == 30 + 20 + 9 and sizes[5] == 10 + 10 + 9            # exact weights have no product tiles
    assert sizes[6] == 5 * 15 + 10 * 5 + 1 + 1
    bad = torch.tensor([0] * W, dtype=torch.int64)
    assert _lib.load().bm_svd_table(W, bad.data_ptr(), args[1].data_ptr(), args[2].data_ptr(), g.data_ptr(), q, 2,
                                    table.data_ptr(), sizes.data_ptr()) != 0
    assert _lib.load().bm_svd_table(W, args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(), g.data_ptr(), 33, 2,
                                    table.data_ptr(), sizes.data_ptr()) != 0


def test_errors(monkeypatch):
    from brainmagick_b200 import svd as S
    model = torch.nn.Sequential(torch.nn.Linear(30, 20))
    monkeypatch.setattr(S, "penalty_rng", random.Random(1234))
    with pytest.raises(NotImplementedError):
        S.svd_penalty(model, exact=True)
    with pytest.raises(RuntimeError, match="CUDA"):                    # no CPU fallback
        S.svd_penalty(model)
    with pytest.raises(TypeError):
        S.svd_penalty(torch.nn.Sequential(torch.nn.Linear(30, 20).double()))
    with pytest.raises(TypeError):
        S.svd_penalty(torch.nn.Sequential(torch.nn.Linear(30, 20, dtype=torch.complex64)))
    with pytest.raises(NotImplementedError):
        S.svd_penalty(model, dim=33)
    assert S.svd_penalty(model, min_size=1e6) == 0.                     # nothing selected
    want = random.Random(1234)
    for _ in range(7):                                                  # one draw per call above and below
        want.random()
    assert S.svd_penalty(model, proba=0.) == 0.                         # the coin: one draw per call, nothing else
    assert S.penalty_rng.getstate() == want.getstate()


@pytest.mark.parametrize("seed, applies", [(1234, True), (0, False)])
def test_capture_refuses_a_coin_whichever_way_it_falls(seed, applies, monkeypatch):
    """proba < 1 under capture raises whether the coin applies the penalty (Random(1234): 0.966 <= 0.999) or skips it
    (Random(0): 0.844 > 0.5), and the draw is still made, as in the reference"""
    import brainmagick_b200.functional as BF
    from brainmagick_b200 import svd as S
    model = torch.nn.Sequential(torch.nn.Linear(30, 20))
    proba = 0.999 if applies else 0.5
    assert (random.Random(seed).random() <= proba) == applies
    monkeypatch.setattr(S, "penalty_rng", random.Random(seed))
    monkeypatch.setattr(BF, "capturing", lambda: True)
    with svd_emulator.emulated():
        with pytest.raises(RuntimeError, match="captured"):
            S.svd_penalty(model, min_size=0.01, proba=proba)
        want = random.Random(seed)
        want.random()
        assert S.penalty_rng.getstate() == want.getstate()
        with pytest.raises(RuntimeError, match="eager"):                # proba 1: no table cached yet
            S.svd_penalty(model, min_size=0.01)
