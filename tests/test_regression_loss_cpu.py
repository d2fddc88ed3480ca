"""CPU checks of the drop-in L1Loss / L2Loss (bm/losses.py:11-26): on the ABI emulator (tests/regression_emulator.py) they
match the verbatim reference's fixtures (oracle/make_regression_golden.py) for every mask form, a time-cropped view and exact
ties; the module surface and the errors; and the C-ABI call stream -- one forward and one backward call per step, with no
host read while a capture is simulated (`functional.capturing` patched, as tests/test_cuda_graph_cpu.py does)."""
import contextlib
import os
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import abi_trace
import regression_emulator
from conftest import GOLDEN_DIR
from test_cuda_graph_cpu import capturing

CASES = ["ragged_mask", "full_mask", "all_true", "all_false", "time_crop", "ties"]


def _fixture(name):
    z = np.load(os.path.join(GOLDEN_DIR, f"regression_{name}.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def _close(got, want, tol=1e-6):
    scale = want.abs().max().item()
    assert (got - want).abs().max().item() <= tol * max(scale, 1e-30), (got, want)


@pytest.mark.parametrize("kind", ["l1", "l2"])
@pytest.mark.parametrize("name", CASES)
def test_drop_in_matches_the_reference_fixture(name, kind):
    import brainmagick_b200 as bb
    f = _fixture(name)
    limit = int(f["limit"])
    est, out = f["est"].clone().requires_grad_(True), f["out"].clone().requires_grad_(True)
    loss_fn = bb.L1Loss() if kind == "l1" else bb.L2Loss()
    with regression_emulator.emulated():
        loss = loss_fn(est[..., limit:], out[..., limit:], f["mask"][..., limit:])
        loss.backward()
    want = f[f"{kind}.loss"]
    if name == "all_false":
        assert torch.isnan(want) and torch.isnan(loss)
        assert not est.grad.any() and not out.grad.any()
        return
    assert abs(loss.item() - want.item()) <= 1e-6 * abs(want.item())
    _close(est.grad, f[f"{kind}.d_est"])
    _close(out.grad, f[f"{kind}.d_out"])


def test_surface_matches_the_reference():
    import brainmagick_b200 as bb
    for cls in (bb.L1Loss, bb.L2Loss):
        loss = cls()
        assert isinstance(loss, torch.nn.Module)
        assert loss.state_dict() == {} and list(loss.parameters()) == []
    assert {"L1Loss", "L2Loss"} <= set(bb.__all__)


def test_errors():
    import brainmagick_b200 as bb
    est, out = torch.randn(2, 3, 8), torch.randn(2, 3, 8)
    mask = torch.ones(2, 1, 8, dtype=torch.bool)
    with pytest.raises(TypeError, match="mask"):
        bb.L1Loss()(est, out)
    with pytest.raises(RuntimeError, match="CUDA"):           # no CPU fallback
        bb.L2Loss()(est, out, mask)
    with regression_emulator.emulated():
        with pytest.raises(TypeError, match="fp32"):
            bb.L1Loss()(est.double(), out.double(), mask)
        with pytest.raises(TypeError, match="bool"):
            bb.L1Loss()(est, out, mask.float())
        with pytest.raises(RuntimeError):                     # does not broadcast, as mask.expand_as in the reference
            bb.L1Loss()(est, out, torch.ones(2, 1, 7, dtype=torch.bool))
        with pytest.raises(IndexError):                       # the reference's output[mask]
            bb.L2Loss()(est, torch.randn(2, 3, 9), mask)
        with pytest.raises(IndexError):
            bb.L2Loss()(est, torch.randn(2, 4, 8), mask)


@pytest.mark.parametrize("kind", ["l1", "l2"])
def test_mask_broadcasts_and_output_gradient_only_when_asked(kind):
    """every broadcast form of the mask, and a 1-D operand, give torch's result"""
    import brainmagick_b200 as bb
    torch.manual_seed(3)
    est, out = torch.randn(3, 4, 11), torch.randn(3, 4, 11)
    ref = torch.nn.L1Loss() if kind == "l1" else torch.nn.MSELoss()
    loss_fn = bb.L1Loss() if kind == "l1" else bb.L2Loss()
    for shape in [(3, 4, 11), (3, 1, 11), (1, 1, 11), (3, 4, 1), (1, 4, 1), (11,)]:
        mask = torch.rand(shape) > 0.3
        mask.view(-1)[0] = True
        e1, e2 = est.clone().requires_grad_(True), est.clone().requires_grad_(True)
        with regression_emulator.emulated():
            got = loss_fn(e1, out, mask)
            got.backward()
        m = mask.expand_as(est)
        want = ref(e2[m], out[m])
        want.backward()
        assert abs(got.item() - want.item()) <= 1e-6 * abs(want.item()), shape
        _close(e1.grad, e2.grad)


def _host_reads_forbidden(monkeypatch):
    """every way the host code of a step could read a tensor's contents raises; the emulated entry points (the device
    side) may"""
    import brainmagick_b200.convseq as CS
    import brainmagick_b200.functional as BF
    device = [False]

    def guarded(name, original):
        def refuse(self, *a, **k):
            if not device[0]:
                raise AssertionError(f"host read: Tensor.{name}")
            return original(self, *a, **k)
        return refuse
    for name in ("item", "tolist", "__bool__", "__int__", "__float__", "__index__", "cpu", "numpy", "nonzero"):
        monkeypatch.setattr(torch.Tensor, name, guarded(name, getattr(torch.Tensor, name)))
    getitem = torch.Tensor.__getitem__

    def no_mask_index(self, idx):
        if not device[0] and any(isinstance(i, torch.Tensor) and i.dtype == torch.bool
                                 for i in (idx if isinstance(idx, tuple) else (idx,))):
            raise AssertionError("boolean-mask indexing reads the True count on the host")
        return getitem(self, idx)
    monkeypatch.setattr(torch.Tensor, "__getitem__", no_mask_index)

    def on_device(call):
        def run(*args):
            device[0] = True
            try:
                return call(*args)
            finally:
                device[0] = False
        return run
    for mod in (BF, CS):
        monkeypatch.setattr(mod, "call", on_device(mod.call))


def _record(fn):
    import brainmagick_b200.functional as BF
    saved = BF._require_cuda_operands
    BF._require_cuda_operands = lambda *ts: None
    try:
        with regression_emulator.encode_emulator._patched_view_ptr(lambda t: c_void_p(t.data_ptr())):
            return abi_trace.record(fn)
    finally:
        BF._require_cuda_operands = saved


@pytest.mark.parametrize("kind", ["l1", "l2"])
def test_each_step_issues_one_forward_and_one_backward_call_and_no_host_read(kind, monkeypatch):
    import brainmagick_b200 as bb
    est_full = torch.randn(4, 6, 40, requires_grad=True)
    out_full = torch.randn(4, 6, 40)
    mask = torch.rand(4, 1, 40) > 0.2
    loss_fn = bb.L1Loss() if kind == "l1" else bb.L2Loss()

    def steps():
        for _ in range(3):
            loss_fn(est_full[..., 5:], out_full[..., 5:], mask[..., 5:]).backward()
    with contextlib.ExitStack() as stack:
        stack.enter_context(capturing(monkeypatch))
        _host_reads_forbidden(monkeypatch)
        trace = _record(steps)
    k = 0 if kind == "l1" else 1
    assert [c[0] for c in trace] == ["bm_masked_loss_fwd", "bm_masked_loss_bwd"] * 3
    fwd, bwd = trace[:2]
    # the cropped views are read in place: their (b, c) strides are the full tensors', the mask's channel stride is 0
    assert fwd[1:12] == [k, True, 240, 40, True, 240, 40, True, 40, 0, 1]
    assert fwd[12:15] == [4, 6, 35]
    assert bwd[1] == k and bwd[14:17] == [4, 6, 35] and bwd[17:19] == [True, False]     # no d_output buffer


def test_encoding_step_issues_no_host_read_under_a_simulated_capture(monkeypatch):
    """An encoding step -- multi-stream SimpleConv on a StaticBatch, L1Loss on estimate[..., limit:] -- on the emulator
    while a capture is simulated: it runs without a host read, and the loss adds exactly one forward and one backward call"""
    import brainmagick_b200 as bb
    from brainmagick_b200 import synthetic
    torch.manual_seed(0)
    B, C, F, T, S, limit = 4, 10, 6, 24, 3, 5
    model = bb.SimpleConv(in_channels=dict(meg=C, features=F), out_channels=C, hidden=dict(meg=16, features=16), depth=2,
                          kernel_size=3, skip=True, subject_layers=True, subject_dim=0, complex_out=True, merger=True,
                          initial_linear=12, merger_channels=12, gelu=True, batch_norm=True, merger_pos_dim=32,
                          n_subjects=S).train()
    meg, feats, subj = torch.randn(B, C, T), torch.randn(B, F, T + 7)[..., 7:], torch.tensor([0, 1, 2, 1])
    batch = synthetic.make_batch(meg, subj, synthetic.normalised_positions(S, C), subj)
    sb = bb.StaticBatch(B, C, S + 2, "cpu").fill_(batch)
    mask = torch.ones(B, 1, T, dtype=torch.bool)
    model.merger.ban_centre_override = torch.rand(2)

    def step():
        est = model(dict(meg=meg, features=feats), sb)
        bb.L1Loss()(est[..., limit:], meg[..., limit:], mask[..., limit:]).backward()
    with regression_emulator.emulated(), capturing(monkeypatch):
        _host_reads_forbidden(monkeypatch)
        step()
        monkeypatch.undo()
    assert all(p.grad is not None for p in model.parameters())
    trace = _record(step)
    assert [c[0] for c in trace if c[0].startswith("bm_masked_loss")] == ["bm_masked_loss_fwd", "bm_masked_loss_bwd"]
