"""CPU checks of the drop-in FeatureDecodingLoss (bm/losses.py:117-173): on the ABI emulator (tests/decoding_loss_emulator.py)
it matches the verbatim reference's fixtures (oracle/make_decoding_loss_golden.py) for every case; the module surface, the
scalers it takes and the reference's errors; and the C-ABI call stream -- one forward and one backward call per step
whatever the data, no host read while a capture is simulated, one read per eager step, and the class weights copied once
until the scaler's counts change."""
import contextlib
import os
from collections import OrderedDict
from ctypes import c_void_p

import numpy as np
import pytest
import torch

import abi_trace
import decoding_loss_emulator
from conftest import GOLDEN_DIR
from test_cuda_graph_cpu import capturing
from test_regression_loss_cpu import _host_reads_forbidden

CASES = ["cat_k2", "mixed", "mixed_weighted", "all_true", "zero_count", "ignore_index", "time_crop", "zero_weight_only"]


class Feature:
    def __init__(self, name, dimension, cardinality=None):
        self.name, self.dimension, self.cardinality = name, dimension, cardinality
        self.categorical = cardinality is not None
        self.normalizable = not self.categorical
        self.output_dimension = dimension if cardinality is None else cardinality


class Builder(OrderedDict):
    """the slicing surface of bm.features.FeaturesBuilder"""

    def get_slice(self, name, model_output=False):
        start = 0
        for key, f in self.items():
            width = f.output_dimension if model_output else f.dimension
            if key == name:
                return slice(start, start + width)
            start += width

    @property
    def dimension(self):
        return sum(f.dimension for f in self.values())

    @property
    def output_dimension(self):
        return sum(f.output_dimension for f in self.values())


class Counts:
    def __init__(self, counts):
        self.categories_count_ = counts


class Scaler:
    """the two things FeatureDecodingLoss reads of a scaler; counts how often the weights are asked for"""

    def __init__(self, weights, counts):
        self.weights, self.asked = weights, 0
        self.feature_scalers = {name: Counts(c) for name, c in counts.items()}

    def get_categorical_feature_weights(self, name):
        self.asked += 1
        return self.weights[name]


def _fixture(name):
    z = np.load(os.path.join(GOLDEN_DIR, f"decoding_{name}.npz"))
    f = {k: z[k] for k in z.files}
    builder = Builder((str(n), Feature(str(n), int(d), int(c) or None))
                      for n, d, c in zip(f["names"], f["dims"], f["cards"]))
    scaler = None
    if bool(f["weighted"]):
        cats = [n for n, feat in builder.items() if feat.categorical]
        scaler = Scaler({n: torch.from_numpy(f[f"weights{i}"]) for i, n in enumerate(cats)},
                        {n: torch.from_numpy(f[f"counts{i}"]) for i, n in enumerate(cats)})
    return f, builder, scaler


def _close(got, want, tol=2e-6):
    want = torch.as_tensor(want)
    assert torch.equal(torch.isnan(got), torch.isnan(want))
    ok = ~torch.isnan(want)
    if ok.any():
        assert (got[ok] - want[ok]).abs().max().item() <= tol * max(want[ok].abs().max().item(), 1e-30)


def _run(builder, scaler, est, out, mask, limit=0):
    import brainmagick_b200 as bb
    e, o = est.clone().requires_grad_(True), out.clone().requires_grad_(True)
    with decoding_loss_emulator.emulated():
        loss = bb.FeatureDecodingLoss(builder, scaler)(e[..., limit:], o[..., limit:], mask[..., limit:])
        loss.backward()
    return loss, e.grad, o.grad


@pytest.mark.parametrize("name", CASES)
def test_drop_in_matches_the_reference_fixture(name):
    f, builder, scaler = _fixture(name)
    loss, d_est, d_out = _run(builder, scaler, torch.from_numpy(f["est"]), torch.from_numpy(f["out"]),
                              torch.from_numpy(f["mask"]), int(f["limit"]))
    _close(loss.detach().reshape(1), f["loss"].reshape(1))
    _close(d_est, f["d_est"])
    _close(d_out, f["d_out"])


def test_surface_and_the_package_scaler():
    """an empty state_dict, the export, and this package's BatchScaler (fitted counts) as the scaler"""
    import brainmagick_b200 as bb
    from brainmagick_b200.norm import NoOpCategoryCountScaler
    f, builder, ref_scaler = _fixture("mixed_weighted")
    loss_fn = bb.FeatureDecodingLoss(builder, None)
    assert isinstance(loss_fn, torch.nn.Module) and loss_fn.state_dict() == {} and list(loss_fn.parameters()) == []
    assert "FeatureDecodingLoss" in bb.__all__
    scaler = bb.BatchScaler(builder)
    for name, counts in ref_scaler.feature_scalers.items():
        assert isinstance(scaler.feature_scalers[name], NoOpCategoryCountScaler)
        scaler.feature_scalers[name].categories_count_ = counts.categories_count_
    loss, d_est, d_out = _run(builder, scaler, torch.from_numpy(f["est"]), torch.from_numpy(f["out"]),
                              torch.from_numpy(f["mask"]))
    _close(loss.detach().reshape(1), f["loss"].reshape(1))
    _close(d_est, f["d_est"])


def _mixed(B=2, T=9, seed=0):
    torch.manual_seed(seed)
    builder = Builder([("mel", Feature("mel", 3)), ("ph", Feature("ph", 1, 5)), ("pos", Feature("pos", 1, 4))])
    est, out = torch.randn(B, 12, T), torch.randn(B, 5, T)
    out[:, 3] = torch.randint(0, 5, (B, T)).float()
    out[:, 4] = torch.randint(0, 4, (B, T)).float()
    return builder, est, out, torch.rand(B, 1, T) > 0.3


def test_errors():
    import brainmagick_b200 as bb
    builder, est, out, mask = _mixed()
    loss_fn = bb.FeatureDecodingLoss(builder, None)
    with pytest.raises(AssertionError, match="Invalid features dim"):
        loss_fn(est[:, :11], out, mask)
    with pytest.raises(TypeError, match="mask"):
        loss_fn(est, out)
    with pytest.raises(RuntimeError, match="CUDA"):             # no CPU fallback
        loss_fn(est, out, mask)
    with decoding_loss_emulator.emulated():
        with pytest.raises(TypeError, match="fp32"):
            loss_fn(est.double(), out.double(), mask)
        with pytest.raises(TypeError, match="bool"):
            loss_fn(est, out, mask.float())
        with pytest.raises(RuntimeError):                       # mask.expand_as(feature_estimate) in the reference
            loss_fn(est, out, torch.ones(2, 2, 9, dtype=torch.bool))
        with pytest.raises(IndexError):                         # a categorical feature needs a [B, 1, T] mask
            loss_fn(est, out, torch.ones(1, 1, 9, dtype=torch.bool))
        with pytest.raises(AssertionError):                     # assert mask.any()
            loss_fn(est, out, torch.zeros(2, 1, 9, dtype=torch.bool))
        bad = out.clone()
        bad[1, 4, 0] = 4.0                                      # K = 4: assert K > output[:, start].max()
        with pytest.raises(AssertionError, match="'pos'"):
            loss_fn(est, bad, torch.zeros(2, 1, 9, dtype=torch.bool) | (torch.arange(9) == 3))
        bad = out.clone()
        bad[0, 3, 2] = -3.0
        m = mask.clone()
        m[0, 0, 2] = True
        with pytest.raises(IndexError, match="out of bounds"):  # a masked target < 0, not -100
            loss_fn(est, bad, m)
        m[0, 0, 2] = False
        loss_fn(est, bad, m)                                    # unmasked: the reference never looks at it
        with pytest.raises(RuntimeError, match="weight tensor"):
            bb.FeatureDecodingLoss(builder, Scaler({"ph": torch.ones(4), "pos": torch.ones(4)}, {}))(est, out, mask)


def _record(fn):
    import brainmagick_b200.functional as BF
    saved = BF._require_cuda_decoding
    BF._require_cuda_decoding = lambda *ts: None
    try:
        with decoding_loss_emulator.regression_emulator.encode_emulator._patched_view_ptr(
                lambda t: c_void_p(t.data_ptr())):
            return abi_trace.record(fn)
    finally:
        BF._require_cuda_decoding = saved


def test_each_step_issues_one_forward_and_one_backward_call_and_no_host_read_while_captured(monkeypatch):
    import brainmagick_b200 as bb
    builder, est, out, mask = _mixed(B=3, T=20)
    scaler = Scaler({"ph": torch.rand(5), "pos": torch.rand(4)}, {"ph": torch.ones(5), "pos": torch.ones(4)})
    loss_fn = bb.FeatureDecodingLoss(builder, scaler)
    est_full = torch.randn(3, 12, 25, requires_grad=True)
    out_full = torch.cat([torch.randn(3, 5, 5), out], dim=2)

    def steps(masks):
        for m in masks:
            loss_fn(est_full[..., 5:], out_full[..., 5:], m).backward()
    with decoding_loss_emulator.emulated():
        steps([mask])                                           # the eager warm-up builds the table and the weights
    assert scaler.asked == 2
    masks = [mask, torch.ones_like(mask), torch.rand(3, 1, 20) > 0.9]
    with contextlib.ExitStack() as stack:
        stack.enter_context(capturing(monkeypatch))
        _host_reads_forbidden(monkeypatch)
        trace = _record(lambda: steps(masks))
    assert [c[0] for c in trace] == ["bm_decoding_loss_fwd", "bm_decoding_loss_bwd"] * 3
    fwd = trace[0]
    # the cropped views are read in place: the full tensors' (b, c) strides, the mask's channel stride 0
    assert fwd[1:10] == [True, 300, 25, True, 125, 25, True, 20, 0] and fwd[11:13] == [3, 20]
    assert scaler.asked == 2                                    # no weight copy after the warm-up


def test_eager_steps_read_one_flag_word_and_rebuild_the_weights_when_the_counts_change(monkeypatch):
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    builder, est, out, mask = _mixed()
    counts = {"ph": torch.ones(5), "pos": torch.ones(4)}
    scaler = Scaler({"ph": torch.rand(5), "pos": torch.rand(4)}, counts)
    loss_fn = bb.FeatureDecodingLoss(builder, scaler)
    reads, device = [0], [False]
    item = torch.Tensor.item

    def counted(self):
        reads[0] += not device[0]
        return item(self)
    with decoding_loss_emulator.emulated():
        call = BF.call

        def on_device(*args):
            device[0] = True
            try:
                return call(*args)
            finally:
                device[0] = False
        monkeypatch.setattr(BF, "call", on_device)
        monkeypatch.setattr(torch.Tensor, "item", counted)
        for _ in range(3):
            loss_fn(est, out, mask)
        assert reads[0] == 3 and scaler.asked == 2
        counts["ph"].mul_(2)                                    # fitted again in place: a new version
        loss_fn(est, out, mask)
        assert scaler.asked == 4
        scaler.feature_scalers["pos"].categories_count_ = torch.ones(4)
        with capturing(monkeypatch), pytest.raises(RuntimeError, match="eager"):
            loss_fn(est, out, mask)


@pytest.mark.parametrize("code,exc", [(904, AssertionError), (905, AssertionError), (906, IndexError)])
def test_a_captured_step_reports_data_errors_through_the_status_word(monkeypatch, code, exc):
    import brainmagick_b200 as bb
    import brainmagick_b200.functional as BF
    builder, est, out, mask = _mixed()
    loss_fn = bb.FeatureDecodingLoss(builder, None)
    with decoding_loss_emulator.emulated():
        loss_fn(est, out, mask)
        if code == 904:
            mask = torch.zeros_like(mask)
        else:
            out = out.clone()
            out[0, 3, 1] = 7.0 if code == 905 else -2.0
            mask = mask.clone()
            mask[0, 0, 1] = True
        with capturing(monkeypatch):
            loss_fn(est, out, mask)                             # nothing raised while captured
        with pytest.raises(exc):
            BF.check_tc_status(torch.device("cpu"))
        BF.check_tc_status(torch.device("cpu"))                 # the word is cleared
