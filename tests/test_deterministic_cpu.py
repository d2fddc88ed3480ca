"""torch.use_deterministic_algorithms(True) without a GPU: which entry points the host code reaches (tests/abi_trace.py), and
that the deterministic call stream computes the reference's numbers (tests/deterministic_emulator.py against the
verbatim-reference fixtures)."""
import pytest
import torch

import abi_trace
import deterministic_emulator
import test_emulated_host_path as host_path
from conftest import GOLDEN_CASES

# entry points whose default form finishes a floating-point reduction with atomics
ATOMIC_FORMS = {"bm_col_stats", "bm_col_sum", "bm_bn_gelu_skip_bwd", "bm_glu_bwd",
                "bm_conv1d_bwd_weight", "bm_initial_linear_bwd", "bm_sensor_chain_bwd", "bm_attention_weights_bwd",
                "bm_head_bwd", "bm_head_bwd_params", "bm_candidate_inv_norms", "bm_clip_scores", "bm_clip_loss_fwd"}
# (entry point, index of a pointer): the atomic reduction that a non-NULL pointer switches on (BatchNorm statistics, a bias
# gradient; bm_bn_act_skip_bwd reduces only with a BatchNorm, i.e. a mean)
ATOMIC_POINTERS = [("bm_tc_conv1d_persistent", 17), ("bm_tc_conv1d_f16", 20), ("bm_conv1d_fwd", 10), ("bm_tc_wgrad", 11),
                   ("bm_bn_act_skip_bwd", 2)]


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def _atomic_calls(trace):
    bad = [c[0] for c in trace if c[0] in ATOMIC_FORMS]
    for name, idx in ATOMIC_POINTERS:
        bad += [f"{name}(pointer {idx})" for c in trace if c[0] == name and c[1 + idx]]
    return bad


ROWS = {"default": {}, "no_merger": dict(merger=False), "no_initial_linear": dict(initial_linear=0),
        "no_subject_layers": dict(subject_layers=False, subject_dim=4), "subsample": dict(subsample_meg_channels=5),
        "relu": dict(gelu=False)}


@pytest.mark.parametrize("cfg", list(abi_trace.CONFIGS))
@pytest.mark.parametrize("row", list(ROWS))
def test_deterministic_step_reaches_no_atomic_reduction(cfg, row, deterministic):
    trace = abi_trace.simpleconv_step(abi_trace.CONFIGS[cfg], True, **ROWS[row])
    assert _atomic_calls(trace) == []
    assert any(c[0].endswith("_det") for c in trace)


def test_flag_off_keeps_the_default_call_stream():
    trace = abi_trace.simpleconv_step(abi_trace.CONFIGS["small"], True)
    assert not any(c[0].endswith("_det") for c in trace)
    assert _atomic_calls(trace)


class _Recording(deterministic_emulator.DeterministicEmulator):
    last = None

    def __init__(self):
        super().__init__()
        _Recording.last = self


@pytest.fixture
def det_emulator(monkeypatch, deterministic):
    """Runs the host-path tests of test_emulated_host_path on the deterministic emulator, flag on."""
    monkeypatch.setattr(host_path.abi_emulator, "Emulator", _Recording)
    yield
    calls = _Recording.last.calls
    assert not (set(calls) & ATOMIC_FORMS), sorted(set(calls) & ATOMIC_FORMS)
    assert any(n.endswith("_det") for n in calls)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_simpleconv_clip_loss_match_reference_deterministically(name, det_emulator):
    host_path.test_default_configuration_on_the_emulator(name)


@pytest.mark.parametrize("name", ["ablation_no_merger", "ablation_no_initial_linear", "ablation_no_subject_layers",
                                  "ablation_subsample_channels", "ablation_relu"])
def test_ablation_rows_match_reference_deterministically(name, det_emulator):
    host_path.test_ablation_rows_on_the_emulator(name)


@pytest.mark.parametrize("case", host_path._deepmel_names())
def test_conv_sequence_matches_reference_deterministically(case, det_emulator):
    host_path.test_deepmel_on_the_emulator(case)
