"""Host-side control flow without a GPU (tests/abi_trace.py records the C-ABI call stream of a step): which kernel
families a configuration runs on.  Numerics are the GPU tests' business."""
import pytest

import abi_trace


def test_default_step_prepares_no_fp16_pieces():
    """By default the step runs the fp32 entry points: no amax pass, no fp16 operand preparation, one weight re-layout
    launch per prepared weight set (the forward and data-gradient operands of a layer in the same launch)."""
    calls = abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True)
    names = [c[0] for c in calls]
    assert {"bm_tc_conv1d_persistent", "bm_tc_wgrad_conv", "bm_tc_pointwise_sel", "bm_tc_wgrad_grouped"} <= set(names)
    assert not set(names) & {"bm_amax", "bm_f16_split", "bm_tc_weight_split_f16", "bm_tc_conv1d_f16", "bm_tc_wgrad_conv_f16"}
    assert names.count("bm_tc_conv1d_persistent") >= 30 and names.count("bm_tc_weight_split") >= 17
    producers = [c for c in calls if c[0] in ("bm_bn_gelu_skip_fwd", "bm_bn_gelu_skip_bwd", "bm_glu_bwd")]
    assert producers and all(c[-2] is False for c in producers)          # amax_out == NULL: no max |output| reductions


def test_default_full_size_step_runs_on_tensor_cores_only():
    """At the BASELINE widths no FP32-FMA contraction is left in the step."""
    names = {c[0] for c in abi_trace.simpleconv_step(abi_trace.CONFIGS["full"], True)}
    assert not names & {"bm_conv1d_fwd", "bm_conv1d_bwd_data", "bm_conv1d_bwd_weight", "bm_conv1d_glu_fwd", "bm_head_fwd",
                        "bm_head_bwd", "bm_sensor_chain_fwd", "bm_sensor_chain_bwd", "bm_attention_weights_fwd"}
    assert {"bm_tc_conv1d_persistent", "bm_tc_wgrad_conv", "bm_tc_pointwise_sel", "bm_tc_wgrad_grouped"} <= names


@pytest.mark.parametrize("override", [dict(glu=0), dict(skip=False), dict(gelu=False), dict(complex_out=False),
                                      dict(merger=False), dict(initial_linear=0), dict(subject_layers=False),
                                      dict(subject_layers=False, subject_dim=5)])
def test_ablation_rows_run_through_the_host_path(override):
    """The ablation rows SimpleConv accepts: the host path completes and differs from the default where it should."""
    base = abi_trace.simpleconv_step(abi_trace.CONFIGS["small"], True)
    got = abi_trace.simpleconv_step(abi_trace.CONFIGS["small"], True, **override)
    names = [c[0] for c in got]
    if "glu" in override:
        assert not any("glu" in n for n in names) and len(got) < len(base)
    if "skip" in override:
        fwd = [c for c in got if c[0] == "bm_bn_gelu_skip_fwd"]
        assert fwd and all(c[6] is False for c in fwd)               # x_old == NULL on every layer
    if "gelu" in override:
        assert "bm_bn_gelu_skip_fwd" not in names and "bm_head_fwd" not in names
        assert names.count("bm_bn_act_skip_fwd") == 11                # 10 layers + the head's activation
    if "merger" in override:
        assert "bm_attention_weights_fwd" not in names and "bm_sensor_mix_fwd" not in names
        assert "bm_initial_linear_fwd" in names and "bm_subject_layers_fwd" in names and "bm_subject_layers_bwd" in names
    if "initial_linear" in override:
        assert "bm_initial_linear_fwd" not in names and "bm_sensor_mix_fwd" in names and "bm_sensor_mix_bwd" in names
    if "subject_layers" in override:
        assert "bm_subject_layers_fwd" not in names and "bm_initial_linear_bwd" in names
        assert "bm_sensor_chain_fwd" not in names                      # the fused chain needs all three stages
    if "complex_out" in override:
        assert not any("head" in n for n in names)
        assert names.count("bm_bn_gelu_skip_fwd") == 9                # the 10th layer is a bare convolution


def test_group_layout_matches_bincount_without_a_sync():
    """functional.group_layout = argsort + CSR offsets of the subject / recording groups with static shapes (torch.bincount
    sizes its output from the data: a device->host sync in the middle of the backward pass)."""
    import torch
    from brainmagick_b200.functional import group_layout
    g = torch.Generator().manual_seed(0)
    for n_groups, B in ((27, 256), (4, 7), (175, 1024), (3, 1)):
        idx = torch.randint(0, n_groups, (B,), generator=g, dtype=torch.int32)
        order, off = group_layout(idx, n_groups)
        want = torch.zeros(n_groups + 1, dtype=torch.int64)
        want[1:] = torch.cumsum(torch.bincount(idx.long(), minlength=n_groups), 0)
        assert off.dtype == torch.int32 and torch.equal(off.long(), want)
        assert torch.equal(order.long(), torch.argsort(idx.long(), stable=True))
        for s in range(n_groups):
            assert (idx[order.long()[off[s]:off[s + 1]]] == s).all()
